"""Throughput of fully observable observations (bb_pool_full_obs / k_full_obs, FullyObsWrapper) on one GPU.

Prints one JSON line: the card and its power limit (read in the same run); per config (every env, and id lists of 1 / 32 /
1 024 envs) the time per call (CUDA events around back-to-back calls after a warm-up, at least --min-seconds timed), the bytes
one call must move computed from shapes (reads: each selected env's W H grid bytes and its 16-byte pose record; writes: the
3 W H-byte image), the achieved bandwidth and its fraction of the H100 SXM data-sheet 3 350 GB/s; and the time of one
DeviceParallelEnv.step of the 65 536-env GoToLocal pool with and without FullyObsWrapper.

usage: python scripts/bench_full_obs.py [--min-seconds 1.0]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_render_grid import PEAK_GBS, card  # noqa: E402

POOLS = [('GoToLocal', 65536), ('BossLevel', 32768)]
SELECTIONS = [None, 1, 32, 1024]


def timed(fn, min_seconds):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls = 4
    while True:
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= 1000.0 * min_seconds:
            return ms / calls, calls
        calls = max(calls * 2, int(calls * 1000.0 * min_seconds / max(ms, 1e-3) * 1.2))


def run_pool(level, n, min_seconds):
    import numpy as np
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64))
    env.reset()
    rng = np.random.RandomState(0)
    for _ in range(10):                           # states away from the first ones
        env.step(torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=env.device))
    W, H = env.width, env.height
    out = []
    for sel in SELECTIONS:
        ids = None if sel is None else rng.randint(0, n, sel).astype(np.int32)
        m = n if sel is None else sel
        buf = torch.empty((m, W, H, 3), dtype=torch.uint8, device=env.device)
        per_call, calls = timed(lambda: env.full_obs(ids, out=buf), min_seconds)
        nbytes = m * (W * H + 16) + m * 3 * W * H
        gbs = nbytes / (per_call * 1e-3) / 1e9
        out.append(dict(level=level, envs=n, selected='all' if sel is None else sel, image_shape=[W, H, 3], calls_timed=calls,
                        ms_per_call=round(per_call, 5), bytes_per_call=nbytes, achieved_gbs=round(gbs, 1),
                        fraction_of_3350=round(gbs / PEAK_GBS, 3)))
    assert env.counters()['errors'] == 0
    env.close()
    torch.cuda.empty_cache()
    return out


def run_facade(full, steps=200):
    import numpy as np
    import torch
    import babyai_b200 as bb
    from babyai_b200.learner import DeviceParallelEnv
    n = 65536
    envs = bb.make_envs('GoToLocal', n, seed=1)
    dev = DeviceParallelEnv(bb.FullyObsWrapper(envs) if full else envs)
    dev.reset()
    acts = np.random.RandomState(1).randint(0, 7, (steps + 20, n)).astype(np.int8)
    for t in range(20):
        next(dev.step(acts[t]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(20, steps + 20):
        obs = next(dev.step(acts[t]))
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    out = dict(wrapper='FullyObsWrapper' if full else 'none', envs=n, steps=steps, image_shape=list(obs.image.shape[1:]),
               ms_per_step=round(ms, 4), fused_io=dev.fused_io)
    del dev
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--min-seconds', type=float, default=1.0)
    args = ap.parse_args()
    from babyai_b200 import build
    build.build()
    name, power = card()
    configs = [c for level, n in POOLS for c in run_pool(level, n, args.min_seconds)]
    facade = [run_facade(full) for full in (False, True, False, True)]
    print(json.dumps(dict(metric='full_obs', gpu=name, power_limit=power, configs=configs, device_parallel_env_step=facade)))


if __name__ == '__main__':
    main()
