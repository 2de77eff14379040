"""Cost of selected steps (bb_pool_step_envs) against a full bb_pool_step of the same pool, on one GPU.

Prints one JSON line: the card and its power limit (read in the same run), then per pool and mode the time of one step_envs
call for n_sel in {1, 32, 1024, 4096, n_envs} (n_envs takes several k_step8_sel launches) beside the time of one bb_pool_step
of the whole pool.  Each figure: CUDA events around back-to-back calls on the current stream after a warm-up, about a second
of calls, with the host's enqueue time per call beside it, and the device time of the k_step8_sel launches per call from
torch.profiler in a run of its own.  In auto-reset mode the figures include the generation passes the per-step schedule forks every G calls; in freeze
mode the pool is reset before each figure (a frozen env's step is a replay).

usage: python scripts/bench_step_envs.py [--pools GoToLocal:65536,BossLevel:32768] [--seconds 1.0]"""
import argparse
import json
import os
import sys

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_render_grid import card  # noqa: E402


def timed(call, seconds):
    """(ms per call, host ms per call, calls): a warm-up, a probe of 10 calls, then about `seconds` of back-to-back calls
    between two CUDA events; the host figure is the wall time of enqueueing them (when it equals the first, the host bounds
    the calls)"""
    import time
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(10):
        call()
    ev1.record()
    torch.cuda.synchronize()
    calls = max(10, int(seconds * 1000 / max(ev0.elapsed_time(ev1) / 10, 1e-3)))
    ev0.record()
    t0 = time.perf_counter()
    for _ in range(calls):
        call()
    host = time.perf_counter() - t0
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / calls, host * 1000 / calls, calls


def kernel_ms(call, name, calls=20):
    """device time of the kernels whose name contains `name`, per call (torch.profiler, a run of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
        torch.cuda.synchronize()
    us = sum(getattr(e, 'device_time_total', 0) for e in prof.key_averages() if name in e.key)
    return us / calls / 1000


def measure(level, n, seconds):
    import numpy as np
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64))
    rng = np.random.RandomState(0)
    acts = torch.as_tensor(rng.randint(0, 7, n).astype(np.int8), device='cuda')
    rows = []
    for mode, mname in ((0, 'autoreset'), (1, 'freeze')):
        if mode != env.mode:
            env.set_mode(mode)
        env.reset()
        full_ms, _, full_calls = timed(lambda: env.step(acts), seconds)
        for n_sel in (1, 32, 1024, 4096, n):
            if mode == 1:
                env.reset()
            ids = rng.permutation(n)[:n_sel].astype(np.int32)
            a = acts[:n_sel]
            ms, host_ms, calls = timed(lambda: env.step_envs(ids, a), seconds)
            k_ms = kernel_ms(lambda: env.step_envs(ids, a), 'k_step8_sel')
            rows.append(dict(mode=mname, n_sel=n_sel, launches=(n_sel + 4095) // 4096, step_envs_ms=round(ms, 4), calls=calls,
                             host_ms=round(host_ms, 4), kernel_ms=round(k_ms, 4),
                             step_ms=round(full_ms, 4), step_calls=full_calls,
                             step_envs_ns_per_env=round(ms * 1e6 / n_sel, 1), step_ns_per_env=round(full_ms * 1e6 / n, 2)))
            print(json.dumps(dict(level=level, n=n, **rows[-1])), file=sys.stderr, flush=True)
    errors = env.counters()['errors']
    env.close()
    return rows, errors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pools', default='GoToLocal:65536,BossLevel:32768')
    ap.add_argument('--seconds', type=float, default=1.0)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'needs a CUDA device'
    name, power = card()
    out = dict(card=name, power_limit=power, pools=[])
    for item in args.pools.split(','):
        level, n = item.split(':')
        rows, errors = measure(level, int(n), args.seconds)
        out['pools'].append(dict(level=level, n_envs=int(n), errors=errors, rows=rows))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
