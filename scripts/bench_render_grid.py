"""Throughput of full-grid frames (bb_pool_render_grid / k_render_grid, MiniGridEnv.render('rgb_array')) on one GPU.

Prints one JSON line: the card and its power limit (read in the same run), per config the frames per second, the bytes one
call writes, the kernel time per call (CUDA events around back-to-back calls after a warm-up, at least 1 s timed), the
achieved store bandwidth and its fraction of the H100 SXM data-sheet 3 350 GB/s; and the first-use host rasterisation time
of the tile table at tile sizes 8 / 32 / 64 (bb_grid_tiles, on the CPU).

usage: python scripts/bench_render_grid.py [--min-seconds 1.0]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
CONFIGS = [('GoToLocal', 65536, 8), ('BossLevel', 32768, 8), ('BossLevel', 2048, 32)]


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(',')]
        return name, power
    except Exception as e:                        # the numbers stand without it, but say why it is missing
        return 'unknown (%s)' % e, 'unknown'


def host_table_seconds(ts):
    import numpy as np
    from babyai_b200 import lib
    L = lib.load()
    t = np.zeros(2 * 5 * 43 * ts * ts * 3, np.uint8)
    t0 = time.perf_counter()
    assert L.bb_grid_tiles(ts, t.ctypes.data_as(C.c_void_p)) == 0
    return time.perf_counter() - t0


def run_config(level, n, ts, min_seconds):
    import numpy as np
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64))
    env.reset()
    rng = np.random.RandomState(0)
    for _ in range(10):                           # states away from the first ones
        env.step(torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=env.device))
    out = torch.empty((n, env.height * ts, env.width * ts, 3), dtype=torch.uint8, device=env.device)
    for _ in range(3):
        env.render_grid(tile_size=ts, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls = 2
    while True:
        e0.record()
        for _ in range(calls):
            env.render_grid(tile_size=ts, out=out)
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= 1000.0 * min_seconds:
            break
        calls = max(calls * 2, int(calls * 1000.0 * min_seconds / max(ms, 1e-3) * 1.2))
    per_call = ms / calls
    nbytes = out.numel()
    gbs = nbytes / (per_call * 1e-3) / 1e9
    assert env.counters()['errors'] == 0
    env.close()
    del out
    torch.cuda.empty_cache()
    return dict(level=level, envs=n, tile_size=ts, frame_shape=[env.height * ts, env.width * ts, 3], calls_timed=calls,
                timed_ms=round(ms, 2), kernel_ms_per_call=round(per_call, 4), bytes_per_call=nbytes,
                frames_per_s=round(n / (per_call * 1e-3), 1), achieved_gbs=round(gbs, 1), fraction_of_3350=round(gbs / PEAK_GBS, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--min-seconds', type=float, default=1.0)
    args = ap.parse_args()
    from babyai_b200 import build
    build.build()
    name, power = card()
    res = dict(metric='render_grid', gpu=name, power_limit=power,
               host_table_seconds={str(ts): round(host_table_seconds(ts), 4) for ts in (8, 32, 64)},
               configs=[run_config(level, n, ts, args.min_seconds) for level, n, ts in CONFIGS])
    print(json.dumps(res))


if __name__ == '__main__':
    main()
