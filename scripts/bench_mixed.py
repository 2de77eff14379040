"""Mixed-level pools against their groups run as separate pools (DESIGN.md sections 4.11 and 7).

For each pool -- GoToLocal 32 768 + BossLevel 32 768 (the BASELINE sizes), and a three-level mix with ragged group sizes --
it times, with CUDA events around back-to-back calls after a warm-up:
  step      bb_pool_step, int8 device actions
  learner   bb_pool_step_learner, host actions in, reward / done out (one synchronisation per call)
  rollout   bb_pool_rollout, T = 40
once on the mixed pool and once on the same groups as separate pools called one after another on one stream.  `step` is also
timed with each separate pool on a stream of its own (what forking the per-step call would buy).  The mixed pool and the
separate pools never exist at the same time: each takes the ring depth an empty device gives it.  Prints one JSON line per
pool, with the card and its power limit read in the same run.

    python scripts/bench_mixed.py [--steps 20] [--warmup 5] [--out results/bench_mixed.json]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')))

POOLS = {
    'GoToLocal32768+BossLevel32768': [('GoToLocal', 32768), ('BossLevel', 32768)],
    'ragged3': [('GoToRedBall', 20011), ('PickupLoc', 9973), ('BossLevel', 12347)],
}
T = 40


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def measure(pools, n, steps, warmup, streams=None):
    """pools: [(env, first row)] stepped one after another (a mixed pool is one env at row 0)"""
    rng = np.random.RandomState(0)
    a1 = torch.as_tensor(rng.randint(0, 7, n).astype(np.int8), device='cuda')
    aT = torch.as_tensor(rng.randint(0, 7, (T, n)).astype(np.int8), device='cuda')
    ah = rng.randint(0, 7, n).astype(np.int8)
    obs, rew = torch.zeros((n, 7, 7, 3), dtype=torch.uint8, device='cuda'), np.zeros(n, np.float32)
    done = np.zeros(n, np.uint8)
    rT = [torch.zeros((T, e.num_envs, 7, 7, 3), dtype=torch.uint8, device='cuda') for e, _ in pools]
    rr = [torch.zeros((T, e.num_envs), device='cuda') for e, _ in pools]
    rd = [torch.zeros((T, e.num_envs), dtype=torch.uint8, device='cuda') for e, _ in pools]
    aTs = [aT[:, s:s + e.num_envs].contiguous() for e, s in pools]
    a1s = [a1[s:s + e.num_envs] for e, s in pools]
    for e, _ in pools:
        e.reset()

    def step():
        for e, a in zip(pools, a1s):
            e[0].step(a)

    def learner():
        for (e, s), a in zip(pools, a1s):
            m = e.num_envs
            e.step_learner(ah[s:s + m], obs[s:s + m], rew[s:s + m], done[s:s + m])

    def rollout():
        for k, (e, _) in enumerate(pools):
            e.rollout(aTs[k], rT[k], rr[k], rd[k])

    out = {'step_ms': timed(step, steps, warmup), 'learner_ms': timed(learner, steps, warmup),
           'rollout_T40_ms': timed(rollout, steps, warmup)}
    if streams:
        cur = torch.cuda.current_stream()

        def step_forked():
            ev = cur.record_event()
            for (e, _), a, st in zip(pools, a1s, streams):
                st.wait_event(ev)
                with torch.cuda.stream(st):
                    e.step(a)
            for st in streams:
                cur.wait_stream(st)
        out['step_forked_ms'] = timed(step_forked, steps, warmup)
    errors = sum(e.counters()['errors'] for e, _ in pools)
    assert errors == 0, errors
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mixed.py measures on a GPU; there is none here')
    from babyai_b200 import BabyAIVecEnv
    device = card()
    results = []
    for name, groups in POOLS.items():
        n = sum(c for _, c in groups)
        seeds = np.arange(n, dtype=np.uint64)
        env = BabyAIVecEnv(groups, seeds=seeds)
        mixed = measure([(env, 0)], n, args.steps, args.warmup)
        env.close()
        del env
        gc.collect()
        torch.cuda.empty_cache()
        sep, s = [], 0
        for lvl, c in groups:
            sep.append((BabyAIVecEnv(lvl, c, seeds=seeds[s:s + c]), s))
            s += c
        separate = measure(sep, n, args.steps, args.warmup, streams=[torch.cuda.Stream() for _ in sep])
        for e, _ in sep:
            e.close()
        del sep
        gc.collect()
        torch.cuda.empty_cache()
        r = {'pool': name, 'groups': groups, 'device': device, 'steps': args.steps, 'mixed': mixed, 'separate': separate}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
