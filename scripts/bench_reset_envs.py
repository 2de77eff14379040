"""Cost of per-env resets (bb_pool_reset_envs) and what they buy the evaluator, on one GPU.

Prints one JSON line: the card and its power limit (read in the same run), then per pool
- the latency of one reset_envs call for n_sel in {1, 32, 1024, n_envs}, with and without seeds, in freeze and in auto-reset
  mode (CUDA events around the call on the current stream; a call that takes over 0.2 s is timed once, the others are the
  median of 10 after a warm-up call).  Reseeding in auto-reset mode regenerates the env's whole ring of D levels, serially;
- episodes per second of babyai_b200.evaluate.batch_evaluate (the stream: finished envs take the next seed at once) and of
  a wave loop over the same seeds through DeviceManyEnvs, with a random-action policy on the device; 2 x n_envs episodes.

usage: python scripts/bench_reset_envs.py [--pools GoToLocal:65536,BossLevel:32768]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_render_grid import card  # noqa: E402


class RandomAgent(object):
    def __init__(self, seed=0):
        import torch
        self.g = torch.Generator(device='cuda')
        self.g.manual_seed(seed)

    def act_batch(self, many_obs):
        import torch
        return {'action': torch.randint(0, 7, (len(many_obs),), device='cuda', generator=self.g)}

    def analyze_feedback(self, reward, done):
        pass


def reset_latency(level, n, mode, n_sel, seeded):
    import numpy as np
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64), mode=mode)
    env.reset()
    rng = np.random.RandomState(n_sel)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def once(k):
        ids = rng.permutation(n)[:n_sel]
        seeds = rng.randint(0, 2 ** 62, n_sel).astype(np.uint64) + k if seeded else None
        torch.cuda.synchronize()
        ev0.record()
        env.reset_envs(ids, seeds)
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    first = once(0)
    ms = [first] if first > 200 else sorted(once(k) for k in range(1, 11))
    errors = env.counters()['errors']
    env.close()
    return dict(ms=ms[len(ms) // 2], calls=len(ms), errors=errors)


def evaluate_rate(level, n):
    import torch
    from babyai_b200.evaluate import batch_evaluate
    from babyai_b200.learner import DeviceManyEnvs
    from babyai_b200.vecenv import EnvList
    episodes, seed = 2 * n, 10 ** 9
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    logs = batch_evaluate(RandomAgent(), level, seed, episodes, num_envs=n)
    torch.cuda.synchronize()
    t_stream = time.perf_counter() - t0
    env = DeviceManyEnvs(EnvList(level, [0] * n))
    agent = RandomAgent()
    env_steps = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for w in range(2):
        env.seed(range(seed + w * n, seed + (w + 1) * n))
        obs = env.reset()
        finished = torch.zeros(n, dtype=torch.bool)
        while not bool(finished.all()):
            obs, _, done, _ = env.step(agent.act_batch(obs)['action'])
            finished |= torch.as_tensor(done)
            env_steps += n
    torch.cuda.synchronize()
    t_wave = time.perf_counter() - t0
    return dict(episodes=episodes, stream_s=round(t_stream, 3), stream_episodes_per_s=round(episodes / t_stream, 1),
                stream_env_steps_played=int(sum(logs['num_frames_per_episode'])),
                wave_s=round(t_wave, 3), wave_episodes_per_s=round(episodes / t_wave, 1), wave_env_steps=env_steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pools', default='GoToLocal:65536,BossLevel:32768')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'needs a CUDA device'
    name, power = card()
    out = dict(card=name, power_limit=power, pools=[])
    for item in args.pools.split(','):
        level, n = item.split(':')
        n = int(n)
        rows = []
        for mode, mname in ((1, 'freeze'), (0, 'autoreset')):
            for seeded in (False, True):
                for n_sel in (1, 32, 1024, n):
                    r = reset_latency(level, n, mode, n_sel, seeded)
                    rows.append(dict(mode=mname, seeds=seeded, n_sel=n_sel, **r))
                    print(json.dumps(dict(level=level, n=n, **rows[-1])), file=sys.stderr, flush=True)
        ev = evaluate_rate(level, n)
        print(json.dumps(dict(level=level, n=n, **ev)), file=sys.stderr, flush=True)
        out['pools'].append(dict(level=level, n_envs=n, reset_envs=rows, evaluate=ev))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
