"""bb_pool_reset_envs / BabyAIVecEnv.reset_envs on the GPU, bit-exact against the oracle (ICLR levels) or the host build (bonus
levels): observations, reward bit patterns, done, direction, missions and hidden state (draw counts included where the two
sides keep the same rings).  Every test ends with counters()['errors'] == 0.

- Equivalence: reset_envs(every id, seeds) is seed(seeds) followed by reset().
- Random schedules: random subsets reset with and without seeds between bb_pool_step calls and bb_pool_rollout launches on the
  fused, in-stream-refill, concurrent-pass and graph paths, in auto-reset and freeze mode, then 3 D further steps (the rings
  stayed supplied); 97 and 1 037 envs, and the BASELINE sizes with a sample that covers every k_reset8 CTA.
- Untouched rows, freeze mode, rejected calls, 64-bit seeds, stream order behind a held producer stream.
- The streaming evaluator (babyai_b200.evaluate.batch_evaluate) against a wave evaluation through DeviceManyEnvs."""
import ctypes as C
import gc

import numpy as np
import pytest

from reset_envs_common import AUTORESET, BONUS_PER_KIND, FREEZE, PolicyAgent, compare_rows, mirror_for

pytestmark = pytest.mark.gpu
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s at the H100's clock


def _np(x):
    return x.cpu().numpy()


def _pool(level, n, seeds, mode):
    from babyai_b200 import BabyAIVecEnv
    return BabyAIVecEnv(level, n, seeds=np.asarray(seeds, np.uint64), mode=mode)


def _same_state(a, b, envs, what):
    """grid and every state field, draws and attempts included"""
    for i in envs:
        ga, ia = a.state(int(i))
        gb, ib = b.state(int(i))
        assert np.array_equal(ga, gb) and ia == ib, (what, int(i), ia, ib)


def _mirror_state(env, mirror, envs, what):
    for i in envs:
        g, info = env.state(int(i))
        mg, mi = mirror.state(int(i))
        for k in ('draws', 'attempts'):
            info.pop(k), mi.pop(k)
        assert np.array_equal(g, mg) and info == mi, (what, int(i), info, mi)
    assert env.missions([int(i) for i in envs]) == [mirror.mission(int(i)) for i in envs], (what, 'missions')


# ------------------------------------------------------------------------------------------------------------------------
# equivalence with seed() + reset()
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc', 'GoTo', 'BossLevel', 'Unlock', 'GoToImpUnlock'] + BONUS_PER_KIND)
def test_reset_every_env_with_seeds_equals_seed_then_reset(level, mode):
    import torch
    n, rng = 97, np.random.RandomState(5)
    a = _pool(level, n, np.arange(n) + 100, mode)
    a.reset()
    for _ in range(5):
        a.step(torch.as_tensor(rng.randint(0, 7, n).astype(np.int8), device='cuda'))
    new = rng.randint(0, 2 ** 63, n).astype(np.uint64) * 2 + 1            # full 64-bit seeds
    ids = rng.permutation(n)
    obs = torch.full((n, 7, 7, 3), 0x5A, dtype=torch.uint8, device='cuda')
    dire = torch.full((n,), -3, dtype=torch.int8, device='cuda')
    a.reset_envs(ids, new[ids], obs=obs, direction=dire)
    b = _pool(level, n, new, mode)
    b.reset()
    assert torch.equal(obs, b.obs) and torch.equal(dire, b.direction), level
    assert a.missions() == b.missions()
    _same_state(a, b, range(n), (level, 'after reset'))
    for t in range(3 * 8):
        act = torch.as_tensor(rng.randint(0, 7, n).astype(np.int8), device='cuda')
        oa = [x.clone() for x in a.step(act)]
        ob = b.step(act)
        assert all(torch.equal(x, y) for x, y in zip(oa, ob)) and torch.equal(a.direction, b.direction), (level, t)
    _same_state(a, b, range(n), (level, 'after steps'))
    assert a.counters()['errors'] == 0 and b.counters()['errors'] == 0


# ------------------------------------------------------------------------------------------------------------------------
# random schedules against the oracle / host build
# ------------------------------------------------------------------------------------------------------------------------
SINGLE_PATHS = {'step': {}, 'fused': {}, 'instream': {'BB_GEN_FUSED': '0'}, 'graph': {'BB_NO_PERSISTENT': '1'}}
MULTI_PATHS = {'step': {}, 'concurrent': {}, 'graph': {'BB_NO_PERSISTENT': '1'}}
SCHEDULES = [(lv, p) for lv in ('GoToLocal',) for p in SINGLE_PATHS] + \
            [(lv, p) for lv in ('BossLevel', 'Unlock', 'KeyCorridorS3R1') for p in MULTI_PATHS]


def _run_schedule(env, mirror, rng, T, per_step, rounds, tail_steps, what):
    """rounds of (a chunk of steps, a random reset_envs) then `tail_steps` more steps; every mirrored env compared at every
    step, every reset, and its state at the end"""
    import torch
    n, dev = env.num_envs, env.device
    outs = [torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device=dev), torch.zeros((T, n), dtype=torch.float32, device=dev),
            torch.zeros((T, n), dtype=torch.uint8, device=dev), torch.zeros((T, n), dtype=torch.int8, device=dev)]

    def chunk(steps):
        for t0 in range(0, steps, T):
            a = rng.randint(0, 7, (T, n)).astype(np.int8)
            if per_step:
                for t in range(T):
                    env.step(torch.as_tensor(a[t], device=dev), *[x[t] for x in outs])
            else:
                env.rollout(torch.as_tensor(a, device=dev), *outs)
            got = [_np(x) for x in outs]
            for t in range(T):
                compare_rows([g[t] for g in got], mirror.step(a[t]), (what, 'step', t0 + t))

    for rnd in range(rounds):
        chunk(T * (1 + rng.randint(0, 3)))
        k = int(rng.randint(1, max(2, n // 3)))
        ids = rng.permutation(n)[:k]
        seeds = rng.randint(0, 2 ** 63, k).astype(np.uint64) * 2 if rnd % 2 == 0 else None
        obs = torch.full((n, 7, 7, 3), 0xC3, dtype=torch.uint8, device=dev)
        dire = torch.full((n,), -5, dtype=torch.int8, device=dev)
        env.reset_envs(ids, seeds, obs=obs, direction=dire)
        mirror.reset_envs(ids, seeds)
        o, d = _np(obs), _np(dire)
        listed = np.zeros(n, bool)
        listed[ids] = True
        assert (o[~listed] == 0xC3).all() and (d[~listed] == -5).all(), (what, rnd, 'unlisted rows written')
        compare_rows((o, None, None, d), {i: mirror.last[i] for i in mirror.ids if listed[i]}, (what, 'reset', rnd))
    chunk(tail_steps)
    _mirror_state(env, mirror, mirror.ids[:64], what)
    assert env.counters()['errors'] == 0, what


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('n', [97, 1037])
@pytest.mark.parametrize('level,path', SCHEDULES)
def test_random_schedule(level, path, n, mode, monkeypatch):
    multi = level != 'GoToLocal'
    for k, v in (MULTI_PATHS if multi else SINGLE_PATHS)[path].items():
        monkeypatch.setenv(k, v)
    if multi:
        monkeypatch.setenv('BB_RING_DEPTH', '64')               # 3 D steps at a depth the oracle keeps up with
    rng = np.random.RandomState(n + 3 * mode + len(path))
    seeds = np.arange(n, dtype=np.uint64) * 7 + 11
    env = _pool(level, n, seeds, mode)
    D = 64 if multi else 128
    mirrored = np.arange(n) if n < 200 else np.unique(np.r_[0, n - 1, rng.choice(n, 120, replace=False)])
    mirror = mirror_for(level, seeds, mode, mirrored)
    env.reset()
    mirror.reset()
    compare_rows((_np(env.obs), None, None, _np(env.direction)), mirror.last, (level, 'reset'))
    T = 1 if path == 'step' else (16 if multi else 20)
    _run_schedule(env, mirror, rng, T, path == 'step', 5, ((3 * D + T - 1) // T) * T, (level, path, n, mode))


@pytest.mark.parametrize('level,n', [('GoToLocal', 65536), ('BossLevel', 32768)])
def test_baseline_sizes_sampled(level, n):
    """a reset of 9 000 (BossLevel: 4 500) ids -- several id chunks -- with seeds and one without, at the BASELINE pool sizes:
    one listed env of every 16-env k_reset8 CTA is mirrored, through 3 D further rollout steps"""
    import torch
    rng = np.random.RandomState(n)
    seeds = np.arange(n, dtype=np.uint64) + 3
    env = _pool(level, n, seeds, AUTORESET)
    env.reset()
    ids = rng.permutation(n)[:9000 if level == 'GoToLocal' else 4500]
    sample = ids[::16]
    new = rng.randint(0, 2 ** 63, ids.size).astype(np.uint64)
    from reset_envs_common import OracleMirror
    mirror = OracleMirror(level, dict(zip(sample.tolist(), new[::16].tolist())), AUTORESET, sample)
    obs = torch.full((n, 7, 7, 3), 0x99, dtype=torch.uint8, device='cuda')
    env.reset_envs(ids, new, obs=obs)
    mirror.reset_envs(sample, new[::16])
    o = _np(obs)
    listed = np.zeros(n, bool)
    listed[ids] = True
    assert (o[~listed] == 0x99).all()
    compare_rows((o, None, None, _np(env.direction)), mirror.last, (level, 'seeded'))
    ids2 = rng.permutation(n)[:5000]
    sample2 = np.intersect1d(ids2, sample)
    env.reset_envs(ids2)
    mirror.reset_envs(sample2)
    compare_rows((_np(env.obs), None, None, _np(env.direction)), {i: mirror.last[i] for i in sample2}, (level, 'unseeded'))
    T = 32
    steps = 3 * 128 if level == 'GoToLocal' else 3 * 512              # 3 D at the default ring depths
    outs = [torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros((T, n), dtype=torch.float32, device='cuda'),
            torch.zeros((T, n), dtype=torch.uint8, device='cuda'), torch.zeros((T, n), dtype=torch.int8, device='cuda')]
    for t0 in range(0, steps, T):
        a = rng.randint(0, 7, (T, n)).astype(np.int8)
        env.rollout(torch.as_tensor(a, device='cuda'), *outs)
        got = [_np(x[:, sample]) for x in outs]
        for t in range(T):
            want = mirror.step(dict(zip(sample.tolist(), a[t, sample].tolist())))
            compare_rows([g[t] for g in got], {j: want[int(i)] for j, i in enumerate(sample)}, (level, t0 + t))
    _mirror_state(env, mirror, sample[:32], level)
    assert env.counters()['errors'] == 0


# ------------------------------------------------------------------------------------------------------------------------
# freeze mode, arguments, streams
# ------------------------------------------------------------------------------------------------------------------------
def test_freeze_reset_envs_step_again_unlisted_frozen_replay():
    import torch
    n, rng = 97, np.random.RandomState(2)
    seeds = np.arange(n) + 40
    env = _pool('GoToRedBallNoDists', n, seeds, FREEZE)
    mirror = mirror_for('GoToRedBallNoDists', seeds, FREEZE)
    env.reset()
    mirror.reset()
    for t in range(60):                                    # many episodes end (and freeze) on this level
        a = rng.randint(0, 7, n).astype(np.int8)
        compare_rows([_np(x) for x in env.step(torch.as_tensor(a, device='cuda'))] + [_np(env.direction)], mirror.step(a), t)
    frozen = np.nonzero(_np(env.done))[0]
    assert len(frozen) > 10
    ids = frozen[::2]
    env.reset_envs(ids)
    mirror.reset_envs(ids)
    a = np.full(n, 2, np.int8)                             # forward
    r = [_np(x) for x in env.step(torch.as_tensor(a, device='cuda'))] + [_np(env.direction)]
    compare_rows(r, mirror.step(a), 'after')
    assert not r[2][ids].all()                              # the reset envs play again ...
    assert r[2][frozen[1::2]].all()                         # ... the others still replay their last result
    assert env.counters()['errors'] == 0


def test_rejected_calls_launch_nothing():
    import torch
    from babyai_b200 import lib
    L = lib.load()
    env = _pool('BossLevel', 97, np.arange(97), AUTORESET)
    env.reset()
    torch.cuda.synchronize()
    l0 = env.launches()
    for ids in ([3, 5, 3], [0, 97], [-1], [96, 200]):
        with pytest.raises(ValueError):
            env.reset_envs(ids)
        a = np.asarray(ids, np.int32)
        assert L.bb_pool_reset_envs(env.h, a.ctypes.data_as(C.c_void_p), None, a.size, C.c_void_p(env.obs.data_ptr()), None, None) != 0
    a = np.asarray([1, 2], np.int32)
    assert L.bb_pool_reset_envs(env.h, a.ctypes.data_as(C.c_void_p), None, 2, None, None, None) != 0      # NULL obs
    assert L.bb_pool_reset_envs(env.h, None, None, 2, C.c_void_p(env.obs.data_ptr()), None, None) != 0    # NULL ids
    with pytest.raises(ValueError):
        env.reset_envs([1, 2], seeds=[5])
    assert env.launches() == l0
    env.reset_envs([])                                     # n_sel = 0: nothing enqueued
    assert L.bb_pool_reset_envs(env.h, None, None, 0, C.c_void_p(env.obs.data_ptr()), None, None) == 0
    assert env.launches() == l0
    assert env.counters()['errors'] == 0


def test_side_stream_behind_a_held_producer_stream():
    """pool.step on a producer stream behind a ~0.1 s spin kernel, then reset_envs on another stream issued at once: the reset
    must come after the step (a fresh episode at step 0), and the pool goes on from there"""
    import torch
    n, level = 97, 'BossLevel'
    rng = np.random.RandomState(4)
    a1, a2 = rng.randint(0, 7, n).astype(np.int8), rng.randint(0, 7, n).astype(np.int8)
    ids = rng.permutation(n)[:30]
    new = rng.randint(0, 2 ** 63, 30).astype(np.uint64)
    d1, d2 = torch.as_tensor(a1, device='cuda'), torch.as_tensor(a2, device='cuda')
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()

    def scenario(sleep):
        seeds = np.arange(n) + 70
        env = _pool(level, n, seeds, AUTORESET)
        env.reset()
        obs = torch.zeros((n, 7, 7, 3), dtype=torch.uint8, device='cuda')
        dire = torch.zeros(n, dtype=torch.int8, device='cuda')
        torch.cuda.synchronize()
        gc.collect()
        gc.disable()
        try:
            with torch.cuda.stream(sa):
                sleep()
                env.step(d1)
            with torch.cuda.stream(sb):
                env.reset_envs(ids, new, obs=obs, direction=dire)
        finally:
            gc.enable()
        torch.cuda.synchronize()
        return env, obs, dire, seeds

    scenario(lambda: None)[0].close()                      # kernels loaded: lazy loading cannot order the calls
    env, obs, dire, seeds = scenario(lambda: torch.cuda._sleep(SLEEP_CYCLES))
    mirror = mirror_for(level, seeds, AUTORESET)
    mirror.reset()
    mirror.step(a1)
    mirror.reset_envs(ids, new)
    compare_rows((_np(obs), None, None, _np(dire)), {int(i): mirror.last[int(i)] for i in ids}, 'reset')
    _mirror_state(env, mirror, ids[:12], 'state after')
    compare_rows([_np(x) for x in env.step(d2)] + [_np(env.direction)], mirror.step(a2), 'step after')
    assert env.counters()['errors'] == 0


# ------------------------------------------------------------------------------------------------------------------------
# the streaming evaluator
# ------------------------------------------------------------------------------------------------------------------------
def _wave_evaluate(level, seed, episodes, num_envs, pixel=False):
    """seeds in waves of num_envs through DeviceManyEnvs: every env plays until the wave's slowest episode has ended"""
    from babyai_b200.learner import DeviceManyEnvs
    from babyai_b200.vecenv import EnvList
    agent = PolicyAgent()
    env = DeviceManyEnvs(EnvList(level, [0] * num_envs, pixel=pixel))
    frames, returns = [], []
    for w in range((episodes + num_envs - 1) // num_envs):
        env.seed(range(seed + w * num_envs, seed + (w + 1) * num_envs))
        obs = env.reset()
        f = np.zeros(num_envs, np.int64)
        r = np.zeros(num_envs)
        t = 0
        while (f == 0).any():
            obs, rew, done, _ = env.step(agent.act_batch(obs)['action'])
            t += 1
            new = np.array(done) & (f == 0)
            f[new] = t
            r[new] = np.asarray(rew)[new]
        frames += list(f)
        returns += list(r)
    return frames, returns


@pytest.mark.timeout(600)
@pytest.mark.parametrize('num_envs', [256, 4096])
@pytest.mark.parametrize('level', ['GoToLocal', 'BossLevel'])
def test_streaming_evaluator_equals_wave_evaluation(level, num_envs):
    from babyai_b200.evaluate import batch_evaluate
    seed, episodes = 10 ** 9, 2 * num_envs
    logs = batch_evaluate(PolicyAgent(), 'BabyAI-%s-v0' % level, seed, episodes, num_envs=num_envs)
    frames, returns = _wave_evaluate(level, seed, episodes, num_envs)
    assert logs['seed_per_episode'] == list(range(seed, seed + episodes))
    assert [int(x) for x in logs['num_frames_per_episode']] == [int(x) for x in frames]
    assert [np.float32(x) for x in logs['return_per_episode']] == [np.float32(x) for x in returns]


def test_streaming_evaluator_pixel_observations():
    """pixel=True: the reset envs' rows of the batch are their new 56x56 pictures (the policy reads the pixels)"""
    from babyai_b200.evaluate import batch_evaluate
    seed, num_envs = 777, 256
    logs = batch_evaluate(PolicyAgent(), 'BabyAI-GoToLocal-v0', seed, 3 * num_envs, pixel=True, num_envs=num_envs)
    frames, returns = _wave_evaluate('GoToLocal', seed, 3 * num_envs, num_envs, pixel=True)
    assert [int(x) for x in logs['num_frames_per_episode']] == [int(x) for x in frames]
    assert [np.float32(x) for x in logs['return_per_episode']] == [np.float32(x) for x in returns]
