"""k_full_obs on the GPU (bb_pool_full_obs, BabyAIVecEnv.full_obs) and the fully observable facades (FullyObsWrapper /
RGBImgObsWrapper lists): images after every call on 26 levels in both modes against the oracle's state (ICLR levels) and the
pool's own state (bonus levels), the golden images through the per-step and rollout paths, after reset_envs / step_envs /
load_envs / copy_envs, ragged / shuffled / repeated id lists at every output alignment, large pools, mixed pools, a side
stream, RGBImgObsWrapper batches, every facade path, and argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle as orc
from common import GOLDEN_LEVELS_GPU
from full_obs_common import BONUS_LEVELS, ICLR_LEVELS, P_RANDOM, expected, load_golden, matches

pytestmark = pytest.mark.gpu

LEVELS_26 = sorted(set(GOLDEN_LEVELS_GPU) | set(ICLR_LEVELS)) + BONUS_LEVELS
assert len(LEVELS_26) == 26


def _np(x):
    return x.cpu().numpy()


def _check(env, imgs, ids, level, ref=None):
    """row k of imgs is the image of env ids[k]: from the oracle's state where given, else from the pool's own"""
    imgs = _np(imgs)
    for k, i in enumerate(ids):
        assert matches(imgs[k], expected(ref if ref is not None else env, int(i), level)), (level, k, int(i))


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('level', LEVELS_26)
def test_after_every_step(level, mode):
    from babyai_b200 import BabyAIVecEnv
    n = 23
    seeds = np.arange(900, 900 + n, dtype=np.uint64)
    env = BabyAIVecEnv(level, n, seeds=seeds, mode=mode)
    # the oracle mirrors auto-reset steps; freeze mode and the bonus levels are checked against the pool's own state
    oracle = orc.OraclePool(level, n, seeds) if mode == 0 and level in ICLR_LEVELS + GOLDEN_LEVELS_GPU else None
    env.reset()
    if oracle is not None:
        oracle.reset()
    rng = np.random.RandomState(len(level))
    for t in range(48):                                            # 3 D steps of the default ring depth (16)
        ids = rng.randint(0, n, rng.randint(1, 2 * n))             # ragged, shuffled, repeats
        _check(env, env.full_obs(), range(n), level, oracle)
        _check(env, env.full_obs(ids), ids, level, oracle)
        a = rng.choice(7, n, p=P_RANDOM).astype(np.int8)
        env.step(torch.as_tensor(a, device=env.device))
        if oracle is not None:
            oracle.step(a)
            assert np.array_equal(_np(env.obs), oracle.obs), (level, t)
    assert env.counters()['errors'] == 0


@pytest.mark.parametrize('path', ['step', 'rollout'])
def test_golden_images(path):
    from babyai_b200 import BabyAIVecEnv
    for g in load_golden():
        n = 3
        env = BabyAIVecEnv(g['level'], n, seeds=np.full(n, g['seed'], np.uint64))
        env.reset()
        acts = torch.as_tensor(np.repeat(g['actions'][:, None], n, 1), device=env.device)
        T = acts.shape[0]
        obs = torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device=env.device)
        rew = torch.zeros((T, n), device=env.device)
        done = torch.zeros((T, n), dtype=torch.uint8, device=env.device)
        t = 0
        for stop in list(range(0, T + 1, 17)) + [T]:
            if stop > t:
                if path == 'rollout':
                    env.rollout(acts[t:stop], obs[:stop - t], rew[:stop - t], done[:stop - t])
                else:
                    for s in range(t, stop):
                        env.step(acts[s])
                t = stop
            got = _np(env.full_obs([2, 0, 1, 0]))
            for k in range(4):
                assert np.array_equal(got[k], g['images'][t]), (g['level'], path, t, k)
        env.close()


@pytest.mark.parametrize('mode', [0, 1])
def test_after_reset_envs_step_envs_load_envs_copy_envs(mode):
    from babyai_b200 import BabyAIVecEnv
    rng = np.random.RandomState(mode)
    for level in ('GoToLocal', 'BossLevel', 'PutNextS5N2Carrying', 'KeyCorridorS3R1'):
        n = 40
        env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64) + 77, mode=mode)
        env.reset()
        saved = env.save_envs()
        for t in range(12):
            ids = rng.permutation(n)[:rng.randint(1, n)]
            what = t % 4
            if what == 0:
                env.reset_envs(ids, seeds=rng.randint(0, 2 ** 40, ids.size).astype(np.uint64) if t % 8 == 0 else None)
            elif what == 1:
                env.step_envs(ids, torch.as_tensor(rng.choice(7, ids.size, p=P_RANDOM).astype(np.int8), device=env.device))
            elif what == 2:
                env.load_envs(saved, ids, rng.randint(0, n, ids.size))
            else:
                env.copy_envs(rng.randint(0, n, ids.size), ids)
            _check(env, env.full_obs(), range(n), level)
            env.step(torch.as_tensor(rng.choice(7, n, p=P_RANDOM).astype(np.int8), device=env.device))
            _check(env, env.full_obs(ids), ids, level)


def test_rows_outside_the_list_untouched_at_every_alignment():
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv('KeyCorridorS3R1', 50, seeds=np.arange(50, dtype=np.uint64))
    env.reset()
    F = 7 * 3 * 3
    rng = np.random.RandomState(3)
    for off in range(4):
        ids = rng.randint(0, 50, 37)
        flat = torch.full((64 + 37 * F + 64,), 0xAB, dtype=torch.uint8, device=env.device)
        out = flat[64 + off:64 + off + 37 * F].view(37, 7, 3, 3)
        assert env.full_obs(ids, out=out) is out
        f = _np(flat)
        assert (f[:64 + off] == 0xAB).all() and (f[64 + off + 37 * F:] == 0xAB).all()
        _check(env, out, ids, 'KeyCorridorS3R1')


@pytest.mark.parametrize('level,n', [('GoToLocal', 65536), ('BossLevel', 32768)])
def test_large_pools(level, n):
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64) * 3 + 1)
    env.reset()
    rng = np.random.RandomState(5)
    for _ in range(3):
        env.step(torch.as_tensor(rng.choice(7, n, p=P_RANDOM).astype(np.int8), device=env.device))
    before = env.launches()
    full = env.full_obs()
    assert env.launches() == before + 1
    sample = rng.randint(0, n, 300)
    _check(env, full[torch.as_tensor(sample, device=env.device)], sample, level)
    ids = rng.randint(0, n, 9000)                                   # three launches of 4 096 ids
    before = env.launches()
    part = env.full_obs(ids)
    assert env.launches() == before + 3
    assert torch.equal(part, full[torch.as_tensor(ids, device=env.device)])


def test_mixed_pool():
    from babyai_b200 import BabyAIVecEnv, lib
    groups = [('GoToLocal', 30), ('BossLevel', 20), ('PickupLoc', 25)]
    env = BabyAIVecEnv(groups, seeds=np.arange(75, dtype=np.uint64))
    env.reset()
    rng = np.random.RandomState(2)
    for _ in range(5):
        env.step(torch.as_tensor(rng.choice(7, 75, p=P_RANDOM).astype(np.int8), device=env.device))
    small = np.concatenate([np.arange(30), np.arange(50, 75)])
    ids = rng.choice(small, 60)
    got = env.full_obs(ids)
    assert got.shape == (60, 8, 8, 3)
    for k, i in enumerate(ids):
        assert matches(_np(got[k]), expected(env, int(i), env.level_of(int(i))))
    boss = env.full_obs(np.arange(30, 50))
    assert boss.shape == (20, 22, 22, 3)
    _check(env, boss, range(30, 50), 'BossLevel')
    with pytest.raises(ValueError):
        env.full_obs([0, 31])
    with pytest.raises(ValueError):
        env.full_obs()
    L = lib.load()
    before = env.launches()
    bad = np.array([0, 31], np.int32)
    out = torch.empty(2 * 22 * 22 * 3, dtype=torch.uint8, device=env.device)
    assert L.bb_pool_full_obs(env.h, bad.ctypes.data_as(C.c_void_p), 2, C.c_void_p(out.data_ptr()), None) != 0
    assert b'one grid size' in L.bb_last_error()
    assert env.launches() == before


def test_side_stream():
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv('BossLevel', 64, seeds=np.arange(64, dtype=np.uint64))
    env.reset()
    side = torch.cuda.Stream()
    rng = np.random.RandomState(4)
    with torch.cuda.stream(side):
        for _ in range(4):
            env.step(torch.as_tensor(rng.choice(7, 64, p=P_RANDOM).astype(np.int8), device=env.device))
            img = env.full_obs()
    side.synchronize()
    _check(env, img, range(64), 'BossLevel')
    img2 = env.full_obs()                                  # back on the default stream: ordered after the side stream's work
    assert torch.equal(img, img2)


def test_argument_checks():
    from babyai_b200 import BabyAIVecEnv, lib
    env = BabyAIVecEnv('GoToLocal', 8, seeds=np.arange(8, dtype=np.uint64))
    env.reset()
    for ids in ([8], [-1], [[0, 1]], [0.5]):
        with pytest.raises(ValueError):
            env.full_obs(ids)
    with pytest.raises(ValueError):
        env.full_obs(out=torch.empty((8, 8, 8, 3), dtype=torch.uint8))
    with pytest.raises(ValueError):
        env.full_obs([1, 2], out=torch.empty((3, 8, 8, 3), dtype=torch.uint8, device=env.device))
    L = lib.load()
    before = env.launches()
    out = torch.empty((8, 8, 8, 3), dtype=torch.uint8, device=env.device)
    assert L.bb_pool_full_obs(env.h, None, 7, C.c_void_p(out.data_ptr()), None) != 0
    bad = np.array([0, 8], np.int32)
    assert L.bb_pool_full_obs(env.h, bad.ctypes.data_as(C.c_void_p), 2, C.c_void_p(out.data_ptr()), None) != 0
    assert L.bb_pool_full_obs(env.h, bad.ctypes.data_as(C.c_void_p), -1, C.c_void_p(out.data_ptr()), None) != 0
    assert L.bb_pool_full_obs(env.h, bad.ctypes.data_as(C.c_void_p), 0, None, None) == 0
    assert env.launches() == before
    assert len(env.full_obs([])) == 0


def test_rgb_wrapper_batches_equal_render_grid_and_golden_frames():
    import babyai_b200 as bb
    from babyai_b200.learner import DeviceParallelEnv
    from render_grid_common import load_golden as load_rgb_golden
    n_frames = 0
    for g in load_rgb_golden():
        envs = bb.RGBImgObsWrapper(bb.EnvList(g['level'], [g['seed']] * 2), tile_size=8)
        dev = DeviceParallelEnv(envs)
        obs = dev.reset()
        t = 0
        for step, ts, hl, _door, want in g['frames']:
            while t < step:
                obs = next(dev.step(np.full(2, g['actions'][t])))
                t += 1
            assert torch.equal(obs.image, dev.pool.render_grid(None, 8, highlight=False))
            if ts == 8 and not hl:
                for k in range(2):
                    assert np.array_equal(_np(obs.image[k]), want), (g['level'], step)
                n_frames += 1
    assert n_frames >= 5


@pytest.mark.parametrize('wrapper', ['full', 'rgb'])
@pytest.mark.parametrize('fused_io', [False, True])
def test_facade_paths(wrapper, fused_io):
    import babyai_b200 as bb
    from babyai_b200.learner import DeviceManyEnvs, DeviceParallelEnv
    from babyai_b200.vecenv import full_image
    level, n = 'PutNextS5N2Carrying', 24
    wrap = bb.FullyObsWrapper if wrapper == 'full' else (lambda e: bb.RGBImgObsWrapper(e, tile_size=3))
    full = 'grid' if wrapper == 'full' else 'rgb'
    rng = np.random.RandomState(6)

    def current(d):
        return full_image(d.pool, full, 3)

    par = DeviceParallelEnv(wrap(bb.make_envs(level, n, seed=4)), fused_io=fused_io)
    obs = par.reset()
    assert torch.equal(obs.image, current(par)) and tuple(obs.image.shape[1:]) == par.observation_space.spaces['image'].shape
    saved = par.save_envs()
    for t in range(30):
        obs = next(par.step(rng.choice(7, n, p=P_RANDOM)))
        assert torch.equal(obs.image, current(par)), t
        if t % 10 == 5:
            ids = rng.permutation(n)[:7]
            obs = par.load_envs(saved, obs, ids=ids)
            assert torch.equal(obs.image, current(par)), t
            obs = par.copy_envs(rng.randint(0, n, 5), rng.permutation(n)[:5], obs)
            assert torch.equal(obs.image, current(par)), t
    many = DeviceManyEnvs(wrap(bb.make_envs(level, n, seed=4)), fused_io=fused_io)
    many.seed(range(1000, 1000 + n))
    obs = many.reset()
    for t in range(30):
        obs = next(many.step(rng.choice(7, n, p=P_RANDOM)))
        assert torch.equal(obs.image, current(many)), t
        if t % 10 == 9:
            ids = rng.permutation(n)[:6]
            obs = many.reset_envs(ids, rng.randint(0, 10 ** 6, 6).astype(np.uint64), obs)
            assert torch.equal(obs.image, current(many)), t
    host = bb.ParallelEnv(wrap(bb.make_envs(level, 5, seed=4)))
    ho = host.reset()
    for t in range(10):
        want = _np(current(host))
        assert all(np.array_equal(ho[i]['image'], want[i]) for i in range(5)) and 'direction' not in ho[0]
        ho = next(host.step(rng.choice(7, 5, p=P_RANDOM)))
