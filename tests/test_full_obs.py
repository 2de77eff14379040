"""Fully observable observations (gym_minigrid 1.0.x FullyObsWrapper / RGBImgObsWrapper) without a GPU: k_full_obs's per-env
source (csrc/full_obs.cuh, compiled for the host by tests/hostemu/full_obs_host.cpp) against the wrapper over the reference's
unmodified level classes and against the golden images, the facades and gymapi over the host build, the argument checks,
and the built library's k_full_obs in sm_90a SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from full_obs_common import (BONUS_LEVELS, ICLR_LEVELS, P_RANDOM, FullTensorPool, encode, expected, load_golden, matches,
                             shim_renderable, wrappers)

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


def _host_pool(level, seeds, mode=0):
    from babyai_b200.levels import level_spec
    from full_obs_host import FullObsHostPool
    return FullObsHostPool(level_spec(level), len(seeds), seeds=np.asarray(seeds, np.uint64), mode=mode)


def test_host_build_replays_golden_images():
    """tests/golden/full_obs: the reference's levels wrapped in FullyObsWrapper after every action; the host build replays the
    actions and its image (at every offset modulo 4 of the output) is equal, and so is the numpy statement from its state"""
    n = 0
    for g in load_golden():
        pool = _host_pool(g['level'], [g['seed']])
        pool.reset()
        for t in range(len(g['actions']) + 1):
            if t:
                pool.step(g['actions'][t - 1:t])
            want = g['images'][t]
            assert np.array_equal(pool.full_obs_env(0, t % 4), want), (g['level'], t)
            assert matches(want, expected(pool, 0, g['level'])), (g['level'], t)
            n += 1
    gold = {g['level']: g['images'].shape[1:3] for g in load_golden()}
    assert n > 800 and gold['KeyCorridorS3R1'] == (7, 3) and gold['MoveTwoAcrossS5N2'] == (9, 5)


@pytest.mark.reference
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('level', ICLR_LEVELS + BONUS_LEVELS)
def test_host_role_equals_wrapper_over_reference_levels(level, mode):
    """FullyObsWrapper over the reference's unmodified level classes on the shim (Philox back-end) == the host build after
    every action of a random trace, in auto-reset (mode 0) and freeze (mode 1) flavour"""
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    import refenv
    refenv.setup('philox')
    FullyObsWrapper, _ = wrappers()
    seed = 500 + 7 * len(level) + mode
    env = FullyObsWrapper(refenv.make_env(level, seed, 'philox'))
    pool = _host_pool(level, [seed], mode)
    want = env.reset()['image']
    pool.reset()
    assert np.array_equal(pool.full_obs_env(0), want), (level, 0)
    rng = np.random.RandomState(len(level) + mode)
    for t in range(240):
        a = int(rng.choice(7, p=P_RANDOM))
        obs, _r, done, _ = env.step(a)
        pool.step(np.array([a], np.int8))
        if done and mode == 0:
            obs = env.reset()
        assert np.array_equal(pool.full_obs_env(0, t % 4), obs['image']), (level, mode, t)
        if done and mode == 1:                         # a frozen env repeats its terminal state until reset
            pool.step(np.array([2], np.int8))
            assert np.array_equal(pool.full_obs_env(0), obs['image']), (level, mode, t, 'frozen')
            want = env.reset()['image']
            pool.reset()
            assert np.array_equal(pool.full_obs_env(0), want), (level, mode, t, 'reset')


def test_put_next_carrying_hides_the_carried_object_at_step_0():
    """the pool still holds obj_a on the grid while step_count is 0; the image reads that cell as empty"""
    pool = _host_pool('PutNextS5N2Carrying', [17])
    pool.reset()
    grid, s = pool.state(0)
    assert s['step_count'] == 0
    img = pool.full_obs_env(0)
    full = encode(grid, s['agent_x'], s['agent_y'], s['agent_dir'])
    diff = np.argwhere((img != full).any(-1))
    assert len(diff) == 1 and tuple(img[tuple(diff[0])]) == (1, 0, 0) and full[tuple(diff[0])][0] in (5, 6, 7)


def _ref_vec(kind, level, seeds, wrap):
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    import refenv
    refenv.setup('philox')
    envs = [wrap(shim_renderable(refenv.make_env(level, s, 'philox'))) for s in seeds]
    if kind == 'ParallelEnv':
        from babyai.rl.utils.penv import ParallelEnv
        return ParallelEnv(envs)
    from babyai.evaluate import ManyEnvs
    return ManyEnvs(envs)


@pytest.mark.reference
@pytest.mark.timeout(300)
@pytest.mark.parametrize('kind', ['ParallelEnv', 'ManyEnvs'])
@pytest.mark.parametrize('wrapper,level', [('full', 'KeyCorridorS3R1'), ('full', 'PutNextS5N2Carrying'), ('rgb', 'MoveTwoAcrossS5N2'),
                                           ('rgb', 'GoToLocal')])
def test_facades_equal_reference_vec_envs_of_wrapped_envs(kind, wrapper, level):
    """babyai_b200.ParallelEnv / ManyEnvs (and the device facades) of a wrapped make_envs list over the host build == the
    reference's ParallelEnv / ManyEnvs of the same envs wrapped in gym_minigrid's wrapper"""
    import babyai_b200 as bb
    from babyai_b200.learner import DeviceManyEnvs, DeviceParallelEnv
    FullyObsWrapper, RGBImgObsWrapper = wrappers()
    n = 4
    envs = bb.make_envs(level, n, seed=3)
    wrapped = bb.FullyObsWrapper(envs) if wrapper == 'full' else bb.RGBImgObsWrapper(envs, tile_size=5)
    ref_wrap = FullyObsWrapper if wrapper == 'full' else (lambda e: RGBImgObsWrapper(e, tile_size=5))
    mode = 0 if kind == 'ParallelEnv' else 1
    ref = _ref_vec(kind, level, envs.seeds, ref_wrap)
    ours = (bb.ParallelEnv if mode == 0 else bb.ManyEnvs)(wrapped, pool=FullTensorPool(level, envs.seeds, mode))
    dev = (DeviceParallelEnv if mode == 0 else DeviceManyEnvs)(wrapped, pool=FullTensorPool(level, envs.seeds, mode))
    if mode == 1:
        ref.seed(envs.seeds)
        ours.seed(envs.seeds)
        dev.seed(envs.seeds)
    shape = ref.envs[0].observation_space.spaces['image'].shape
    if wrapper == 'rgb':                                   # gym_minigrid declares (W ts, H ts, 3); the array is (H ts, W ts, 3)
        shape = (shape[1], shape[0], 3)
    assert ours.observation_space.spaces['image'].shape == dev.observation_space.spaces['image'].shape == shape
    try:
        ro, oo, do = ref.reset(), ours.reset(), dev.reset()
        rng = np.random.RandomState(1)
        for t in range(60):
            for i in range(n):
                assert set(oo[i].keys()) == {'image', 'mission'} and oo[i]['mission'] == ro[i]['mission']
                assert np.array_equal(oo[i]['image'], ro[i]['image']), (t, i)
                assert np.array_equal(do.image[i].numpy(), ro[i]['image']), (t, i)
            a = rng.choice(7, n, p=P_RANDOM)
            ro, rr, rd, _ = ref.step(a)
            oo, orr, od, _ = ours.step(a)
            do, dr, dd, _ = dev.step(a)
            assert list(rd) == list(od) == [bool(x) for x in dd]
    finally:
        if kind == 'ParallelEnv':
            for r in ref.locals:
                r.send(('reset', None))
                r.recv()
            for p in ref.processes:
                p.terminate()


@pytest.mark.parametrize('fused_io', [False, True])
def test_device_facade_images_follow_the_state(fused_io):
    """DeviceParallelEnv over the host build: every batch (reset, per-step and fused steps) holds full_obs of every env's
    current state"""
    import babyai_b200 as bb
    from babyai_b200.learner import DeviceParallelEnv
    envs = bb.FullyObsWrapper(bb.make_envs('PutNextS5N2Carrying', 5, seed=2))
    pool = FullTensorPool('PutNextS5N2Carrying', envs.seeds)
    dev = DeviceParallelEnv(envs, pool=pool, fused_io=fused_io)
    obs = dev.reset()
    rng = np.random.RandomState(4)
    for t in range(80):
        for i in range(5):
            assert matches(obs.image[i].numpy(), expected(pool, i, 'PutNextS5N2Carrying')), (t, i)
        obs = next(dev.step(rng.choice(7, 5, p=P_RANDOM)))


@pytest.mark.reference
@pytest.mark.parametrize('level', ['KeyCorridorS3R1', 'BossLevel'])
def test_gym_minigrid_wrappers_run_on_single_env(level):
    """gymapi.SingleEnv has what gym_minigrid's wrappers read (width, height, grid.encode(), agent_pos, agent_dir, render):
    the wrappers as written run on it, and equal the same wrappers over the reference's level"""
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    import refenv
    refenv.setup('philox')
    from babyai_b200 import gymapi
    FullyObsWrapper, RGBImgObsWrapper = wrappers()
    for wrap in (FullyObsWrapper, lambda e: RGBImgObsWrapper(e, tile_size=4)):
        single = gymapi.make('BabyAI-%s-v0' % level, pool=FullTensorPool(level, [0], mode=1))
        ours = wrap(single)
        ref = wrap(shim_renderable(refenv.make_env(level, 77, 'philox')))
        assert single.width == ref.unwrapped.width and single.height == ref.unwrapped.height
        assert ours.observation_space.spaces['image'].shape == ref.observation_space.spaces['image'].shape
        ours.seed(77)
        ro, oo = ref.reset(), ours.reset()
        rng = np.random.RandomState(2)
        for t in range(50):
            assert np.array_equal(oo['image'], ro['image']) and oo['mission'] == ro['mission'], (level, t)
            assert np.array_equal(single.grid.encode(), ref.unwrapped.grid.encode()), (level, t)
            a = int(rng.choice(7, p=P_RANDOM))
            ro, _, rd, _ = ref.step(a)
            oo, _, od, _ = ours.step(a)
            assert rd == od
            if rd:
                ro, oo = ref.reset(), ours.reset()


def test_wrappers_validate_their_lists():
    import babyai_b200 as bb
    from babyai_b200.vecenv import _spaces
    envs = bb.make_envs('GoToLocal', 3)
    full = bb.FullyObsWrapper(envs)
    rgb = bb.RGBImgObsWrapper(envs, tile_size=6)
    assert full.image_shape() == (8, 8, 3) and full[0].observation_space.spaces['image'].shape == (8, 8, 3)
    assert bb.RGBImgObsWrapper(bb.make_envs('KeyCorridorS3R1', 2), 8).image_shape() == (24, 56, 3)
    assert bb.FullyObsWrapper(bb.make_envs('MoveTwoAcrossS5N2', 2)).image_shape() == (9, 5, 3)
    assert rgb.image_shape() == (48, 48, 3) and envs.image_shape() is None
    assert _spaces()[0].spaces['image'].shape == (7, 7, 3)
    for ts in (0, 65, 2.5, True):
        with pytest.raises(ValueError):
            bb.RGBImgObsWrapper(envs, tile_size=ts)
    with pytest.raises(TypeError):
        bb.FullyObsWrapper(list(envs))
    for wrapped in (full, rgb, bb.RGBImgPartialObsWrapper(envs)):
        with pytest.raises(ValueError):
            bb.FullyObsWrapper(wrapped)
    with pytest.raises(ValueError):                      # GoToLocal 8x8 and BossLevel 22x22
        bb.FullyObsWrapper(bb.make_envs({'GoToLocal': 2, 'BossLevel': 2}))
    same = bb.FullyObsWrapper(bb.make_envs({'GoToLocal': 2, 'PickupLoc': 2}))
    assert same.image_shape() == (8, 8, 3)
    for a, b in ((full, envs), (full, rgb), (rgb, bb.RGBImgObsWrapper(envs, tile_size=7)), (full, bb.RGBImgPartialObsWrapper(envs))):
        with pytest.raises(ValueError):
            a + b
    both = full + bb.FullyObsWrapper(bb.make_envs('PickupLoc', 2))
    assert both.full == 'grid' and both.level_counts() == [('GoToLocal', 3), ('PickupLoc', 2)]
    with pytest.raises(ValueError):
        full + bb.FullyObsWrapper(bb.make_envs('BossLevel', 2))


def test_c_abi_checks_arguments_without_a_device():
    from babyai_b200 import lib
    L = lib.load()
    ids = (C.c_int32 * 2)(0, 1)
    buf = (C.c_uint8 * 64)()
    assert L.bb_pool_full_obs(None, ids, 2, buf, None) != 0 and b'bad arguments' in L.bb_last_error()
    assert L.bb_pool_full_obs(None, None, 0, None, None) != 0


def test_sass_has_k_full_obs_without_local_memory():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    from babyai_b200 import build as b
    lib = b.build()
    out = subprocess.run([exe, '-sass', lib], capture_output=True, text=True, timeout=300).stdout
    assert 'sm_90a' in out
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = fns.setdefault(m.group(1), []) if 'k_full_obs' in m.group(1) else None
        elif cur is not None and re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+\S', line):
            cur.append(line)
    assert len(fns) == 2, sorted(fns)                      # all envs in order, an id list
    for name, code in fns.items():
        assert not any(re.search(r'\b(LDL|STL)\b', i) for i in code), name
        assert any(re.search(r'\bSTG\.E\b', i) for i in code) and any(re.search(r'\bSTG\.E\.U8\b', i) for i in code), name
        assert any(re.search(r'\bSTS\.U8\b', i) for i in code) and any(re.search(r'\bLDS\.U8\b', i) for i in code), name
