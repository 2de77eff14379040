"""Mixed-level pools without a GPU.

- Token width: a group of a mixed pool generates its levels with lp.max_tokens raised to the widest group's (72 with a
  BossLevel group).  The host build of the generators (tests/hostemu/mixed_tokens_host.cpp) generates every level -- ICLR and
  bonus families, Unlock's untracked carry included -- at its natural width and at 72 from the same stream: grid, objects,
  instruction record, draws, attempts and tokens up to the natural width must agree, with zeros after it.
- The Python side: (level, count) groups, their validation, make_envs seeds over the whole list, EnvList concatenation, the
  pixel wrapper, the grouping of a plain list of reference envs, and what the facades hand the pool (a stand-in pool class).
- The C library's checks of bb_pool_create_mixed's arguments, which run before any device is touched."""
import ctypes as C
import os

import numpy as np
import pytest

from babyai_b200 import lib as bl
from babyai_b200 import vecenv
from babyai_b200.levels import BONUS_LEVELS, LEVELS, LevelSpec, level_spec

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'hostemu', 'mixed_tokens_host.cpp')
OUT = os.path.join(HERE, 'hostemu', 'libmixed_tokens_host.so')
WIDE = 72


def _mt():
    import hostemu
    deps = [SRC, os.path.join(HERE, '..', 'babyai_b200', 'csrc', 'env_logic.cuh'), os.path.join(HERE, '..', 'babyai_b200', 'csrc', 'level_params.h')]
    if not (os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in deps)):
        hostemu._compile(['g++', '-O1', '-std=c++17', '-Wall', '-Wno-unknown-pragmas', '-ffp-contract=off', '-shared', '-fPIC', SRC], OUT)
    L = C.CDLL(OUT)
    L.mt_max_tokens.argtypes = [C.c_void_p]
    L.mt_compare.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p]
    return L


@pytest.mark.parametrize('level', sorted(LEVELS))
def test_generators_at_the_mixed_token_width(level):
    L = _mt()
    spec = level_spec(level)
    natural = L.mt_max_tokens(C.byref(spec))
    assert 8 <= natural <= WIDE and natural % 8 == 0
    levels = 4 if spec.num_rows * spec.num_cols > 4 else 12
    for seed in (1, (1 << 40) + 17):
        tok = np.zeros((levels, WIDE), np.int16)
        rc = L.mt_compare(C.byref(spec), seed, levels, WIDE, tok.ctypes.data_as(C.c_void_p))
        assert rc == 0, (level, seed, 'level %d differs' % (rc - 1))
        assert (tok[:, 0] != 0).all()                            # every level got a mission


def test_token_widths_differ_between_families():
    """the width test above is not vacuous: most levels are narrower than BossLevel's 72"""
    L = _mt()
    widths = {name: L.mt_max_tokens(C.byref(level_spec(name))) for name in LEVELS}
    assert widths['BossLevel'] == WIDE and widths['GoToLocal'] < WIDE and widths['Unlock'] < WIDE
    assert any(widths[b] < WIDE for b in BONUS_LEVELS)


# ---- the Python side ---------------------------------------------------------------------------------------------------
def test_level_groups():
    assert vecenv.level_groups('GoToLocal') is None
    assert vecenv.level_groups({'GoToLocal': 3, 'BossLevel': 2}) == [('GoToLocal', 3), ('BossLevel', 2)]
    assert vecenv.level_groups([('GoTo', 1), ('GoTo', 4)]) == [('GoTo', 1), ('GoTo', 4)]
    for bad in ([], [('GoTo', 0)], [('GoTo', 1.5)], [('GoTo', True)], [('GoTo',)], ['GoTo'], [(3, 4)], {'GoTo': -1},
                [('GoTo', 2 ** 31 - 1), ('GoTo', 1)]):
        with pytest.raises(ValueError):
            vecenv.level_groups(bad)
    with pytest.raises(KeyError):
        vecenv.level_groups([('NoSuchLevel', 2)])


def test_make_envs_groups_and_seeds():
    e = vecenv.make_envs({'GoToLocal': 3, 'BossLevel': 2}, seed=4)
    assert e.level == [('GoToLocal', 3), ('BossLevel', 2)] and len(e) == 5
    assert e.seeds == [400, 401, 402, 403, 404]                  # 100 * seed + i over the whole list (train_rl.py:53-60)
    assert [h.index for h in e] == list(range(5))
    assert vecenv.make_envs([('GoTo', 2)], seed=1).level == 'GoTo'
    assert vecenv.make_envs({'GoTo': 2, 'Open': 1}, num_envs=3).seeds == [100, 101, 102]
    with pytest.raises(ValueError):
        vecenv.make_envs({'GoTo': 2, 'Open': 1}, num_envs=4)
    assert vecenv.make_envs('GoTo', 3, seed=2).seeds == [200, 201, 202]


def test_env_lists_concatenate():
    a, b = vecenv.make_envs('GoToLocal', 2, seed=1), vecenv.make_envs({'BossLevel': 1, 'GoToLocal': 2}, seed=7)
    c = a + b
    assert isinstance(c, vecenv.EnvList)
    assert c.level == [('GoToLocal', 2), ('BossLevel', 1), ('GoToLocal', 2)]
    assert c.seeds == [100, 101, 700, 701, 702] and len(c) == 5
    assert c.level_counts() == [('GoToLocal', 2), ('BossLevel', 1), ('GoToLocal', 2)]
    with pytest.raises(ValueError):
        a + vecenv.RGBImgPartialObsWrapper(b)
    px = vecenv.RGBImgPartialObsWrapper(c)
    assert px.pixel and px.level == c.level and px.seeds == c.seeds
    assert px[0].observation_space.spaces['image'].shape == (56, 56, 3)


def _gym(name):
    return type('Level_' + name, (), {'level_name': name})()


def test_plain_reference_lists_group_by_runs_of_one_level():
    envs = [_gym('GoToLocal')] * 3 + [_gym('BossLevel')] * 2 + [_gym('GoToLocal')]
    e = vecenv._as_env_list(envs, need_seeds=False)
    assert e.level == [('GoToLocal', 3), ('BossLevel', 2), ('GoToLocal', 1)] and len(e) == 6
    assert vecenv._as_env_list([_gym('GoTo')] * 4, need_seeds=False).level == 'GoTo'
    with pytest.raises(TypeError):
        vecenv._as_env_list(envs, need_seeds=True)
    with pytest.raises(TypeError):
        vecenv._as_env_list([_gym('GoTo'), object()], need_seeds=False)


class _FakePool(object):
    """records what a facade builds its pool from"""
    made = []

    def __init__(self, level, num_envs=None, seeds=None, device=0, mode=0):
        groups = vecenv.level_groups(level) or [(level, num_envs)]
        self.level, self.num_envs, self.seeds, self.mode = level, sum(c for _, c in groups), seeds, mode
        _FakePool.made.append(self)


def test_facades_build_one_mixed_pool(monkeypatch):
    from babyai_b200 import learner
    monkeypatch.setattr(vecenv, 'BabyAIVecEnv', _FakePool)
    monkeypatch.setattr(learner, 'BabyAIVecEnv', _FakePool)
    monkeypatch.setattr(vecenv.torch.Tensor, 'pin_memory', lambda t: t)
    envs = vecenv.make_envs({'GoToLocal': 3, 'PickupLoc': 2}, seed=2)
    _FakePool.made[:] = []
    vecenv.ParallelEnv(envs)
    learner.DeviceParallelEnv(envs)
    vecenv.ManyEnvs([_gym('GoTo')] * 2 + [_gym('Open')])
    learner.DeviceManyEnvs([_gym('GoTo')] * 2 + [_gym('Open')])
    p, d, m, dm = _FakePool.made
    for pool in (p, d):
        assert pool.level == [('GoToLocal', 3), ('PickupLoc', 2)] and pool.num_envs == 5 and pool.seeds == [200, 201, 202, 203, 204]
        assert pool.mode == vecenv.MODE_AUTORESET
    for pool in (m, dm):
        assert pool.level == [('GoTo', 2), ('Open', 1)] and pool.mode == vecenv.MODE_FREEZE


# ---- the C library's argument checks (no device needed: they run first) ------------------------------------------------
def test_create_mixed_checks_arguments_first():
    if not os.path.exists(bl.LIB_PATH):
        import babyai_b200.build as b
        b.build()
    L = bl.load()
    specs = (LevelSpec * 3)(level_spec('GoToLocal'), level_spec('BossLevel'), level_spec('GoToLocal'))
    h = C.c_void_p()

    def create(counts, n_groups=None, sp=specs):
        c = (C.c_int32 * len(counts))(*counts)
        rc = L.bb_pool_create_mixed(sp, c, len(counts) if n_groups is None else n_groups, 0, C.byref(h))
        return rc, L.bb_last_error().decode()

    assert create([4, 0, 2]) == (1, 'every group needs at least one env')
    assert create([4, -3, 2])[0] == 1
    assert create([2 ** 31 - 2, 1, 1]) == (1, 'a pool holds at most INT32_MAX envs')
    assert create([1, 1], n_groups=0) == (1, 'bad arguments')
    bad = (LevelSpec * 2)(level_spec('GoToLocal'), LevelSpec())
    bad[1].kind = 99
    rc, msg = create([2, 2], sp=bad)
    assert rc == 1 and msg and 'CUDA' not in msg
    assert L.bb_pool_create_mixed(None, None, 1, 0, C.byref(h)) == 1
    assert L.bb_pool_num_groups(None) == 0
    import torch
    if not torch.cuda.is_available():
        rc, msg = create([4, 4, 1])
        assert rc == 1 and 'CUDA' in msg                         # valid arguments: then the device is needed
