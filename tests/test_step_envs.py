"""Selected steps (bb_pool_step_envs, csrc/step8_sel.cuh) without a GPU: k_step8_sel's role on the host with one OS thread per
lane (tests/hostemu/step_envs_host.py), over the ring-layout pool with shallow rings that wrap often:
- against per-env references where only the listed envs step: one single-env oracle pool per env (ICLR levels) or one
  single-env host build (bonus levels), in both modes, with ragged and shuffled lists -- observation, reward, done, direction,
  mission, grid, pose and step count of every listed env after every call;
- unlisted envs: their records (state, ring, stream) and their output rows are byte-identical before and after every call;
- every id in order is k_step8's role, for int8 and int64 actions (outputs, counters, states, missions, ring positions and
  streams);
- one env stepped alone through many episode ends, and listed frozen envs;
- forks: save env a, load it into K children and expand each child with its own actions, against K `copy.deepcopy`s of the
  reference's unmodified level class on the shim, through an episode end;
- the built library: k_step8_sel stages with cp.async and uses no local memory."""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import reset_envs_host
import step_envs_host
from babyai_b200.levels import detokenize, level_spec
from step_envs_common import AUTORESET, FREEZE, SelMirror, compare_rows

P_ACT = [0.2, 0.2, 0.3, 0.1, 0.06, 0.12, 0.02]
D = 4                                                          # ring depth of the host pools: every ring turns over quickly


def _pool(level, seeds, mode=AUTORESET, depth=D):
    p = step_envs_host.StepEnvsPool(level_spec(level), len(seeds), np.asarray(seeds, np.uint64), depth=depth, mode=mode)
    size = reset_envs_host.ResetHostPool(level_spec(level), 1)
    p.width, p.height = size.width, size.height
    return p


def _same_as_mirror(pool, mirror, i, what):
    grid, info = pool.state(i, pool.width, pool.height)
    mg, mi = mirror.state(i)
    assert np.array_equal(grid, mg), (what, i, 'grid')
    assert [int(x) for x in info[:6]] == [mi[k] for k in ('agent_x', 'agent_y', 'agent_dir', 'carrying', 'step_count', 'max_steps')], (what, i)
    assert detokenize(pool.tokens(i)) == mirror.mission(i), (what, i, 'mission')


def _check_selected_steps(level, mode, seed, calls=90):
    n, rng = 37, np.random.RandomState(seed)                  # 3 CTAs of 16 envs when every id is listed, the last one ragged
    seeds = np.arange(n, dtype=np.uint64) * 3 + 200 + seed
    pool = _pool(level, seeds, mode)
    mirror = SelMirror(level, seeds, mode)
    mirror.reset()
    ended = replayed = 0
    for t in range(calls):
        k = [1, 3, 5, 17, n][t % 5]
        ids = rng.permutation(n)[:k].astype(np.int32)
        acts = rng.choice(7, size=k, p=P_ACT).astype(np.int8)
        before = pool.save_envs()
        obs = np.full((n, 7, 7, 3), 0xA5, np.uint8)
        rew, done, dirs = np.full(n, -9.5, np.float32), np.full(n, 0x77, np.uint8), np.full(n, -7, np.int8)
        frozen = set(mirror.frozen)
        obs, rew, done, dirs, cnt = pool.step_envs(ids, acts, obs, rew, done, dirs)
        want = mirror.step_envs(ids, acts)
        compare_rows((obs, rew, done, dirs), want, (level, mode, t))
        listed = np.zeros(n, bool)
        listed[ids] = True
        assert (obs[~listed] == 0xA5).all() and (rew[~listed] == -9.5).all(), (level, t, 'unlisted rows written')
        assert (done[~listed] == 0x77).all() and (dirs[~listed] == -7).all(), (level, t, 'unlisted rows written')
        after = pool.save_envs()
        assert np.array_equal(after[~listed], before[~listed]), (level, t, 'an unlisted env changed')
        for i in ids:
            _same_as_mirror(pool, mirror, int(i), (level, mode, t))
        ended += int(done[ids].sum())
        replayed += len(frozen & set(ids.tolist()))
    assert cnt[3] == 0 and pool.error_flag() == 0
    return ended, replayed


@pytest.mark.timeout(900)
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc', 'GoTo', 'BossLevel', 'Unlock', 'GoToImpUnlock', 'SynthSeq'])
def test_iclr_role_equals_oracle(level, mode):
    _check_selected_steps(level, mode, len(level) + mode)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['KeyCorridorS3R1', 'PutNextS4N1', 'OpenDoorsOrderN2', 'UnlockToUnlock', 'GoToObjDoor'])
def test_bonus_role_equals_host_build(level, mode):
    _check_selected_steps(level, mode, len(level) + mode)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
def test_episodes_end_and_frozen_envs_replay(mode):
    """a level whose episodes end within 64 steps: listed envs end episodes (auto-reset: swap in ring levels; freeze: replay)"""
    ended, replayed = _check_selected_steps('GoToRedBallNoDists', mode, 11, calls=300)
    assert ended >= 10, ended
    if mode == FREEZE:
        assert replayed >= 10, replayed


@pytest.mark.parametrize('level', ['GoToRedBallNoDists', 'Unlock', 'KeyCorridorS3R1'])
def test_one_env_alone_through_ring_wraps(level):
    """env 2 of 5 stepped alone, mostly `done` actions, until it has ended 4 D episodes (its ring wraps four times); the
    others never move, and their records are the same bytes at the end"""
    n, rng = 5, np.random.RandomState(4)
    seeds = np.arange(n, dtype=np.uint64) + 70
    pool = _pool(level, seeds)
    mirror = SelMirror(level, seeds, AUTORESET, [2])
    mirror.reset()
    others = [0, 1, 3, 4]
    before = pool.save_envs(others)
    ends = t = 0
    while ends < 4 * D:
        assert t < 20000, (level, 'episodes do not end')
        a = np.asarray([6 if rng.rand() < 0.8 else rng.randint(7)], np.int8)
        obs, rew, done, dirs, cnt = pool.step_envs([2], a)
        compare_rows((obs, rew, done, dirs), mirror.step_envs([2], a), (level, t))
        ends += int(done[2])
        t += 1
    _same_as_mirror(pool, mirror, 2, level)
    assert pool.ring(2)[0] == 1 + ends
    assert np.array_equal(pool.save_envs(others), before)
    assert cnt[0] == t and cnt[1] == ends and cnt[3] == 0 and pool.error_flag() == 0


@pytest.mark.parametrize('action_bytes', [1, 8])
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['GoToLocal', 'BossLevel', 'Unlock', 'KeyCorridorS3R1'])
def test_every_id_in_order_equals_step8_role(level, mode, action_bytes):
    n, rng = 37, np.random.RandomState(8)
    seeds = np.arange(n, dtype=np.uint64) + 1000
    A, B = _pool(level, seeds, mode), _pool(level, seeds, mode)
    ids = np.arange(n, dtype=np.int32)
    for t in range(40):
        a = rng.choice(7, size=n, p=P_ACT).astype(np.int8)
        oa, ra, da, qa, ca = A.step8(a)
        ob, rb, db, qb, cb = B.step_envs(ids, a.astype(np.int64) if action_bytes == 8 else a)
        assert np.array_equal(oa, ob) and np.array_equal(ra.view(np.uint32), rb.view(np.uint32)), (level, t)
        assert np.array_equal(da, db) and np.array_equal(qa, qb) and np.array_equal(ca, cb), (level, t)
    for i in range(n):                                         # (the two host refills count generation attempts differently)
        assert np.array_equal(A.state(i, A.width, A.height)[0], B.state(i, B.width, B.height)[0]), (level, i)
        assert np.array_equal(A.state(i, A.width, A.height)[1], B.state(i, B.width, B.height)[1]), (level, i)
        assert np.array_equal(A.tokens(i), B.tokens(i)) and A.ring(i)[:3] == B.ring(i)[:3], (level, i)
    assert ca[3] == 0 and (mode == FREEZE or ca[0] == 40 * n)


@pytest.mark.reference
@pytest.mark.timeout(900)
@pytest.mark.parametrize('level', ['GoToLocal', 'PutNextLocal', 'Unlock', 'KeyCorridorS3R1'])
def test_fork_and_expand_equals_deepcopy(level):
    """env a taken mid-episode by the reference and the pool alike; copy_envs into K children, each child expanded with its own
    actions, against K `copy.deepcopy`s of the reference env, until every child has ended an episode"""
    import refenv
    refenv.setup('philox')
    seed, K, a_env = 6000 + len(level), 4, 1
    rng = np.random.RandomState(seed)
    seeds = [seed + 7 * i for i in range(1 + K + 2)]
    seeds[a_env] = seed
    pool = _pool(level, seeds)
    ref = refenv.make_env(level, seed)
    ref.reset()
    for t in range(25):                                        # to mid-episode
        a = int(rng.choice(7, p=P_ACT))
        ob, r, d, _ = ref.step(a)
        if d:
            ob = ref.reset()
        o = pool.step_envs([a_env], np.asarray([a], np.int8))[0]
        assert np.array_equal(o[a_env], np.asarray(ob['image'], np.uint8)), (level, 'before', t)
    children = [2, 3, 4, 5]
    twins = [copy.deepcopy(ref) for _ in children]
    pool.copy_envs([a_env] * K, children)
    ended = np.zeros(K, bool)
    t = 0
    while not ended.all():
        assert t < 3000, (level, 'episodes do not end')
        acts = np.asarray([rng.choice(7, p=P_ACT) if rng.rand() < 0.7 else 6 for _ in children], np.int8)
        obs, rew, done, dirs, cnt = pool.step_envs(children, acts)
        for j, (c, tw) in enumerate(zip(children, twins)):
            ob, r, d, _ = tw.step(int(acts[j]))
            if d:
                ob = tw.reset()
            assert np.array_equal(obs[c], np.asarray(ob['image'], np.uint8)), (level, t, c)
            assert np.float32(rew[c]).view(np.uint32) == np.float32(r).view(np.uint32) and bool(done[c]) == bool(d), (level, t, c)
            assert int(dirs[c]) == int(ob['direction']) and detokenize(pool.tokens(c)) == ob['mission'], (level, t, c)
            ended[j] |= bool(d)
        t += 1
    assert cnt[3] == 0 and pool.error_flag() == 0


def test_step8_sel_kernels_stage_with_cp_async_and_use_no_local_memory():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    from babyai_b200 import build as b
    lib = b.build()
    out = subprocess.run([exe, '-sass', lib], capture_output=True, text=True, timeout=300).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = fns.setdefault(m.group(1), [])
        elif cur is not None and re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+\S', line):
            cur.append(line)
    found = {k: v for k, v in fns.items() if re.match(r'_Z\d+k_step8_selI', k)}
    assert sorted(re.search(r'ILi(\d)ELb(\d)', k).groups() for k in found) == [('1', '0'), ('1', '1'), ('8', '0'), ('8', '1')], list(found)
    for k, code in found.items():
        assert not any(re.search(r'\b(LDL|STL)\b', i) for i in code), (k, 'local memory')
        assert sum('LDGSTS' in i for i in code) >= 8, (k, 'the env record is staged with cp.async')
