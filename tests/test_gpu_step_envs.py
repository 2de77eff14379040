"""bb_pool_step_envs / BabyAIVecEnv.step_envs on the GPU, bit-exact against bb_pool_step, the oracle (ICLR levels) or the host
build (bonus levels), one single-env pool per env where only the listed envs step: observations, reward bit patterns, done,
direction, missions and hidden state.  Every test ends with counters()['errors'] == 0.

- Every id in order is bb_pool_step: outputs and counters, 3 D steps, 26 levels, both modes, int8 and int64 actions.
- Random subsets between bb_pool_step calls, bb_pool_rollout launches on the fused, in-stream-refill, concurrent-pass and graph
  paths, reset_envs with and without seeds, save / load rewinds and copy_envs forks, then 3 D further steps; 97 and 1 037 envs,
  and the BASELINE sizes with selections of several launches and one mirrored env per k_step8_sel CTA.
- The schedule on a ring of 8 levels: one env stepped alone through many episode ends between full steps.
- Untouched rows and records of unlisted envs, forks expanded with step_envs, rejected calls, stream order behind a held
  producer stream, render_grid and reset_envs right after a selected step."""
import ctypes as C
import gc

import numpy as np
import pytest

from reset_envs_common import BONUS_PER_KIND
from step_envs_common import AUTORESET, FREEZE, SelMirror, compare_rows

pytestmark = pytest.mark.gpu
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s at the H100's clock
P_ACT = [0.2, 0.2, 0.3, 0.1, 0.06, 0.12, 0.02]


def _np(x):
    return x.cpu().numpy()


def _pool(level, n, seeds, mode):
    from babyai_b200 import BabyAIVecEnv
    return BabyAIVecEnv(level, n, seeds=np.asarray(seeds, np.uint64), mode=mode)


def _dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device='cuda')


def _sentinels(n):
    import torch
    return [torch.full((n, 7, 7, 3), 0xA5, dtype=torch.uint8, device='cuda'), torch.full((n,), -9.5, device='cuda'),
            torch.full((n,), 0x77, dtype=torch.uint8, device='cuda'), torch.full((n,), -7, dtype=torch.int8, device='cuda')]


def _step_envs_checked(env, mirror, ids, acts, what):
    """step_envs into sentinel-filled outputs: the listed rows equal the mirror's, every other row keeps its sentinel"""
    n = env.num_envs
    outs = _sentinels(n)
    env.step_envs(ids, _dev(acts), *outs)
    o, r, d, q = [_np(x) for x in outs]
    listed = np.zeros(n, bool)
    listed[np.asarray(ids)] = True
    assert (o[~listed] == 0xA5).all() and (r[~listed] == -9.5).all(), (what, 'unlisted rows written')
    assert (d[~listed] == 0x77).all() and (q[~listed] == -7).all(), (what, 'unlisted rows written')
    compare_rows((o, r, d, q), mirror.step_envs(ids, acts), what)
    return o, r, d, q


def _mirror_state(env, mirror, envs, what):
    for i in envs:
        g, info = env.state(int(i))
        mg, mi = mirror.state(int(i))
        for k in ('draws', 'attempts'):
            info.pop(k), mi.pop(k)
        assert np.array_equal(g, mg) and info == mi, (what, int(i), info, mi)
    assert env.missions([int(i) for i in envs]) == [mirror.mission(int(i)) for i in envs], (what, 'missions')


# ------------------------------------------------------------------------------------------------------------------------
# every id in order is bb_pool_step
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc', 'GoTo', 'BossLevel', 'Unlock', 'GoToImpUnlock'] + BONUS_PER_KIND)
def test_every_id_in_order_equals_step(level, mode, monkeypatch):
    import torch
    monkeypatch.setenv('BB_RING_DEPTH', '16')                  # 3 D steps run through every ring several times
    n, D, rng = 97, 16, np.random.RandomState(len(level) + mode)
    for width in (torch.int8, torch.int64):
        a, b = _pool(level, n, np.arange(n) + 300, mode), _pool(level, n, np.arange(n) + 300, mode)
        a.reset()
        b.reset()
        ids = np.arange(n)
        for t in range(3 * D):
            act = torch.as_tensor(rng.choice(7, size=n, p=P_ACT), device='cuda').to(width)
            oa = [x.clone() for x in a.step(act)] + [a.direction.clone()]
            ob = list(b.step_envs(ids, act)) + [b.direction]
            assert all(torch.equal(x, y) for x, y in zip(oa, ob)), (level, mode, width, t)
        assert a.counters() == b.counters() and a.counters()['errors'] == 0, (level, mode, width)
        assert a.missions() == b.missions()
        for i in (0, n // 2, n - 1):
            assert a.state(i)[1] == b.state(i)[1] and np.array_equal(a.state(i)[0], b.state(i)[0]), (level, i)


# ------------------------------------------------------------------------------------------------------------------------
# random subsets against the oracle / host build, interleaved with every other entry point
# ------------------------------------------------------------------------------------------------------------------------
SINGLE_PATHS = {'step': {}, 'fused': {}, 'instream': {'BB_GEN_FUSED': '0'}, 'graph': {'BB_NO_PERSISTENT': '1'}}
MULTI_PATHS = {'step': {}, 'concurrent': {}, 'graph': {'BB_NO_PERSISTENT': '1'}}
SCHEDULES = [(lv, p) for lv in ('GoToLocal',) for p in SINGLE_PATHS] + \
            [(lv, p) for lv in ('BossLevel', 'Unlock', 'KeyCorridorS3R1') for p in MULTI_PATHS]


def _run_schedule(env, mirror, rng, T, per_step, rounds, tail_steps, what):
    import torch
    n, dev = env.num_envs, env.device
    outs = [torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device=dev), torch.zeros((T, n), dtype=torch.float32, device=dev),
            torch.zeros((T, n), dtype=torch.uint8, device=dev), torch.zeros((T, n), dtype=torch.int8, device=dev)]

    def chunk(steps):
        for t0 in range(0, steps, T):
            a = rng.randint(0, 7, (T, n)).astype(np.int8)
            if per_step:
                for t in range(T):
                    env.step(_dev(a[t]), *[x[t] for x in outs])
            else:
                env.rollout(_dev(a), *outs)
            got = [_np(x) for x in outs]
            for t in range(T):
                compare_rows([g[t] for g in got], mirror.step(a[t]), (what, 'step', t0 + t))

    saved = None
    for rnd in range(rounds):
        chunk(T * (1 + rng.randint(0, 2)))
        for j in range(6):                                     # selected steps: ragged subsets, int8 or int64 actions
            k = int(rng.choice([1, 3, 17, n // 2, n]))
            ids = rng.permutation(n)[:k]
            acts = rng.choice(7, size=k, p=P_ACT).astype(np.int64 if j % 2 else np.int8)
            _step_envs_checked(env, mirror, ids, acts, (what, rnd, j))
        op, touched = rnd % 4, []
        if op == 0 or op == 1:                                 # reset_envs with (op 0) and without seeds
            k = int(rng.randint(1, max(2, n // 3)))
            touched = rng.permutation(n)[:k]
            seeds = rng.randint(0, 2 ** 62, k).astype(np.uint64) if op == 0 else None
            env.reset_envs(touched, seeds)
            mirror.reset_envs(touched, seeds)
        elif op == 2:                                          # copy_envs: forks of mirrored envs
            src = rng.choice(mirror.ids, 5)
            touched = rng.permutation(np.setdiff1d(mirror.ids, src))[:5]
            env.copy_envs(src, touched)
            mirror.copy_envs(src, touched)
            saved = (mirror.ids[:9].copy(), env.save_envs(mirror.ids[:9]), mirror.save(mirror.ids[:9]))
        elif saved is not None:                                # load_envs: rewind to the records of the last fork round
            touched, rec, snap = saved
            env.load_envs(rec, touched)
            mirror.load(snap, touched)
        o, d = _np(env.obs), _np(env.direction)               # the rows the call wrote
        compare_rows((o, None, None, d), {int(i): mirror.last[int(i)] for i in touched if int(i) in mirror.envs}, (what, 'op', rnd))
    chunk(tail_steps)
    _mirror_state(env, mirror, mirror.ids[:64], what)
    assert env.counters()['errors'] == 0, what


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('n', [97, 1037])
@pytest.mark.parametrize('level,path', SCHEDULES)
def test_random_subsets(level, path, n, mode, monkeypatch):
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
    mirror = SelMirror(level, seeds, mode, mirrored)
    env.reset()
    mirror.reset()
    T = 1 if path == 'step' else (16 if multi else 20)
    _run_schedule(env, mirror, rng, T, path == 'step', 6, ((3 * D + T - 1) // T) * T, (level, path, n, mode))


@pytest.mark.parametrize('level,n,k', [('GoToLocal', 65536, 9000), ('BossLevel', 32768, 4500)])
def test_baseline_sizes_sampled(level, n, k):
    """selections of 9 000 (BossLevel: 4 500) ids -- three (two) k_step8_sel launches -- at the BASELINE pool sizes; the first
    list entry of every 16-entry CTA is mirrored, and full steps come between the selected ones"""
    rng = np.random.RandomState(n)
    seeds = np.arange(n, dtype=np.uint64) + 3
    env = _pool(level, n, seeds, AUTORESET)
    env.reset()
    ids = rng.permutation(n)[:k]
    sample = ids[::16]
    mirror = SelMirror(level, seeds, AUTORESET, sample)
    mirror.reset()
    cur = ids
    for t in range(12):
        acts = rng.choice(7, size=k, p=P_ACT).astype(np.int8)
        outs = _sentinels(n)
        env.step_envs(cur, _dev(acts), *outs)
        want = mirror.step_envs(cur, acts)
        got = [_np(x) for x in outs]
        compare_rows(got, want, (level, 'selected', t))
        other = np.setdiff1d(np.arange(n), ids)
        assert (got[0][other] == 0xA5).all() and (got[2][other] == 0x77).all()
        if t % 4 == 3:                                         # now and then a full step
            a = rng.randint(0, 7, n).astype(np.int8)
            got = [_np(x) for x in env.step(_dev(a))] + [_np(env.direction)]
            compare_rows(got, mirror.step(a), (level, 'full', t))
    _mirror_state(env, mirror, sample[:32], level)
    assert env.counters()['errors'] == 0


# ------------------------------------------------------------------------------------------------------------------------
# the schedule, untouched envs, forks
# ------------------------------------------------------------------------------------------------------------------------
def test_schedule_on_a_small_ring(monkeypatch):
    """a ring of 8 levels (a generation pass every 2 steps): env 5 stepped alone through 3 D episode ends, a full step every
    9th call -- the selected calls count as steps of the schedule, so the rings stay supplied"""
    monkeypatch.setenv('BB_RING_DEPTH', '8')
    n, D, rng = 97, 8, np.random.RandomState(6)
    seeds = np.arange(n) + 17
    env = _pool('GoToRedBallNoDists', n, seeds, AUTORESET)
    mirror = SelMirror('GoToRedBallNoDists', seeds, AUTORESET)
    env.reset()
    mirror.reset()
    ends = t = 0
    while ends < 3 * D:
        assert t < 5000
        if t % 9 == 8:
            a = rng.choice(7, size=n, p=P_ACT).astype(np.int8)
            got = [_np(x) for x in env.step(_dev(a))] + [_np(env.direction)]
            compare_rows(got, mirror.step(a), ('full', t))
        else:
            a = np.asarray([rng.choice(7, p=P_ACT)], np.int8)
            _, _, d, _ = _step_envs_checked(env, mirror, [5], a, ('alone', t))
            ends += int(d[5])
        t += 1
    _mirror_state(env, mirror, range(n), 'end')
    assert env.counters()['errors'] == 0


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', ['GoToLocal', 'BossLevel'])
def test_unlisted_envs_and_rows_untouched(level, mode, monkeypatch):
    import torch
    monkeypatch.setenv('BB_RING_DEPTH', '16')
    n, rng = 97, np.random.RandomState(mode)
    seeds = np.arange(n) + 900
    env = _pool(level, n, seeds, mode)
    mirror = SelMirror(level, seeds, mode)
    env.reset()                                                # every ring full: a pass that falls due has nothing to add
    mirror.reset()
    for t in range(40):
        k = int(rng.choice([1, 5, 40]))
        ids = rng.permutation(n)[:k]
        before = _np(env.save_envs(out=torch.zeros((n, env.record_bytes), dtype=torch.uint8, device='cuda')))
        _step_envs_checked(env, mirror, ids, rng.choice(7, size=k, p=P_ACT).astype(np.int8), (level, t))
        after = _np(env.save_envs(out=torch.zeros((n, env.record_bytes), dtype=torch.uint8, device='cuda')))   # (a record's unused tail is not written)
        listed = np.zeros(n, bool)
        listed[ids] = True
        assert np.array_equal(after[~listed], before[~listed]), (level, t, 'an unlisted env changed')
    assert env.counters()['errors'] == 0


@pytest.mark.parametrize('level', ['GoToLocal', 'Unlock'])
def test_fork_and_expand(level, monkeypatch):
    """copy_envs(src, children) then step_envs(children, one action each), compared to forks of the mirror, through episode
    ends; then the best child copied back over the source"""
    monkeypatch.setenv('BB_RING_DEPTH', '16')
    n, rng, K = 97, np.random.RandomState(9), 7
    seeds = np.arange(n) + 4000
    env = _pool(level, n, seeds, AUTORESET)
    mirror = SelMirror(level, seeds, AUTORESET)
    env.reset()
    mirror.reset()
    ends = 0
    for rnd in range(40):
        src = int(rng.randint(n))
        children = rng.permutation(np.setdiff1d(np.arange(n), [src]))[:K]
        env.copy_envs([src] * K, children)
        mirror.copy_envs([src] * K, children)
        for t in range(8):
            acts = rng.choice(7, size=K, p=P_ACT).astype(np.int8)
            _, r, d, _ = _step_envs_checked(env, mirror, children, acts, (level, rnd, t))
            ends += int(d[children].sum())
        best = int(children[np.argmax(_np(env.reward)[children])])
        env.copy_envs([best], [src])
        mirror.copy_envs([best], [src])
        _mirror_state(env, mirror, [src, best], (level, rnd))
    assert level != 'GoToLocal' or ends >= 3, ends             # (Unlock's episodes outlast these expansions)
    assert env.counters()['errors'] == 0


# ------------------------------------------------------------------------------------------------------------------------
# arguments, streams, other entry points
# ------------------------------------------------------------------------------------------------------------------------
def test_rejected_calls_launch_nothing():
    import torch
    from babyai_b200 import lib
    L = lib.load()
    n = 97
    env = _pool('BossLevel', n, np.arange(n), AUTORESET)
    env.reset()
    torch.cuda.synchronize()
    l0 = env.launches()
    p = lambda t: C.c_void_p(t.data_ptr())
    a8 = torch.zeros(4, dtype=torch.int8, device='cuda')
    for ids in ([3, 5, 3], [0, 97], [-1], [96, 200]):
        with pytest.raises(ValueError):
            env.step_envs(ids, a8[:len(ids)])
        i = np.asarray(ids, np.int32)
        assert L.bb_pool_step_envs(env.h, i.ctypes.data_as(C.c_void_p), i.size, p(a8), 1, p(env.obs), p(env.reward), p(env.done), None, None) != 0
    i = np.asarray([1, 2], np.int32)
    with pytest.raises(ValueError):
        env.step_envs(i, a8[:3])                               # one action per id
    with pytest.raises(ValueError):
        env.step_envs(i, torch.zeros(2, dtype=torch.int16, device='cuda'))
    assert L.bb_pool_step_envs(env.h, i.ctypes.data_as(C.c_void_p), 2, p(a8), 2, p(env.obs), p(env.reward), p(env.done), None, None) != 0
    for k in range(3):                                         # NULL obs, reward, done
        bufs = [p(env.obs), p(env.reward), p(env.done)]
        bufs[k] = None
        assert L.bb_pool_step_envs(env.h, i.ctypes.data_as(C.c_void_p), 2, p(a8), 1, *bufs, None, None) != 0
    assert L.bb_pool_step_envs(env.h, None, 2, p(a8), 1, p(env.obs), p(env.reward), p(env.done), None, None) != 0
    assert L.bb_pool_step_envs(env.h, i.ctypes.data_as(C.c_void_p), 2, None, 1, p(env.obs), p(env.reward), p(env.done), None, None) != 0
    assert env.launches() == l0
    env.step_envs([], torch.zeros(0, dtype=torch.int8, device='cuda'))      # n_sel = 0: nothing enqueued, not a step
    assert env.launches() == l0 and env.counters()['steps'] == 0 and env.counters()['errors'] == 0


def test_side_stream_behind_a_held_producer_stream():
    """pool.step on a producer stream behind a ~0.1 s spin kernel, then step_envs on another stream issued at once: the
    selected step must come after the full one"""
    import torch
    n, level = 97, 'BossLevel'
    rng = np.random.RandomState(4)
    a1 = rng.randint(0, 7, n).astype(np.int8)
    ids = rng.permutation(n)[:30]
    a2 = rng.randint(0, 7, 30).astype(np.int8)
    d1, d2 = _dev(a1), _dev(a2)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()

    def scenario(sleep):
        seeds = np.arange(n) + 70
        env = _pool(level, n, seeds, AUTORESET)
        env.reset()
        outs = _sentinels(n)
        torch.cuda.synchronize()
        gc.collect()
        gc.disable()
        try:
            with torch.cuda.stream(sa):
                sleep()
                env.step(d1)
            with torch.cuda.stream(sb):
                env.step_envs(ids, d2, *outs)
        finally:
            gc.enable()
        torch.cuda.synchronize()
        return env, outs, seeds

    scenario(lambda: None)[0].close()                          # kernels loaded: lazy loading cannot order the calls
    env, outs, seeds = scenario(lambda: torch.cuda._sleep(SLEEP_CYCLES))
    mirror = SelMirror(level, seeds, AUTORESET)
    mirror.reset()
    mirror.step(a1)
    compare_rows([_np(x) for x in outs], mirror.step_envs(ids, a2), 'selected step')
    _mirror_state(env, mirror, ids[:12], 'state after')
    assert env.counters()['errors'] == 0


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
def test_render_grid_and_reset_envs_after_selected_steps(mode):
    from render_grid_common import frame_of, matches
    n, rng = 64, np.random.RandomState(mode + 2)
    seeds = np.arange(n) + 5
    env = _pool('KeyCorridorS3R2', n, seeds, mode)
    mirror = SelMirror('KeyCorridorS3R2', seeds, mode)
    env.reset()
    mirror.reset()
    for t in range(30):
        ids = rng.permutation(n)[:int(rng.randint(1, n))]
        acts = rng.choice(7, size=ids.size, p=P_ACT).astype(np.int8)
        env.step_envs(ids, _dev(acts))                          # into the pool's own buffers: env.obs is the current view
        compare_rows([_np(env.obs), _np(env.reward), _np(env.done), _np(env.direction)], mirror.step_envs(ids, acts), t)
        frames = _np(env.render_grid(ids[:6], tile_size=8))
        obs = _np(env.obs)
        for j, i in enumerate(ids[:6]):
            assert matches(frames[j], frame_of(env, int(i), obs[i], 8)), (t, int(i))
        if t % 5 == 4:
            r = rng.permutation(ids)[:3]
            env.reset_envs(r)
            mirror.reset_envs(r)
            compare_rows((_np(env.obs), None, None, _np(env.direction)), {int(i): mirror.last[int(i)] for i in r}, ('reset', t))
    _mirror_state(env, mirror, range(n), 'end')
    assert env.counters()['errors'] == 0
