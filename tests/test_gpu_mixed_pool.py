"""Mixed-level pools (bb_pool_create_mixed / BabyAIVecEnv with (level, count) groups) on the GPU.  The reference of every test
is the definition of a mixed pool: its groups run as separate single-level BabyAIVecEnvs with the same seeds, compared byte for
byte -- observations, reward bit patterns, done, direction, mission tokens (the group's own width, zeros after it), the hidden
state of every env and the counters.  At the BASELINE sizes a slice of each group is checked against the C oracle instead.

- Level mixes: single-room (k_rollout) beside multi-room (k_step8 / k_rollout_cta), a bonus level, Unlock; one level in two
  groups; group sizes 1, 17, 32, 97, 1 037; both modes; 3 D steps of bb_pool_step with int8 and int64 actions.
- bb_pool_rollout with mixed T on the fused, in-stream-refill, concurrent-pass and graph paths.
- reset_envs with and without 64-bit seeds, step_envs with interleaved and shuffled id lists (unlisted rows untouched).
- step_host / step_learner / reset_host, a side-stream call behind a held producer stream, render_grid, excluded calls,
  n_groups = 1, the facades (DeviceParallelEnv + ObssPreprocessor, DeviceManyEnvs, ParallelEnv)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
AUTORESET, FREEZE = 0, 1
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s at the H100's clock


def _np(x):
    return x.cpu().numpy()


def _dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device='cuda')


def _seeds(groups, base):
    """one seed list per group, 64-bit values included"""
    return [np.arange(c, dtype=np.uint64) * np.uint64(7919) + np.uint64(base + 1000 * g) + (np.uint64(1) << np.uint64(40))
            for g, (_, c) in enumerate(groups)]


class Pair(object):
    """a mixed pool and its groups as separate pools, with the same seeds"""

    def __init__(self, groups, mode=AUTORESET, base=1):
        from babyai_b200 import BabyAIVecEnv
        self.groups = groups
        seeds = _seeds(groups, base)
        self.mixed = BabyAIVecEnv(groups, seeds=np.concatenate(seeds), mode=mode)
        self.sep = [BabyAIVecEnv(name, c, seeds=s, mode=mode) for (name, c), s in zip(groups, seeds)]
        self.starts = np.cumsum([0] + [c for _, c in groups])[:-1]
        self.n = self.mixed.num_envs

    def rows(self, g):
        return slice(int(self.starts[g]), int(self.starts[g]) + self.groups[g][1])

    def check_outputs(self, mixed_outs, sep_outs, what, axis=0):
        for k, (m, parts) in enumerate(zip(mixed_outs, zip(*sep_outs))):
            for g, part in enumerate(parts):
                got = np.take(m, np.arange(self.rows(g).start, self.rows(g).stop), axis=axis)
                assert got.tobytes() == np.ascontiguousarray(part).tobytes(), (what, 'output', k, 'group', g, self.groups[g])

    def check_state(self, what, every=1):
        tok = _np(self.mixed.mission_tokens)
        for g, e in enumerate(self.sep):
            st = _np(e.mission_tokens)
            r = self.rows(g)
            assert np.array_equal(tok[r, :st.shape[1]], st), (what, 'tokens', g)
            assert (tok[r, st.shape[1]:] == 0).all(), (what, 'token padding', g)
            for i in range(0, e.num_envs, every):
                gm, im = self.mixed.state(r.start + i)
                gs, is_ = e.state(i)
                for k in ('draws', 'attempts'):                 # how far a generator runs ahead depends on timing (k_gen_small's budget)
                    im.pop(k), is_.pop(k)
                assert np.array_equal(gm, gs) and im == is_, (what, 'state', g, i, im, is_)
        cs = [e.counters() for e in self.sep]
        assert self.mixed.counters() == {k: sum(c[k] for c in cs) for k in cs[0]}, (what, 'counters')
        assert self.mixed.counters()['errors'] == 0

    def reset(self):
        self.mixed.reset()
        for e in self.sep:
            e.reset()
        self.check_outputs([_np(self.mixed.obs), _np(self.mixed.direction)], [[_np(e.obs), _np(e.direction)] for e in self.sep], 'reset')


MIXES = {
    'room+multiroom': [('GoToLocal', 97), ('BossLevel', 17)],
    'bonus+unlock': [('GoToRedBall', 32), ('Unlock', 64), ('OpenTwoDoors', 17), ('GoToLocal', 1)],
    'one-level-twice': [('PickupLoc', 17), ('GoToObj', 32), ('PickupLoc', 1037)],
}


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('mix', sorted(MIXES))
def test_step_equals_groups(mix, mode, monkeypatch):
    import torch
    monkeypatch.setenv('BB_RING_DEPTH', '16')
    p = Pair(MIXES[mix], mode)
    p.reset()
    rng = np.random.RandomState(len(mix) + mode)
    for t in range(3 * 16):
        dtype = torch.int64 if t % 3 == 2 else torch.int8
        a = torch.as_tensor(rng.randint(0, 7, p.n)).to(dtype).cuda()
        p.mixed.step(a)
        for g, e in enumerate(p.sep):
            e.step(a[p.rows(g)].contiguous())
        p.check_outputs([_np(x) for x in (p.mixed.obs, p.mixed.reward, p.mixed.done, p.mixed.direction)],
                        [[_np(x) for x in (e.obs, e.reward, e.done, e.direction)] for e in p.sep], 'step %d' % t)
    p.check_state('after steps')


ROLLOUT_PATHS = {
    'fused': {},
    'in-stream-refill': {'BB_GEN_FUSED': '0'},
    'concurrent': {'BB_GEN_CONCURRENT': '1'},
    'graph': {'BB_NO_PERSISTENT': '1', 'BB_RING_DEPTH': '16'},
}


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('path', sorted(ROLLOUT_PATHS))
def test_rollout_equals_groups(path, mode, monkeypatch):
    import torch
    for k, v in ROLLOUT_PATHS[path].items():
        monkeypatch.setenv(k, v)
    p = Pair([('GoToRedBall', 64), ('BossLevel', 33), ('GoToLocal', 97), ('Unlock', 32)], mode, base=7)
    p.reset()
    rng = np.random.RandomState(5 + mode)
    for T in (40, 12, 40, 1, 25):
        a = rng.randint(0, 7, (T, p.n)).astype(np.int8)
        outs = [torch.zeros((T, p.n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros((T, p.n), device='cuda'),
                torch.zeros((T, p.n), dtype=torch.uint8, device='cuda'), torch.zeros((T, p.n), dtype=torch.int8, device='cuda')]
        p.mixed.rollout(_dev(a), *outs)
        sep = []
        for g, e in enumerate(p.sep):
            r = p.rows(g)
            so = [torch.zeros((T, e.num_envs) + tuple(x.shape[2:]), dtype=x.dtype, device='cuda') for x in outs]
            e.rollout(_dev(a[:, r]), *so)
            sep.append([_np(x) for x in so])
        p.check_outputs([_np(x) for x in outs], sep, 'rollout T=%d' % T, axis=1)
    p.check_state('after rollouts', every=3)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
def test_reset_envs_and_step_envs_split_by_group(mode, monkeypatch):
    import torch
    monkeypatch.setenv('BB_RING_DEPTH', '16')
    p = Pair([('GoToLocal', 17), ('BossLevel', 32), ('KeyInBox', 1), ('GoToLocal', 97)], mode, base=3)
    p.reset()
    rng = np.random.RandomState(9 + mode)
    for it in range(12):
        k = rng.randint(1, p.n)
        ids = rng.permutation(p.n)[:k] if it % 2 else np.sort(rng.permutation(p.n)[:k])
        if it % 3 == 0:                                         # interleaved across groups
            ids = np.asarray(sorted(ids, key=lambda i: (i % 5, i)))
        sentinels = [torch.full((p.n, 7, 7, 3), 0xA5, dtype=torch.uint8, device='cuda'), torch.full((p.n,), -9.5, device='cuda'),
                     torch.full((p.n,), 0x77, dtype=torch.uint8, device='cuda'), torch.full((p.n,), -7, dtype=torch.int8, device='cuda')]
        listed = np.zeros(p.n, bool)
        listed[ids] = True
        grp = p.mixed.group_of(ids)
        if it % 2 == 1:                                         # with 64-bit seeds, and without (the next level of each stream)
            seeds = (rng.randint(0, 2 ** 62, ids.size).astype(np.uint64) << np.uint64(1)) if it % 4 == 1 else None
            p.mixed.reset_envs(ids, seeds, obs=sentinels[0], direction=sentinels[3])
            sep = []
            for g, e in enumerate(p.sep):
                sel = grp == g
                o, q = torch.full((e.num_envs, 7, 7, 3), 0xA5, dtype=torch.uint8, device='cuda'), torch.full((e.num_envs,), -7, dtype=torch.int8, device='cuda')
                if sel.any():
                    e.reset_envs(ids[sel] - p.starts[g], None if seeds is None else seeds[sel], obs=o, direction=q)
                sep.append([_np(o), _np(q)])
            p.check_outputs([_np(sentinels[0]), _np(sentinels[3])], sep, 'reset_envs %d' % it)
        else:
            a = rng.randint(0, 7, ids.size).astype(np.int8)
            p.mixed.step_envs(ids, _dev(a), *sentinels)
            sep = []
            for g, e in enumerate(p.sep):
                sel = grp == g
                so = [torch.full_like(x[p.rows(g)], 0) for x in sentinels]
                for x, s0 in zip(so, sentinels):
                    x.copy_(s0[p.rows(g)])
                if sel.any():
                    e.step_envs(ids[sel] - p.starts[g], _dev(a[sel]), *so)
                sep.append([_np(x) for x in so])
            p.check_outputs([_np(x) for x in sentinels], sep, 'step_envs %d' % it)
        o = _np(sentinels[0])
        assert (o[~listed] == 0xA5).all(), 'unlisted rows written'
        if it % 3 == 2:                                         # full steps in between
            a = _dev(rng.randint(0, 7, p.n).astype(np.int8))
            p.mixed.step(a)
            for g, e in enumerate(p.sep):
                e.step(a[p.rows(g)].contiguous())
    p.check_state('after selected calls')


def test_host_buffer_calls_and_learner_step():
    p = Pair([('GoToLocal', 97), ('BossLevel', 17), ('PickupLoc', 32)], base=11)
    n = p.n
    obs, dire = np.zeros((n, 7, 7, 3), np.uint8), np.zeros(n, np.int8)
    p.mixed.reset_host(obs, dire)
    so = []
    for e in p.sep:
        o, q = np.zeros((e.num_envs, 7, 7, 3), np.uint8), np.zeros(e.num_envs, np.int8)
        e.reset_host(o, q)
        so.append([o, q])
    p.check_outputs([obs, dire], so, 'reset_host')
    rng = np.random.RandomState(2)
    import torch
    for t in range(40):
        a = rng.randint(0, 7, n).astype(np.int8)
        rew, done = np.zeros(n, np.float32), np.zeros(n, np.uint8)
        if t % 2:
            p.mixed.step_host(a, obs, rew, done, dire)
            outs = [obs, rew, done, dire]
        else:
            od, qd = torch.zeros((n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros(n, dtype=torch.int8, device='cuda')
            p.mixed.step_learner(a, od, rew, done, qd)
            outs = [_np(od), rew, done, _np(qd)]
        sep = []
        for g, e in enumerate(p.sep):
            o, r, d, q = np.zeros((e.num_envs, 7, 7, 3), np.uint8), np.zeros(e.num_envs, np.float32), np.zeros(e.num_envs, np.uint8), np.zeros(e.num_envs, np.int8)
            e.step_host(a[p.rows(g)], o, r, d, q)
            sep.append([o, r, d, q])
        p.check_outputs(outs, sep, 'host step %d' % t)
    p.check_state('after host steps')


def test_side_stream_behind_a_held_producer_stream():
    """a rollout on a producer stream behind a ~0.1 s spin kernel, then a step on another stream issued at once: the step
    must come after the rollout (the groups order their state between streams)"""
    import torch
    p = Pair([('GoToLocal', 97), ('BossLevel', 33)], base=5)
    p.reset()
    rng = np.random.RandomState(3)
    T = 20
    a1, a2 = rng.randint(0, 7, (T, p.n)).astype(np.int8), rng.randint(0, 7, p.n).astype(np.int8)
    d1, d2 = _dev(a1), _dev(a2)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ro = [torch.zeros((T, p.n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros((T, p.n), device='cuda'),
          torch.zeros((T, p.n), dtype=torch.uint8, device='cuda')]
    so = [torch.zeros((p.n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros(p.n, device='cuda'),
          torch.zeros(p.n, dtype=torch.uint8, device='cuda')]
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):
        torch.cuda._sleep(SLEEP_CYCLES)
        p.mixed.rollout(d1, *ro)
    with torch.cuda.stream(sb):
        p.mixed.step(d2, *so)
    torch.cuda.synchronize()
    for g, e in enumerate(p.sep):
        r = p.rows(g)
        o = [torch.zeros((T, e.num_envs) + tuple(x.shape[2:]), dtype=x.dtype, device='cuda') for x in ro]
        e.rollout(_dev(a1[:, r]), *o)
        e.step(_dev(a2[r]))
        assert np.array_equal(_np(ro[0])[:, r], _np(o[0])) and np.array_equal(_np(so[0])[r], _np(e.obs)), ('stream order', g)
        assert np.array_equal(_np(so[1])[r].view(np.uint32), _np(e.reward).view(np.uint32)), ('stream order', g)
    p.check_state('after streams', every=4)


def test_render_grid_one_size_and_mixed_sizes_rejected():
    p = Pair([('GoToLocal', 17), ('BossLevel', 9), ('PickupLoc', 12)], base=2)
    p.reset()
    ids = np.array([27, 3, 30, 0, 16, 37])                     # GoToLocal and PickupLoc: both 8 x 8
    got = _np(p.mixed.render_grid(ids, tile_size=8))
    for k, i in enumerate(ids):
        g = int(p.mixed.group_of(i))
        want = _np(p.sep[g].render_grid([int(i - p.starts[g])], tile_size=8))[0]
        assert np.array_equal(got[k], want), ('frame', k)
    boss = _np(p.mixed.render_grid(np.arange(17, 26), tile_size=3))
    assert np.array_equal(boss, _np(p.sep[1].render_grid(None, tile_size=3)))
    launches = p.mixed.launches()
    with pytest.raises(ValueError):
        p.mixed.render_grid([0, 17])
    with pytest.raises(ValueError):
        p.mixed.render_grid()
    import torch
    ids = (C.c_int32 * 2)(0, 17)
    out = torch.empty(2 * 22 * 22 * 3 * 64, dtype=torch.uint8, device='cuda')
    assert p.mixed.L.bb_pool_render_grid(p.mixed.h, ids, 2, 8, 1, C.c_void_p(out.data_ptr()), None) != 0
    assert b'grid size' in p.mixed.L.bb_last_error()
    assert p.mixed.launches() == launches


def test_excluded_calls_are_rejected_and_launch_nothing():
    import torch
    p = Pair([('GoToLocal', 32), ('BossLevel', 32)], base=4)
    p.reset()
    L, h = p.mixed.L, p.mixed.h
    launches = p.mixed.launches()
    rec = torch.zeros((64, 4096), dtype=torch.uint8, device='cuda')
    f = C.c_float()
    assert L.bb_pool_env_record_bytes(h) == 0 and b'mixed pool' in L.bb_last_error()
    assert L.bb_pool_save_envs(h, None, 64, C.c_void_p(rec.data_ptr()), None) != 0 and b'mixed pool' in L.bb_last_error()
    assert L.bb_pool_load_envs(h, None, None, 64, C.c_void_p(rec.data_ptr()), 64, None, None, None) != 0
    a = torch.zeros(64, dtype=torch.int8, device='cuda')
    assert L.bb_pool_step_timed(h, C.c_void_p(a.data_ptr()), 1, C.c_void_p(p.mixed.obs.data_ptr()), C.c_void_p(p.mixed.reward.data_ptr()),
                                C.c_void_p(p.mixed.done.data_ptr()), None, C.byref(f), C.byref(f)) != 0
    assert L.bb_pool_rollout_timed(h, C.c_void_p(a.data_ptr()), 1, C.c_void_p(p.mixed.obs.data_ptr()), C.c_void_p(p.mixed.reward.data_ptr()),
                                   C.c_void_p(p.mixed.done.data_ptr()), None, C.byref(f), C.byref(f)) != 0
    for call in (lambda: p.mixed.save_envs(), lambda: p.mixed.copy_envs([0], [1]), lambda: p.mixed.record_bytes,
                 lambda: p.mixed.step_timed(a), lambda: p.mixed.load_envs(rec)):
        with pytest.raises(RuntimeError):
            call()
    assert p.mixed.launches() == launches
    # the pool is unharmed
    a = _dev(np.random.RandomState(0).randint(0, 7, 64).astype(np.int8))
    p.mixed.step(a)
    for g, e in enumerate(p.sep):
        e.step(a[p.rows(g)].contiguous())
    p.check_outputs([_np(p.mixed.obs)], [[_np(e.obs)] for e in p.sep], 'step after rejected calls')


def test_introspection_and_one_group_is_a_plain_pool():
    from babyai_b200 import BabyAIVecEnv, lib
    from babyai_b200.levels import LevelSpec, level_spec
    L = lib.load()
    p = Pair([('GoToLocal', 17), ('BossLevel', 9), ('GoToLocal', 3)], base=8)
    assert L.bb_pool_num_groups(p.mixed.h) == 3 and p.mixed.num_envs == 29
    assert (p.mixed.width, p.mixed.height) == (22, 22)
    for g, (name, c) in enumerate(p.groups):
        s, n, spec = C.c_int32(), C.c_int32(), LevelSpec()
        assert L.bb_pool_group(p.mixed.h, g, C.byref(s), C.byref(n), C.byref(spec)) == 0
        assert (s.value, n.value) == (p.starts[g], c) and bytes(spec) == bytes(level_spec(name))
        assert p.mixed.level_of(int(p.starts[g])) == name
    assert p.mixed.groups == [('GoToLocal', 0, 17), ('BossLevel', 17, 9), ('GoToLocal', 26, 3)]
    assert p.mixed.max_tokens == max(e.max_tokens for e in p.sep)
    # n_groups = 1 is bb_pool_create
    seeds = np.arange(50, dtype=np.uint64) + 9
    one, plain = BabyAIVecEnv([('GoTo', 50)], seeds=seeds), BabyAIVecEnv('GoTo', 50, seeds=seeds)
    assert not one.mixed and L.bb_pool_num_groups(one.h) == 1 and one.record_bytes == plain.record_bytes
    one.reset(), plain.reset()
    a = _dev(np.random.RandomState(1).randint(0, 7, 50).astype(np.int8))
    one.step(a), plain.step(a)
    assert np.array_equal(_np(one.obs), _np(plain.obs)) and one.launches() == plain.launches()


def test_baseline_sizes_against_the_oracle():
    """32 768 GoToLocal + 32 768 BossLevel, three rollouts of 40 steps: a slice at the start, in the middle and at the end of
    each group against the oracle"""
    import torch
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    G = 32768
    seeds = np.arange(2 * G, dtype=np.uint64) + np.uint64(100)
    env = BabyAIVecEnv([('GoToLocal', G), ('BossLevel', G)], seeds=seeds)
    slices = [np.arange(0, 24), np.arange(G // 2 - 8, G // 2 + 8), np.arange(G - 8, G + 16), np.arange(2 * G - 16, 2 * G)]
    refs = []
    for sl in slices:
        for g in (0, 1):
            sub = sl[(sl >= g * G) & (sl < (g + 1) * G)]
            if sub.size:
                refs.append((sub, orc.OraclePool(['GoToLocal', 'BossLevel'][g], sub.size, seeds[sub])))
    obs0 = _np(env.reset())
    for sub, ref in refs:
        assert np.array_equal(obs0[sub], ref.reset()), 'reset'
    T, n = 40, 2 * G
    outs = [torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros((T, n), device='cuda'),
            torch.zeros((T, n), dtype=torch.uint8, device='cuda')]
    for rep in range(3):
        a = np.random.RandomState(rep).randint(0, 7, (T, n)).astype(np.int8)
        env.rollout(_dev(a), *outs)
        o, r, d = [_np(x) for x in outs]
        for t in range(T):
            for sub, ref in refs:
                oo, rr, dd = ref.step(a[t, sub])
                assert np.array_equal(o[t, sub], oo) and np.array_equal(r[t, sub].view(np.uint32), rr.view(np.uint32)) \
                    and np.array_equal(d[t, sub], dd), ('rollout', rep, t, sub[0])
    assert env.counters()['errors'] == 0
    tok = _np(env.mission_tokens)
    assert tok.shape == (n, 72) and (tok[:G, 16:] == 0).all()


def test_facades_on_a_mixed_list():
    import torch
    from babyai_b200 import DeviceManyEnvs, DeviceParallelEnv, ObssPreprocessor, ParallelEnv, make_envs
    from babyai_b200.vecenv import EnvList
    envs = make_envs({'GoToLocal': 40, 'BossLevel': 24}, seed=3)
    assert envs.seeds == [300 + i for i in range(64)]           # seeds count over the whole list
    parts = [EnvList('GoToLocal', envs.seeds[:40]), EnvList('BossLevel', envs.seeds[40:])]
    pre = ObssPreprocessor(trim=False)
    dm, ds = DeviceParallelEnv(envs), [DeviceParallelEnv(e) for e in parts]

    def same(a, bs, what):
        """the mixed batch `a` against the per-group batches `bs` concatenated, tokens padded to the mixed pool's width"""
        pa, pb = pre(a), [pre(b) for b in bs]
        width = pa.instr.shape[1]
        tok = torch.cat([torch.nn.functional.pad(b.instr, (0, width - b.instr.shape[1])) for b in pb])
        assert torch.equal(pa.image, torch.cat([b.image for b in pb])) and torch.equal(pa.instr, tok), what

    same(dm.reset(), [d.reset() for d in ds], 'reset')
    rng = np.random.RandomState(0)
    for t in range(30):
        a = rng.randint(0, 7, 64)
        om, rm, dnm, _ = dm.step(a)
        outs = [tuple(d.step(a[s:s + d.pool.num_envs])) for d, s in zip(ds, (0, 40))]
        same(om, [o[0] for o in outs], 'step %d' % t)
        assert np.array_equal(rm, np.concatenate([o[1] for o in outs])) and np.array_equal(dnm, np.concatenate([o[2] for o in outs]))
    # DeviceManyEnvs on the plain gym list batch_evaluate builds: maximal runs of one level become the groups
    fake = [type('Level_GoToLocal', (), {'level_name': 'GoToLocal'})() for _ in range(10)] + \
           [type('Level_PickupLoc', (), {'level_name': 'PickupLoc'})() for _ in range(6)]
    many = DeviceManyEnvs(fake)
    assert many.pool.groups == [('GoToLocal', 0, 10), ('PickupLoc', 10, 6)]
    seeds = list(range(500, 516))
    many.seed(seeds)
    sm = [DeviceManyEnvs(make_envs('GoToLocal', 10)), DeviceManyEnvs(make_envs('PickupLoc', 6))]
    sm[0].seed(seeds[:10]), sm[1].seed(seeds[10:])
    same(many.reset(), [m.reset() for m in sm], 'many reset')
    for t in range(20):
        a = rng.randint(0, 7, 16)
        om, rm, dnm, _ = many.step(a)
        outs = [tuple(sm[0].step(a[:10])), tuple(sm[1].step(a[10:]))]
        same(om, [o[0] for o in outs], 'many step %d' % t)
        assert rm == outs[0][1] + outs[1][1] and dnm == outs[0][2] + outs[1][2]
    # the host-buffer facade
    pm, ps = ParallelEnv(envs), [ParallelEnv(e) for e in parts]
    om = pm.reset()
    os_ = ps[0].reset() + ps[1].reset()
    assert [o['mission'] for o in om] == [o['mission'] for o in os_]
    assert all(np.array_equal(x['image'], y['image']) for x, y in zip(om, os_))
