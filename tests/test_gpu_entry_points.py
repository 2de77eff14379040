"""Every entry point of the pool against the oracle, and the pool's ordering of its own state between streams.

A. Ordering.  A producer stream holds a ~0.1 s spin kernel and pool calls behind it; the call under test is issued right away
   on another stream.  Without a dependency it runs first, every time, and the outputs differ from the oracle's.  Each
   scenario starts at a sync point with its generation pass finished and stays far inside one ring depth, so no level-supply
   wait can order the calls by accident; the caller's own tensors are created and synchronised before it.
B. The entry points nothing else compares with the oracle: step_host (pageable, page-locked under each BB_HOST_ZEROCOPY, no
   direction buffer, buffer sets that change), reset_host, step_learner (mapped and copy paths, side stream, mixed with step
   and rollout), step_timed and rollout_timed.
C. render_rgb at the shapes where k_render_rgb changes behaviour: empty, tiny, one more than a resident wave, several waves,
   an odd observation address, a misaligned output (rejected), an output above 4 GiB.

Comparisons are bit-exact: observation bytes, reward bit patterns, done, direction, missions of sampled envs, and every test
checks counters()['errors'] == 0.  Levels: GoToLocal (single room: k_rollout with T = 1 per step), BossLevel (multi-room:
k_step8 / k_rollout_cta) and Unlock (the untracked-carry kernels), 97 envs (a ragged CTA)."""
import ctypes as C
import gc

import numpy as np
import pytest

from render_grid_common import frame_of, matches
from test_rgb import pool_tiles

pytestmark = pytest.mark.gpu

LEVELS = ['GoToLocal', 'BossLevel', 'Unlock']
N = 97
AUTORESET, FREEZE = 0, 1
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 0.1 s at the H100's clock


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _lib():
    from babyai_b200 import lib
    return lib, lib.load()


class Ref(object):
    """The oracle stepped in the order of the pool's calls.  Freeze mode: an env that has ended repeats its last
    observation, reward and direction with done = 1 (the oracle itself keeps stepping it)."""

    def __init__(self, level, n, seeds, mode):
        import oracle as orc
        self.o = orc.OraclePool(level, n, seeds)
        self.n, self.freeze = n, mode == FREEZE
        self.frozen = np.zeros(n, bool)
        self.last = None

    def reset(self):
        self.frozen[:] = False
        obs = self.o.reset().copy()
        self.last = [obs, np.zeros(self.n, np.float32), np.zeros(self.n, np.uint8), self.o.direction.copy()]
        return obs, self.last[3]

    def step(self, a):
        o, r, d = self.o.step(np.asarray(a, np.int8), autoreset=not self.freeze)
        want = [o.copy(), r.copy(), d.copy(), self.o.direction.copy()]
        if self.freeze:
            f = self.frozen
            for k in (0, 1, 3):
                want[k][f] = self.last[k][f]
            want[2][f] = 1
            self.frozen |= want[2].astype(bool)
        self.last = want
        return want


def _np(x):
    return x.cpu().numpy() if hasattr(x, 'cpu') else np.asarray(x)


def same(got, want, what):
    """got: (obs, reward, done, direction or None) of the pool; want: the Ref's step outputs"""
    obs, rew, done = _np(got[0]), _np(got[1]), _np(got[2])
    n = len(want[1])
    bad = np.nonzero((obs.reshape(n, -1) != want[0].reshape(n, -1)).any(1))[0]
    assert len(bad) == 0, (what, 'obs differs for envs', bad[:8])
    assert np.array_equal(rew.astype(np.float32).view(np.uint32), want[1].view(np.uint32)), (what, 'reward')
    assert np.array_equal(done.astype(bool), want[2].astype(bool)), (what, 'done')
    if got[3] is not None:
        assert np.array_equal(_np(got[3]), want[3]), (what, 'direction')


def same_reset(obs, direction, want, what):
    bad = np.nonzero((_np(obs).reshape(len(want[1]), -1) != want[0].reshape(len(want[1]), -1)).any(1))[0]
    assert len(bad) == 0, (what, 'reset obs differs for envs', bad[:8])
    if direction is not None:
        assert np.array_equal(_np(direction), want[1]), (what, 'reset direction')


def check_pool(env, ref, what=''):
    probe = np.unique(np.r_[0, env.num_envs - 1, np.random.RandomState(env.num_envs).randint(0, env.num_envs, 12)])
    assert env.missions(probe) == [ref.o.mission(int(i)) for i in probe], (what, 'missions')
    assert env.counters()['errors'] == 0, what


def make(level, mode=AUTORESET, n=N, seed=1000):
    from babyai_b200 import BabyAIVecEnv
    seeds = np.arange(n, dtype=np.uint64) + seed
    return BabyAIVecEnv(level, n, seeds=seeds, mode=mode), Ref(level, n, seeds, mode)


def dev_out(env, T=None):
    """output tensors for the envs of `env` (None: N envs)"""
    import torch
    n, lead = (N if env is None else env.num_envs), (() if T is None else (T,))
    return [torch.zeros(lead + (n, 7, 7, 3), dtype=torch.uint8, device='cuda'),
            torch.zeros(lead + (n,), dtype=torch.float32, device='cuda'),
            torch.zeros(lead + (n,), dtype=torch.uint8, device='cuda'),
            torch.zeros(lead + (n,), dtype=torch.int8, device='cuda')]


def host_out(n, pinned=False):
    """(torch tensors that own the memory, their numpy views); pinned: page-locked"""
    import torch
    t = [torch.zeros((n, 7, 7, 3), dtype=torch.uint8), torch.zeros(n, dtype=torch.float32),
         torch.zeros(n, dtype=torch.uint8), torch.zeros(n, dtype=torch.int8)]
    if pinned:
        t = [x.pin_memory() for x in t]
    return t, [x.numpy() for x in t]


def spoil(bufs):
    """fill host outputs with values no step produces: an output the call does not write cannot pass for a right one"""
    for x in bufs:
        x[...] = -1 if x.dtype != np.uint8 else 0x55


def acts(rng, n, T=None, dtype=np.int8):
    return rng.randint(0, 7, n if T is None else (T, n)).astype(dtype)


def ready(level, mode=AUTORESET, n=N, seed=1000):
    """a reset pool and one step on the legacy stream, all finished: the scenario that follows starts after the generation
    pass the first step forked, and no step of it forks another (a pass is forked every 32nd step)"""
    import torch
    env, ref = make(level, mode, n, seed)
    env.reset()
    same_reset(env.obs, env.direction, ref.reset(), 'reset')
    a = acts(np.random.RandomState(seed), n)
    same(env.step(torch.as_tensor(a, device=env.device)) + (env.direction,), ref.step(a), 'first step')
    torch.cuda.synchronize()
    return env, ref


def rollout_same(outs, ref, a, what):
    for t in range(a.shape[0]):
        same([x[t] for x in outs], ref.step(a[t]), (what, t))


def step_host(env, a, bufs, direction=True):
    lib, L = _lib()
    a = np.ascontiguousarray(a, np.int8)
    o, r, d, q = bufs
    lib.check(L.bb_pool_step_host(env.h, _p(a), _p(o), _p(r), _p(d), _p(q) if direction else None))


def reset_host(env, bufs, direction=True):
    lib, L = _lib()
    lib.check(L.bb_pool_reset_host(env.h, _p(bufs[0]), _p(bufs[3]) if direction else None))


# ------------------------------------------------------------------------------------------------------------------------
# A. ordering
# ------------------------------------------------------------------------------------------------------------------------
def queued(level, mode, calls):
    """A scenario: calls(env, sleep) enqueues pool calls behind sleep() on a producer stream and the call under test on
    another.  It runs once on a spare pool of the same level first: CUDA loads a kernel at its first launch, and loading may
    synchronise the device, which would order the calls by accident.  Then on a pool at a sync point, with no garbage left to
    collect (bb_pool_destroy of a leftover pool synchronises the device too) and no collection while the calls are queued.
    Every tensor calls() touches exists already.  Returns the pool and its oracle."""
    import torch
    spare, _ = ready(level, mode)
    calls(spare, lambda: None)
    torch.cuda.synchronize()
    spare.close()
    env, ref = ready(level, mode)
    gc.collect()
    gc.disable()
    try:
        calls(env, lambda: torch.cuda._sleep(SLEEP_CYCLES))
    finally:
        gc.enable()
    torch.cuda.synchronize()
    return env, ref


@pytest.mark.parametrize('level', LEVELS)
@pytest.mark.parametrize('call', ['step_host', 'reset_host', 'step_timed', 'rollout_timed'])
def test_internal_stream_call_waits_for_the_callers_stream(level, call):
    """pool work on the caller's (legacy) stream behind a spin kernel, then a call that runs on the pool's internal stream"""
    import torch
    rng = np.random.RandomState(7)
    T = 6
    a1, a2 = acts(rng, N, T), acts(rng, N, T)
    out1, out2 = dev_out(None, T), dev_out(None, T)
    _own, hb = host_out(N)
    d1, d2 = torch.as_tensor(a1, device='cuda'), torch.as_tensor(a2, device='cuda')

    def calls(env, sleep):
        sleep()
        if call == 'rollout_timed':
            env.rollout(d1, *out1)
        else:
            env.step(d1[0], *[x[0] for x in out1])
        if call == 'step_host':
            env.step_host(a2[0], *hb)
        elif call == 'reset_host':
            env.reset_host(hb[0], hb[3])
        elif call == 'step_timed':
            env.step_timed(d2[0])
        else:
            env.rollout_timed(d2, *out2)

    env, ref = queued(level, AUTORESET, calls)
    if call == 'rollout_timed':
        rollout_same(out1, ref, a1, 'producer')
        rollout_same(out2, ref, a2, call)
    else:
        same([x[0] for x in out1], ref.step(a1[0]), 'producer')
        if call == 'step_host':
            same(hb, ref.step(a2[0]), call)
        elif call == 'reset_host':
            same_reset(hb[0], hb[3], ref.reset(), call)
        else:
            same((env.obs, env.reward, env.done, env.direction), ref.step(a2[0]), call)
    # and the pool goes on from the right state
    same(env.step(d1[1]) + (env.direction,), ref.step(a1[1]), 'after')
    check_pool(env, ref, call)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', LEVELS)
@pytest.mark.parametrize('call', ['step', 'rollout', 'reset', 'step_learner', 'render_grid'])
def test_call_on_a_second_side_stream_waits_for_the_first(level, mode, call):
    import torch
    from babyai_b200 import BabyAIVecEnv
    rng = np.random.RandomState(8)
    T = 5
    a1, a2 = acts(rng, N, 2), acts(rng, N, T)
    out1, out2 = dev_out(None, 2), dev_out(None, T)
    d1, d2 = torch.as_tensor(a1, device='cuda'), torch.as_tensor(a2, device='cuda')
    hr, hd = np.zeros(N, np.float32), np.zeros(N, np.uint8)
    probe = BabyAIVecEnv(level, 1)
    frames = torch.zeros((N, probe.height * 8, probe.width * 8, 3), dtype=torch.uint8, device='cuda')
    probe.close()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()

    def calls(env, sleep):
        with torch.cuda.stream(sa):
            sleep()
            env.step(d1[0], *[x[0] for x in out1])
            env.step(d1[1], *[x[1] for x in out1])
        with torch.cuda.stream(sb):
            if call == 'step':
                env.step(d2[0], *[x[0] for x in out2])
            elif call == 'rollout':
                env.rollout(d2, *out2)
            elif call == 'reset':
                env.reset(out2[0][0], out2[3][0])
            elif call == 'step_learner':
                env.step_learner(a2[0], out2[0][0], hr, hd, out2[3][0])
            else:
                env.render_grid(tile_size=8, out=frames)

    env, ref = queued(level, mode, calls)
    rollout_same(out1, ref, a1, 'producer')
    if call == 'step':
        same([x[0] for x in out2], ref.step(a2[0]), call)
    elif call == 'rollout':
        rollout_same(out2, ref, a2, call)
    elif call == 'reset':
        same_reset(out2[0][0], out2[3][0], ref.reset(), call)
    elif call == 'step_learner':
        same((out2[0][0], hr, hd, out2[3][0]), ref.step(a2[0]), call)
    else:
        f = frames.cpu().numpy()
        obs = out1[0][1].cpu().numpy()
        for i in range(N):
            assert matches(f[i], frame_of(env, i, obs[i], 8, True, level)), (call, i)
    check_pool(env, ref, call)


@pytest.mark.parametrize('level', LEVELS)
def test_legacy_stream_to_side_stream_and_back(level):
    import torch
    rng = np.random.RandomState(9)
    a = acts(rng, N, 4)
    d = torch.as_tensor(a, device='cuda')
    out = dev_out(None, 4)
    s = torch.cuda.Stream()

    def calls(env, sleep):
        sleep()                                           # legacy stream
        env.step(d[0], *[x[0] for x in out])
        with torch.cuda.stream(s):
            env.step(d[1], *[x[1] for x in out])
            sleep()
            env.step(d[2], *[x[2] for x in out])
        env.step(d[3], *[x[3] for x in out])              # legacy again

    env, ref = queued(level, AUTORESET, calls)
    rollout_same(out, ref, a, 'legacy -> side -> legacy')
    check_pool(env, ref)


def test_first_render_rgb_on_a_side_stream():
    """the tile table of a fresh pool is uploaded before a kernel on any stream reads it"""
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv('GoToLocal', 8, seeds=np.arange(8, dtype=np.uint64))
    obs = random_obs(4096, 3)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = env.render_rgb(obs)
    s.synchronize()
    assert torch.equal(out, assemble_dev(obs, dev_tiles()))
    env.close()


# ------------------------------------------------------------------------------------------------------------------------
# B. the entry-point matrix
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', LEVELS)
@pytest.mark.parametrize('buffers', ['pageable', 'pinned-zc0', 'pinned-zc1', 'pinned-zc2'])
def test_step_host(monkeypatch, level, mode, buffers):
    """bb_pool_step_host with and without a direction buffer (through the C ABI: the wrapper always passes one)"""
    if buffers != 'pageable':
        monkeypatch.setenv('BB_HOST_ZEROCOPY', buffers[-1])
    env, ref = make(level, mode)
    _own, h = host_out(N, pinned=buffers != 'pageable')
    reset_host(env, h)
    same_reset(h[0], h[3], ref.reset(), 'reset_host')
    rng = np.random.RandomState(10)
    for t in range(40):
        a = acts(rng, N)
        with_dir = t % 3 != 1
        spoil(h)
        step_host(env, a, h, direction=with_dir)
        same(h[:3] + [h[3] if with_dir else None], ref.step(a), (buffers, t))
        if not with_dir:
            assert (h[3] == -1).all(), 'a direction was written without a buffer'
    check_pool(env, ref)


@pytest.mark.parametrize('level', LEVELS)
def test_step_host_buffer_sets_that_change(level):
    """pinned -> pageable -> another pinned set -> the first again: each call must use what its buffers are now"""
    env, ref = make(level)
    sets = [host_out(N, True), host_out(N, False), host_out(N, True)]
    env.reset_host(sets[0][1][0], sets[0][1][3])
    same_reset(sets[0][1][0], sets[0][1][3], ref.reset(), 'reset_host')
    rng = np.random.RandomState(11)
    for t in range(32):
        h = sets[[0, 1, 2, 0][(t // 4) % 4]][1]
        spoil(h)
        a = acts(rng, N)
        step_host(env, a, h, direction=t % 5 != 2)
        same(h[:3] + [h[3] if t % 5 != 2 else None], ref.step(a), t)
    check_pool(env, ref)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', LEVELS)
def test_reset_host(level, mode):
    """at the start and mid-episode, with and without a direction buffer"""
    env, ref = make(level, mode)
    _own, h = host_out(N)
    rng = np.random.RandomState(12)
    for k, with_dir in enumerate((True, False, True)):
        spoil(h)
        reset_host(env, h, direction=with_dir)
        want = ref.reset()
        same_reset(h[0], h[3] if with_dir else None, want, ('reset', k))
        if not with_dir:
            assert (h[3] == -1).all()
        for t in range(7 + 5 * k):
            a = acts(rng, N)
            spoil(h)
            env.step_host(a, *h)
            same(h, ref.step(a), (k, t))
    check_pool(env, ref)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', LEVELS)
@pytest.mark.parametrize('zerocopy', ['0', '1'])
def test_step_learner(monkeypatch, level, mode, zerocopy):
    """mapped staging buffers (1) and copies (0), with and without dir_dev, on a side stream, between step and rollout calls
    (the first learner step after a rollout tops the rings up: sched_leave_rollout)"""
    import torch
    monkeypatch.setenv('BB_HOST_ZEROCOPY', zerocopy)
    env, ref = make(level, mode)
    rng = np.random.RandomState(13)
    s = torch.cuda.Stream()
    hr, hd = np.zeros(N, np.float32), np.zeros(N, np.uint8)
    T = 6
    with torch.cuda.stream(s):
        env.reset()
        same_reset(env.obs, env.direction, ref.reset(), 'reset')
        out = dev_out(env, T)
        for rep in range(3):
            for t in range(4):
                a = acts(rng, N)
                with_dir = (t + rep) % 2 == 0
                out[3][0].fill_(-1)
                spoil((hr, hd))
                env.step_learner(a, out[0][0], hr, hd, out[3][0] if with_dir else None)
                same((out[0][0], hr, hd, out[3][0] if with_dir else None), ref.step(a), (rep, 'learner', t))
                if not with_dir:
                    assert (out[3][0] == -1).all()
            a = acts(rng, N)
            same(env.step(torch.as_tensor(a, device=env.device)) + (env.direction,), ref.step(a), (rep, 'step'))
            a = acts(rng, N, T)
            env.rollout(torch.as_tensor(a, device=env.device), *out)
            rollout_same(out, ref, a, (rep, 'rollout'))
    check_pool(env, ref)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level', LEVELS)
def test_step_timed(level, mode):
    """int8 and int64 actions, between bb_pool_step calls; freeze mode against the oracle without auto-reset"""
    import torch
    env, ref = make(level, mode)
    env.reset()
    same_reset(env.obs, env.direction, ref.reset(), 'reset')
    rng = np.random.RandomState(14)
    out = dev_out(env)
    for t in range(30):
        a = acts(rng, N)
        if t % 3 == 2:
            same(env.step(torch.as_tensor(a, device=env.device), *out) + (out[3],), ref.step(a), ('step', t))
            continue
        d = torch.as_tensor(a.astype(np.int64) if t % 3 else a, device=env.device)
        ms_step, ms_gen = env.step_timed(d)
        assert ms_step > 0 and ms_gen > 0
        same((env.obs, env.reward, env.done, env.direction), ref.step(a), ('step_timed', t, d.dtype))
    check_pool(env, ref)


def test_step_timed_rejects_other_action_widths():
    import torch
    env, ref = ready('GoToLocal')
    L0 = env.launches()
    with pytest.raises(RuntimeError, match='action_bytes'):
        env.step_timed(torch.zeros(N, dtype=torch.int32, device=env.device))
    assert env.launches() == L0
    a = acts(np.random.RandomState(15), N)
    env.step_timed(torch.as_tensor(a, device=env.device))
    same((env.obs, env.reward, env.done, env.direction), ref.step(a), 'after the rejected call')
    check_pool(env, ref)


@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
@pytest.mark.parametrize('level,T', [('GoToLocal', 40), ('GoToLocal', 64), ('BossLevel', 40), ('Unlock', 40)])
def test_rollout_timed(level, T, mode):
    """T = 40: the persistent kernels, timed; T = 64 on a single-room level in auto-reset mode: the per-step graph (times 0);
    between rollout calls on the caller's stream"""
    import torch
    env, ref = make(level, mode)
    env.reset()
    same_reset(env.obs, env.direction, ref.reset(), 'reset')
    rng = np.random.RandomState(16)
    out = dev_out(env, T)
    graph = level == 'GoToLocal' and T == 64 and mode == AUTORESET
    for rep in range(4):
        a = acts(rng, N, T)
        d = torch.as_tensor(a, device=env.device)
        if rep % 2:
            env.rollout(d, *out)
        else:
            ms_kernel, ms_refill = env.rollout_timed(d, *out)
            assert (ms_kernel == 0 and ms_refill == 0) if graph else ms_kernel > 0, (ms_kernel, ms_refill)
        rollout_same(out, ref, a, rep)
    check_pool(env, ref)


# ------------------------------------------------------------------------------------------------------------------------
# C. render_rgb
# ------------------------------------------------------------------------------------------------------------------------
def dev_tiles():
    import torch
    return torch.as_tensor(pool_tiles(), device='cuda')


def assemble_dev(obs, tiles):
    """test_rgb.assemble on the device: a gather over the 513-tile table, uint8 [n, 7, 7, 3] -> [n, 56, 56, 3]"""
    import torch
    o = obs.reshape(-1, 7, 7, 3).long()
    cell = o[..., 0] | (o[..., 1] << 3) | (o[..., 2] << 6)
    ids = torch.where(o[..., 0] == 0, 256, cell)
    ids[:, 3, 6] = torch.where(o[:, 3, 6, 0] == 0, 256, 257 + cell[:, 3, 6])
    return tiles[ids].permute(0, 2, 3, 1, 4, 5).reshape(-1, 56, 56, 3)


def random_obs(n, seed, out=None):
    """observation bytes that select every tile: type 0..7 (0 = unseen), colour 0..7, state 0..3"""
    import torch
    g = torch.Generator(device='cuda').manual_seed(seed)
    o = torch.randint(0, 8, (n, 7, 7, 3), dtype=torch.uint8, device='cuda', generator=g)
    o[..., 2] &= 3
    if out is None:
        return o
    out.copy_(o)
    return out


def same_images(got, obs, tiles, chunk=32768):
    got, obs = got.reshape(-1, 56, 56, 3), obs.reshape(-1, 7, 7, 3)
    for k in range(0, obs.shape[0], chunk):
        want = assemble_dev(obs[k:k + chunk], tiles)
        if not bool((got[k:k + chunk] == want).all()):
            bad = (got[k:k + chunk] != want).reshape(want.shape[0], -1).any(1).nonzero()
            raise AssertionError('image %d differs (%d images)' % (k + int(bad[0]), len(bad)))


def test_render_rgb_shapes_and_waves():
    """empty (returns 0, launches nothing), 1, 7, one more than a resident wave of k_render_rgb (sm_count x 8 blocks of 8
    warps), three waves and a ragged tail, an observation buffer at an odd address, a misaligned output (rejected)"""
    import torch
    from babyai_b200 import BabyAIVecEnv
    lib, L = _lib()
    env = BabyAIVecEnv('GoToLocal', 8, seeds=np.arange(8, dtype=np.uint64))
    tiles = dev_tiles()
    wave = torch.cuda.get_device_properties(env.device).multi_processor_count * 8 * 8
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    obs = random_obs(8, 1)
    out = torch.zeros((9, 56, 56, 3), dtype=torch.uint8, device='cuda')
    L0 = env.launches()
    assert L.bb_pool_render_rgb(env.h, C.c_void_p(obs.data_ptr()), C.c_void_p(out.data_ptr()), 0, st) == 0
    assert env.launches() == L0 and int(out.sum()) == 0
    assert L.bb_pool_render_rgb(env.h, C.c_void_p(obs.data_ptr()), C.c_void_p(out.data_ptr() + 8), 1, st) != 0
    assert L.bb_pool_render_rgb(env.h, C.c_void_p(obs.data_ptr()), C.c_void_p(out.data_ptr() + 1), 1, st) != 0
    assert env.launches() == L0
    for n in (1, 7, wave + 1, 3 * wave + 37):
        obs = random_obs(n, n)
        out = torch.full((n + 1, 56, 56, 3), 0xEE, dtype=torch.uint8, device='cuda')
        env.render_rgb(obs, out[:n])
        same_images(out[:n], obs, tiles)
        assert bool((out[n] == 0xEE).all()), ('wrote past the last image', n)
        assert env.launches() == L0 + 1
        L0 += 1
    n = wave + 5
    buf = torch.zeros(n * 147 + 1, dtype=torch.uint8, device='cuda')
    obs = random_obs(n, 5, buf[1:].view(n, 7, 7, 3))
    assert obs.data_ptr() % 2 == 1
    same_images(env.render_rgb(obs), obs, tiles)
    env.close()


def test_render_rgb_rollout_buffer_above_4_gib():
    """a [8, 65 536] rollout's observations in one call: 4.9 GB of images, compared in slices"""
    import torch
    from babyai_b200 import BabyAIVecEnv
    T, n = 8, 65536
    env = BabyAIVecEnv('GoToLocal', n, seeds=np.arange(n, dtype=np.uint64))
    env.reset()
    out = dev_out(env, T)
    g = torch.Generator(device='cuda').manual_seed(17)
    env.rollout(torch.randint(0, 7, (T, n), dtype=torch.int8, device='cuda', generator=g), *out)
    pics = env.render_rgb(out[0])
    assert pics.shape == (T, n, 56, 56, 3) and pics.numel() > 4 * 2 ** 30
    same_images(pics, out[0], dev_tiles())
    assert env.counters()['errors'] == 0
    del pics
    env.close()
