"""The rollout path (bb_pool_rollout: k_rollout, k_rollout_cta, the CUDA-graph fallback, the level-supply schedules) against
the reference traces, the C oracle and the host build, at the sizes and call sequences where it changes shape: many CTAs and
a ragged last one, a second wave of CTAs, changing rollout lengths, freeze mode, done-action mode, the bonus levels and the
tuning knobs that select other kernels.  Bit-exact, as in the rest of the suite: observation bytes, reward bit patterns, done,
direction, missions, counters."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from common import BONUS_GOLDENS, DONE_GOLDENS, GOLDEN_LEVELS, SUCCESS_GOLDENS, golden_level, replay_golden_rollout  # noqa: E402

ALL_GOLDENS = GOLDEN_LEVELS + SUCCESS_GOLDENS + DONE_GOLDENS + BONUS_GOLDENS


def _single_room(level):
    from babyai_b200.levels import level_spec
    s = level_spec(level)
    return s.num_rows * s.num_cols == 1


def _bufs(T, n):
    import torch
    return (torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device='cuda'), torch.zeros((T, n), dtype=torch.float32, device='cuda'),
            torch.zeros((T, n), dtype=torch.uint8, device='cuda'), torch.zeros((T, n), dtype=torch.int8, device='cuda'))


def _rollout_vs(env, ref, acts, tag, sel=None, autoreset=True, nthreads=1, frozen=None):
    """one env.rollout(acts) against T steps of `ref` (an OraclePool, or a HostEmuPool when autoreset is None); `sel`: the
    env indices `ref` holds.  Freeze mode (autoreset=False): envs in `frozen` must repeat their last output."""
    import torch
    T, n = acts.shape
    obs, rew, done, dirs = _bufs(T, n)
    env.rollout(torch.as_tensor(acts, device='cuda'), obs, rew, done, dirs)
    pick = (lambda x: x.cpu().numpy()) if sel is None else (lambda x: x[:, torch.as_tensor(sel, device='cuda')].cpu().numpy())
    ho, hr, hd, hq = pick(obs), pick(rew), pick(done), pick(dirs)
    a = acts if sel is None else acts[:, sel]
    eps = 0
    for t in range(T):
        if autoreset is None:
            oo, rr, dd = [np.array(x) for x in ref.step(a[t])]
        else:
            oo, rr, dd = [np.array(x) for x in ref.step(a[t], autoreset=autoreset, nthreads=nthreads)]
        qq = np.array(ref.direction)
        if frozen is not None:
            for i in np.nonzero(frozen[0])[0]:
                oo[i], rr[i], dd[i], qq[i] = frozen[1][i]
        bad = np.nonzero((ho[t] != oo).reshape(len(oo), -1).any(1))[0]
        assert len(bad) == 0, (tag, t, 'obs differs for envs', bad[:8] if sel is None else np.asarray(sel)[bad[:8]])
        assert np.array_equal(hr[t].view(np.uint32), rr.view(np.uint32)), (tag, t, 'reward', np.nonzero(hr[t] != rr)[0][:8])
        assert np.array_equal(hd[t], dd.astype(np.uint8)), (tag, t, 'done', np.nonzero(hd[t] != dd)[0][:8])
        assert np.array_equal(hq[t], qq), (tag, t, 'direction')
        if frozen is not None:
            for i in np.nonzero(dd & ~frozen[0])[0]:
                frozen[0][i] = True
                frozen[1][i] = (oo[i].copy(), rr[i], dd[i], qq[i])
        eps += int(dd.sum())
    return eps


def _step_vs(env, ref, act, tag):
    import torch
    o, r, d = env.step(torch.as_tensor(act, device='cuda'))
    oo, rr, dd = ref.step(act)
    assert np.array_equal(o.cpu().numpy(), oo), (tag, 'obs')
    assert np.array_equal(r.cpu().numpy().view(np.uint32), rr.view(np.uint32)) and np.array_equal(d.cpu().numpy(), dd), (tag, 'reward / done')
    assert np.array_equal(env.direction.cpu().numpy(), ref.direction), (tag, 'direction')
    return int(dd.sum())


def _missions_vs(env, ref, tag, idx):
    assert env.missions(idx) == [ref.mission(i) for i in idx], tag


# ---- 1. every golden file through bb_pool_rollout (and bb_pool_step), replicated over many CTAs --------------------
def _replica_count(level):
    # single-room: 64 envs per k_rollout CTA, 65 CTAs + a ragged one; multi-room: 32 per k_rollout_cta CTA, 32 + a ragged one
    return 4096 + 37 if _single_room(level) else 1024 + 13


@pytest.mark.timeout(180)
@pytest.mark.parametrize('name', ALL_GOLDENS)
def test_golden_replicated_through_rollout_and_step(name, monkeypatch):
    """Reference traces through bb_pool_rollout with a chunk schedule of mixed lengths (T = 64 takes the graph path on
    single-room levels; every change of T restarts the refill schedule), then the same replicated replay through
    bb_pool_step.  done_* files run in done-action mode."""
    if name.startswith('done_'):
        monkeypatch.setenv('BABYAI_DONE_ACTIONS', '1')
    n = _replica_count(golden_level(name))
    eps = replay_golden_rollout(name, n)
    assert eps > 0 or name in ('Open', 'PutNext', 'UnblockPickup', 'GoToObjMaze', 'GoToObjMazeOpen', 'GoToObjMazeS7')
    assert replay_golden_rollout(name, n, per_step=True) == eps


# ---- 3. the benchmark configurations at their full size against the C oracle -----------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize('level,n', [('GoToLocal', 65536), ('PickupLoc', 65536), ('GoTo', 32768), ('BossLevel', 32768)])
def test_bench_size_golden_replay(level, n):
    """BASELINE configs 2-5 at their per-GPU size: the replicated reference traces through bb_pool_rollout (65 536 envs take
    1 024 k_rollout CTAs, more than one resident wave)."""
    assert replay_golden_rollout(level, n) > 0


def _warm_up(env, ref, n, steps, seed):
    """`steps` random actions through bb_pool_rollout (40 per call) and the oracle; nothing compared"""
    import torch
    rng = np.random.RandomState(seed)
    obs, rew, done, dirs = _bufs(40, n)
    for k in range(0, steps, 40):
        acts = rng.randint(0, 7, (40, n)).astype(np.int8)
        env.rollout(torch.as_tensor(acts, device='cuda'), obs, rew, done, dirs)
        for t in range(40):
            ref.step(acts[t], nthreads=16)


@pytest.mark.timeout(900)
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc'])
def test_bench_size_single_room_every_env_matches_oracle(level):
    """BASELINE configs 2 and 3: 65 536 envs, every env compared with the oracle after the fused generator warps reached
    their steady state (80 steps >= max_steps): four 40-step rollouts and a ragged one, CTAs of the second wave included."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    n = 65536
    seeds = np.array([100 + i for i in range(n)], dtype=np.uint64)
    env, ref = BabyAIVecEnv(level, n, seeds=seeds), orc.OraclePool(level, n, seeds)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    _warm_up(env, ref, n, 80, seed=21)
    rng = np.random.RandomState(22)
    eps = 0
    for k, T in enumerate([40, 40, 40, 40, 23]):
        eps += _rollout_vs(env, ref, rng.randint(0, 7, (T, n)).astype(np.int8), (level, k), nthreads=16)
    _missions_vs(env, ref, level, list(range(0, n, 97)) + [n - 1])
    c = env.counters()
    assert eps > n // 4 and c['errors'] == 0 and c['steps'] == n * 263


@pytest.mark.timeout(900)
@pytest.mark.parametrize('level', ['GoTo', 'BossLevel'])
def test_bench_size_multi_room_sample_matches_oracle(level):
    """BASELINE configs 4 and 5: 32 768 envs (1 024 k_rollout_cta CTAs of 32 envs); the oracle follows 4 096 of them: three
    envs of every CTA, the whole last CTA and the highest env indices."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    n = 32768
    rng = np.random.RandomState(5)
    sel = np.unique(np.r_[(np.arange(n // 32)[:, None] * 32 + rng.randint(0, 32, (n // 32, 3))).ravel(), np.arange(n - 32, n)])
    sel = np.unique(np.r_[sel, rng.choice(np.setdiff1d(np.arange(n), sel), 4096 - len(sel), replace=False)])
    assert len(sel) == 4096 and len(np.unique(sel // 32)) == n // 32
    seeds = np.array([100 + i for i in range(n)], dtype=np.uint64)
    env, ref = BabyAIVecEnv(level, n, seeds=seeds), orc.OraclePool(level, len(sel), seeds[sel])
    assert np.array_equal(env.reset().cpu().numpy()[sel], ref.reset())
    eps = 0
    for k, T in enumerate([40, 40, 40, 40, 40, 40, 23]):
        eps += _rollout_vs(env, ref, rng.randint(0, 7, (T, n)).astype(np.int8), (level, k), sel=sel, nthreads=16)
    got = env.missions(sel)
    assert got == [ref.mission(i) for i in range(len(sel))]
    assert env.counters()['errors'] == 0


# ---- 4. modes, call sequences, CTA boundaries (ICLR levels, against the oracle) ----------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize('level,n,steps', [('PickupLoc', 200, 80), ('GoTo', 130, 600)])
def test_freeze_mode_through_rollout(level, n, steps):
    """BB_MODE_FREEZE through bb_pool_rollout (k_rollout / k_rollout_cta): finished envs repeat their last output; then
    MODE_AUTORESET, reset() and more rollouts against the oracle with auto-reset."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    from babyai_b200.vecenv import MODE_AUTORESET, MODE_FREEZE
    seeds = np.arange(n, dtype=np.uint64) + 31337
    env, ref = BabyAIVecEnv(level, n, seeds=seeds, mode=MODE_FREEZE), orc.OraclePool(level, n, seeds)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    rng = np.random.RandomState(8)
    frozen = (np.zeros(n, bool), [None] * n)
    for k, T in enumerate([40, 7, 33] + [40] * ((steps - 80) // 40)):
        _rollout_vs(env, ref, rng.randint(0, 7, (T, n)).astype(np.int8), (level, 'freeze', k), autoreset=False, frozen=frozen)
    assert frozen[0].all()
    env.set_mode(MODE_AUTORESET)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    _missions_vs(env, ref, (level, 'missions after reset'), range(n))
    for k, T in enumerate([40, 40, 13]):
        _rollout_vs(env, ref, rng.randint(0, 7, (T, n)).astype(np.int8), (level, 'autoreset', k))
    assert env.counters()['errors'] == 0


@pytest.mark.timeout(300)
@pytest.mark.parametrize('level,n', [('PickupLoc', 300), ('GoToLocal', 200), ('GoTo', 100)])
def test_call_sequences_through_rollout_and_step(level, n):
    """One pool through rollouts of T in {1, 7, 40, 43, 64, 129}, per-step calls in between and seed() + reset() with fresh
    seeds partway: persistent launches, graph launches, fused top-ups and sync points in every order."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    seeds = np.arange(n, dtype=np.uint64) + 555
    env, ref = BabyAIVecEnv(level, n, seeds=seeds), orc.OraclePool(level, n, seeds)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    rng = np.random.RandomState(13)
    plan = [1, 7, 40, 's', 43, 40, 64, 's', 's', 129, 40, 'seed', 64, 1, 40, 43, 's', 7, 129, 40, 40]
    for k, item in enumerate(plan):
        if item == 's':
            _step_vs(env, ref, rng.randint(0, 7, n).astype(np.int8), (level, k, 'step'))
        elif item == 'seed':
            fresh = np.arange(n, dtype=np.uint64) * 7 + 10 ** 9
            env.seed(fresh)
            ref = orc.OraclePool(level, n, fresh)
            assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
        else:
            _rollout_vs(env, ref, rng.randint(0, 7, (item, n)).astype(np.int8), (level, k, item))
        if k % 5 == 4:
            _missions_vs(env, ref, (level, k), range(n))
    assert env.counters()['errors'] == 0


@pytest.mark.timeout(120)
@pytest.mark.parametrize('level', ['PickupLoc', 'GoToObjMazeS4R2'])
@pytest.mark.parametrize('n', [1, 15, 16, 17, 31, 32, 33, 63, 64, 65])
def test_sizes_around_cta_widths(level, n):
    """Pool sizes around the CTA widths (k_rollout 64 envs, k_rollout_cta 32, k_step8 16 = 4 warps of 4 envs) through
    rollout and step."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    seeds = np.arange(n, dtype=np.uint64) * 5 + 77
    env, ref = BabyAIVecEnv(level, n, seeds=seeds), orc.OraclePool(level, n, seeds)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    rng = np.random.RandomState(n)
    eps = 0
    for k in range(4):
        eps += _rollout_vs(env, ref, rng.randint(0, 7, (40, n)).astype(np.int8), (level, n, k))
        for s in range(20):
            eps += _step_vs(env, ref, rng.randint(0, 7, n).astype(np.int8), (level, n, k, s))
    _missions_vs(env, ref, (level, n), range(n))
    c = env.counters()
    assert c['errors'] == 0 and c['steps'] == n * 240 and c['episodes'] == eps


# ---- 5. the bonus levels at scale, distinct seeds, against the host build ------------------------------------------------
@pytest.mark.timeout(180)
@pytest.mark.parametrize('variant', ['autoreset', 'freeze', 'other_kernel'])
@pytest.mark.parametrize('name', BONUS_GOLDENS)
def test_bonus_level_rollout_matches_host_build(name, variant, monkeypatch):
    """512 envs with distinct seeds x 160 steps through bb_pool_rollout (autoreset, freeze mode, and autoreset with the
    persistent kernel the level does not use by default: BB_ROLLOUT_KERNEL) against hostemu.HostEmuPool, the host build of
    the kernels' per-env source that test_bonus_levels.py pins to the reference step by step.  Both sides compile
    env_logic.cuh, so this catches what is GPU-side only -- staging, barriers, swap-ins, the ring supply, the output stores --
    but not a logic error in the shared source; the reference traces (bonus_*, replayed above) catch those, for the 16 seeds
    they hold."""
    import hostemu
    from babyai_b200 import BabyAIVecEnv
    from babyai_b200.levels import detokenize, level_spec
    level = golden_level(name)
    if variant == 'other_kernel':
        monkeypatch.setenv('BB_ROLLOUT_KERNEL', 'cta' if _single_room(level) else 'lane')
    mode = 1 if variant == 'freeze' else 0
    n = 512
    seeds = np.arange(n, dtype=np.uint64) * 3 + 424242
    env, ref = BabyAIVecEnv(level, n, seeds=seeds, mode=mode), hostemu.HostEmuPool(level_spec(level), n, seeds, mode)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    rng = np.random.RandomState(17)
    p = [0.12, 0.12, 0.3, 0.14, 0.14, 0.14, 0.04]             # pickups, drops and toggles
    for k in range(4):
        _rollout_vs(env, ref, rng.choice(7, size=(40, n), p=p).astype(np.int8), (level, variant, k), autoreset=None)
        idx = list(range(0, n, 9)) + [n - 1]
        assert env.missions(idx) == [detokenize(ref.tokens(i)) for i in idx], (level, variant, k)
    assert env.counters()['errors'] == 0


# ---- 6. the tuning knobs that select other kernels or other supply schedules ---------------------------------------------
KNOBS = [('BB_ROLLOUT_KERNEL', 'cta'), ('BB_ROLLOUT_KERNEL', 'lane'), ('BB_ROLLOUT_SPEC', '0'), ('BB_GEN_CONCURRENT', '0'),
         ('BB_GEN_CONCURRENT', '1'), ('BB_GEN_CHAIN_CAP', '4'), ('BB_GEN_PERIOD', '16'), ('BB_STEP_KERNEL', 'cols'),
         ('BB_NO_PERSISTENT', '1'), ('BB_GEN_GENERIC', '1'), ('BB_GEN_LANES', '32'), ('BB_GEN_BLOCKS_PER_SM', '2'),
         ('BB_GEN_BESIDE_BLOCKS_PER_SM', '2'), ('BB_GEN_FUSED', '2')]


@pytest.mark.timeout(240)
@pytest.mark.parametrize('level', ['PickupLoc', 'GoTo'])
@pytest.mark.parametrize('knob,value', KNOBS)
def test_knob_matrix(monkeypatch, knob, value, level):
    """Each data-path knob of DESIGN section 4.5 at a non-default value: rollouts of three lengths, then per-step calls, then
    rollouts again, against the oracle."""
    import oracle as orc
    from babyai_b200 import BabyAIVecEnv
    monkeypatch.setenv(knob, value)
    n = 333
    seeds = np.arange(n, dtype=np.uint64) + 2024
    env, ref = BabyAIVecEnv(level, n, seeds=seeds), orc.OraclePool(level, n, seeds)
    assert np.array_equal(env.reset().cpu().numpy(), ref.reset())
    rng = np.random.RandomState(3)
    eps = 0
    for k, T in enumerate([40, 40, 17, 40, 64, 40]):
        eps += _rollout_vs(env, ref, rng.randint(0, 7, (T, n)).astype(np.int8), (knob, value, level, k))
        if k == 2:
            for s in range(45):
                eps += _step_vs(env, ref, rng.randint(0, 7, n).astype(np.int8), (knob, value, level, 'step', s))
    _missions_vs(env, ref, (knob, value, level), range(n))
    c = env.counters()
    assert c['errors'] == 0 and c['episodes'] == eps and eps > 0
