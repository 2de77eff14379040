"""Shared helpers for the parity tests: replay a golden trace / a random action
stream through any pool-like object (oracle, host emulation, CUDA pool)."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CONFIG_LEVELS = ['GoToRedBall', 'GoToLocal', 'PickupLoc', 'GoTo', 'BossLevel']
GOLDEN_LEVELS = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith('.npz') and not f.startswith(('succ_', 'rgb_', 'done_', 'bonus_')))      # all 47 served levels (CPU replays)
# success-heavy reference traces (97 % bot actions, >= 50 successful episodes each; make_golden.py --success): 'succ_<Level>'
# reference traces generated with BABYAI_DONE_ACTIONS=1 (verifier.use_done_actions; make_golden.py --done-actions): 'done_<Level>'
DONE_GOLDENS = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith('.npz') and f.startswith('done_'))
# reference traces of the 50 bonus levels (babyai/levels/bonus_levels.py; make_golden.py --bonus): 'bonus_<Level>'
BONUS_GOLDENS = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith('.npz') and f.startswith('bonus_'))
SUCCESS_GOLDENS = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith('.npz') and f.startswith('succ_'))
# the traces test_gpu_parity.py replays through the per-step API; test_zz_gpu_widening.py replays the rest of GOLDEN_LEVELS,
# and test_gpu_rollout_parity.py replays every file (this list included) through bb_pool_rollout and bb_pool_step at scale
GOLDEN_LEVELS_GPU = ['BossLevel', 'BossLevelNoUnlock', 'GoTo', 'GoToLocal', 'GoToObjMazeS4R2', 'GoToOpen', 'GoToRedBall',
                     'GoToRedBallGrey', 'GoToSeq', 'MiniBossLevel', 'Open', 'Pickup', 'PickupLoc', 'PutNext', 'PutNextLocal',
                     'PutNextLocalS5N3', 'Synth', 'SynthSeq', 'UnblockPickup']


def load_golden(level):
    z = np.load(os.path.join(GOLDEN, level + '.npz'))
    d = {k: z[k] for k in z.files}
    d['missions'] = json.loads(str(d['missions']))
    return d


def golden_level(name):
    """the level a golden file was generated on: 'done_bonus_KeyCorridorS3R3' -> 'KeyCorridorS3R3'"""
    for prefix in ('succ_', 'done_', 'bonus_'):
        if name.startswith(prefix):
            name = name[len(prefix):]
    return name


def replay_golden(level, make_pool, get_mission):
    """make_pool(level, n, seeds) -> object with reset() -> obs[n,7,7,3], step(a) -> (obs, reward, done),
    .direction; get_mission(pool, i) -> str.  All K traces are run as ONE pool of K envs."""
    g = load_golden(level)
    level = golden_level(level)
    K, T = g['actions'].shape
    pool = make_pool(level, K, g['seeds'])
    obs = np.asarray(pool.reset())
    assert np.array_equal(obs.reshape(K, -1), g['obs0']), (level, 'reset obs')
    assert np.array_equal(np.asarray(pool.direction), g['dir0'])
    ep = [0] * K
    for i in range(K):
        assert get_mission(pool, i) == g['missions'][i][0]
    for t in range(T):
        obs, rew, done = pool.step(g['actions'][:, t])
        obs, rew, done = np.asarray(obs), np.asarray(rew), np.asarray(done)
        assert np.array_equal(done.astype(bool), g['done'][:, t].astype(bool)), (level, t, 'done')
        assert np.array_equal(rew.astype(np.float32).view(np.uint32), g['reward'][:, t].view(np.uint32)), (level, t, 'reward', rew, g['reward'][:, t])
        bad = np.nonzero((obs.reshape(K, -1) != g['obs'][:, t]).any(1))[0]
        assert len(bad) == 0, (level, t, 'obs differs for traces', bad)
        assert np.array_equal(np.asarray(pool.direction), g['direction'][:, t]), (level, t, 'direction')
        for i in np.nonzero(done)[0]:
            ep[i] += 1
            assert get_mission(pool, i) == g['missions'][i][ep[i]], (level, t, i)
    return int(g['done'].sum())


# rollout lengths for replay_golden_rollout, repeated up to the trace length: T = 64 takes the CUDA-graph path on
# single-room levels (persistent needs D >= 3T at D = 128), a change of T restarts the refill schedule and tops the rings up
ROLLOUT_SCHEDULE = (40, 40, 17, 1, 64, 40, 13)


def golden_assignment(K, n, seed=0):
    """env j of a replicated replay runs trace a[j]: every trace at least once, the rest drawn at random"""
    rng = np.random.RandomState(seed)
    a = np.concatenate([np.arange(K), rng.randint(0, K, n - K)])
    rng.shuffle(a)
    return a


def _first_mismatch(got, want):
    """(step within the chunk, env) of the first difference of two [T, n, ...] tensors"""
    bad = (got != want).reshape(got.shape[0], got.shape[1], -1).any(-1).nonzero()
    return tuple(int(x) for x in bad[0])


def replay_golden_rollout(name, n_envs, schedule=ROLLOUT_SCHEDULE, per_step=False, sample=64):
    """A golden file replicated over n_envs envs of one CUDA pool: env j replays trace a[j] (golden_assignment), with that
    trace's seed and actions; same-seed replicas are independent envs, so each must reproduce its trace exactly.  The pool is
    stepped through bb_pool_rollout in chunks of the lengths in `schedule` (per_step=True: through bb_pool_step, one call
    per step) and every chunk is compared on the device with the golden data gathered by a: observation bytes, reward bit
    patterns, done, direction.  At every chunk boundary the missions of a sample of envs must be those of the episode each
    env is in; at the end the counters must add up.  Returns the number of episode ends."""
    import torch
    from babyai_b200 import BabyAIVecEnv
    g = load_golden(name)
    K, T = g['actions'].shape
    n = n_envs
    a = golden_assignment(K, n)
    env = BabyAIVecEnv(golden_level(name), n, seeds=g['seeds'][a])
    dev = env.device
    idx = torch.as_tensor(a, device=dev)
    gobs = torch.as_tensor(g['obs'], device=dev)                            # [K, T, 147]
    grew = torch.as_tensor(g['reward'].view(np.int32), device=dev)
    gdone = torch.as_tensor(g['done'], device=dev)
    gdir = torch.as_tensor(g['direction'], device=dev)
    acts = torch.as_tensor(np.ascontiguousarray(g['actions'][a].T), device=dev)     # [T, n]
    rng = np.random.RandomState(1)
    probe = np.unique(np.r_[0, n - 1, rng.randint(0, n, sample)])
    obs0 = env.reset().reshape(n, -1)
    want0 = torch.as_tensor(g['obs0'], device=dev)[idx]
    assert torch.equal(obs0, want0), (name, 'reset obs', _first_mismatch(obs0[None], want0[None]))
    assert np.array_equal(env.direction.cpu().numpy(), g['dir0'][a]), (name, 'reset direction')
    assert env.missions(probe) == [g['missions'][a[j]][0] for j in probe], (name, 'reset missions')
    Tmax = max(schedule)
    obs = torch.zeros((Tmax, n, 7, 7, 3), dtype=torch.uint8, device=dev)
    rew = torch.zeros((Tmax, n), dtype=torch.float32, device=dev)
    done = torch.zeros((Tmax, n), dtype=torch.uint8, device=dev)
    dirs = torch.zeros((Tmax, n), dtype=torch.int8, device=dev)
    episodes = torch.zeros(n, dtype=torch.int64, device=dev)
    t0, k = 0, 0
    while t0 < T:
        Tc = min(schedule[k % len(schedule)], T - t0)
        k += 1
        if per_step:
            for t in range(Tc):
                env.step(acts[t0 + t], obs[t], rew[t], done[t], dirs[t])
        else:
            env.rollout(acts[t0:t0 + Tc], obs[:Tc], rew[:Tc], done[:Tc], dirs[:Tc])
        got = [obs[:Tc].reshape(Tc, n, -1), rew[:Tc].view(torch.int32), done[:Tc], dirs[:Tc]]
        want = [x[:, t0:t0 + Tc][idx].transpose(0, 1) for x in (gobs, grew, gdone, gdir)]
        for what, x, y in zip(('obs', 'reward', 'done', 'direction'), got, want):
            if not torch.equal(x, y):
                t, j = _first_mismatch(x, y)
                raise AssertionError('%s: %s differs at step %d, env %d (trace %d)' % (name, what, t0 + t, j, a[j]))
        episodes += done[:Tc].sum(0)
        t0 += Tc
        ep = episodes.cpu().numpy()
        got_m = env.missions(probe)
        want_m = [g['missions'][a[j]][ep[j]] for j in probe]
        assert got_m == want_m, (name, 'missions after step', t0, [(j, x, y) for j, x, y in zip(probe, got_m, want_m) if x != y][:4])
    c = env.counters()
    want_c = dict(steps=n * T, episodes=int(g['done'][a].sum()), successes=int((g['reward'][a] > 0).sum()), errors=0)
    assert c == want_c, (name, c, want_c)
    env.close()
    return want_c['episodes']


def compare_pools(a, b, n, steps, act_seed=0, mission_a=None, mission_b=None, state=True, check_draws=False, action_p=None):
    """Drive two pools with the same random actions (uniform, or distribution action_p); everything must be identical."""
    rng = np.random.RandomState(act_seed)
    oa, ob = np.asarray(a.reset()).copy(), np.asarray(b.reset()).copy()
    assert np.array_equal(oa, ob), 'reset obs'
    episodes = 0
    for t in range(steps):
        act = (rng.randint(0, 7, n) if action_p is None else rng.choice(7, size=n, p=action_p)).astype(np.int8)
        oa, ra, da = [np.asarray(x).copy() for x in a.step(act)]
        ob, rb, db = [np.asarray(x).copy() for x in b.step(act)]
        assert np.array_equal(da.astype(bool), db.astype(bool)), (t, 'done')
        assert np.array_equal(ra.view(np.uint32), rb.view(np.uint32)), (t, 'reward')
        bad = np.nonzero((oa != ob).reshape(n, -1).any(1))[0]
        assert len(bad) == 0, (t, 'obs', bad)
        assert np.array_equal(np.asarray(a.direction), np.asarray(b.direction)), (t, 'direction')
        episodes += int(da.astype(bool).sum())
        if state and (t % 7 == 0 or t == steps - 1):
            for i in range(n):
                g0, i0 = a.state(i)
                g1, i1 = b.state(i)
                assert np.array_equal(g0, g1), (t, i, 'grid')
                if not check_draws:
                    for k in ('draws', 'attempts'):
                        i0.pop(k), i1.pop(k)
                assert i0 == i1, (t, i, i0, i1)
                if mission_a is not None:
                    assert mission_a(a, i) == mission_b(b, i), (t, i)
    return episodes
