"""Per-env reset and reseed (bb_pool_reset_envs) without a GPU:
- the host build's and the oracle's per-env reset against the reference's unmodified level classes on the shim: a reseed is a
  freshly made reference env with that seed, a reset without a seed is `env.reset()` mid-episode on the same reference env;
- k_reset8's role (csrc/reset8.cuh, one OS thread per lane) and the selected passes around it against the host build, on
  every level family, ragged id lists and the untracked-carry instantiation included;
- the reference's unmodified `batch_evaluate` and babyai_b200.evaluate.batch_evaluate over the host build: equal logs;
- the built library: the new kernels use no local memory."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import reset_envs_host
from babyai_b200.levels import detokenize, level_spec
from reset_envs_common import AUTORESET, BONUS_PER_KIND, FREEZE, OracleMirror, PolicyAgent

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


# ------------------------------------------------------------------------------------------------------------------------
# the host build and the oracle against the reference
# ------------------------------------------------------------------------------------------------------------------------
def _ref_obs(ob):
    return np.asarray(ob['image'], np.uint8).reshape(-1), int(ob['direction']), ob['mission']


def _check_against_reference(level, use_oracle):
    import refenv
    refenv.setup('philox')
    n, rng = 5, np.random.RandomState(3)
    seeds = [900 + 11 * i for i in range(n)]
    refs = [refenv.make_env(level, s) for s in seeds]
    want = [_ref_obs(e.reset()) for e in refs]
    if use_oracle:
        pool = OracleMirror(level, seeds, AUTORESET)
        pool.reset()
        got = lambda i: (pool.last[i][0].reshape(-1), int(pool.last[i][3]), pool.mission(i))
    else:
        pool = reset_envs_host.ResetHostPool(level_spec(level), n, np.asarray(seeds, np.uint64), AUTORESET)
        pool.reset()
        got = lambda i: (pool.obs[i].reshape(-1), int(pool.direction[i]), detokenize(pool.tokens(i)))
    for i in range(n):
        g = got(i)
        assert np.array_equal(g[0], want[i][0]) and g[1:] == want[i][1:], (level, 'reset', i)
    for rnd in range(3):
        for t in range(12):                                         # a few steps: mid-episode (auto-reset on both sides)
            a = rng.randint(0, 7, n).astype(np.int8)
            if use_oracle:
                out = pool.step(a)
            else:
                pool.step(a)
            for i, e in enumerate(refs):
                ob, _, d, _ = e.step(int(a[i]))
                if d:
                    ob = e.reset()
                g = got(i)
                assert np.array_equal(g[0], _ref_obs(ob)[0]), (level, rnd, t, i)
        # reseed two envs (a freshly made reference env), reset two others without a seed (env.reset() mid-episode)
        ids = rng.permutation(n)[:4]
        new = [10 ** 6 + 1000 * rnd + int(i) for i in ids[:2]]
        pool.reset_envs(ids[:2], new)
        pool.reset_envs(ids[2:])
        for i, s in zip(ids[:2], new):
            refs[i] = refenv.make_env(level, s)
        for i in ids:
            r = _ref_obs(refs[i].reset())
            g = got(int(i))
            assert np.array_equal(g[0], r[0]) and g[1:] == r[1:], (level, rnd, 'reset_envs', int(i))


@pytest.mark.reference
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc', 'GoTo', 'BossLevel', 'Unlock', 'GoToImpUnlock', 'SynthSeq'])
@pytest.mark.parametrize('impl', ['oracle', 'host'])
def test_iclr_reset_envs_equals_reference(level, impl):
    _check_against_reference(level, impl == 'oracle')


@pytest.mark.reference
@pytest.mark.parametrize('level', ['KeyCorridorS3R1', 'PutNextS6N3Carrying', 'OpenDoorsOrderN4', 'UnlockToUnlock', 'GoToObjDoor'])
def test_bonus_reset_envs_equals_reference(level):
    _check_against_reference(level, False)


# ------------------------------------------------------------------------------------------------------------------------
# k_reset8's role against the host build
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = ['GoToRedBall', 'GoToLocal', 'PutNextLocal', 'PickupLoc', 'GoTo', 'BossLevel', 'Unlock', 'GoToImpUnlock',
            'KeyCorridorS3R1', 'PutNextS4N1', 'OpenDoorsOrderN2', 'UnlockPickup']


def _same_state(simt, host, i, level):
    sg, si = simt.state(i, host.width, host.height)
    hg, hi = host.state(i)
    assert np.array_equal(sg, hg), (level, i, 'grid')
    assert list(si[:6]) == [hi[k] for k in ('agent_x', 'agent_y', 'agent_dir', 'carrying', 'step_count', 'max_steps')], (level, i)
    t = simt.tokens(i)
    assert np.array_equal(t, host.tokens(i)[:len(t)]), (level, i, 'tokens')


@pytest.mark.parametrize('level', FAMILIES)
@pytest.mark.parametrize('mode', [AUTORESET, FREEZE])
def test_reset_role_equals_host_build(level, mode):
    n = 37                                                     # 3 CTAs of 16 envs, the last one ragged
    rng = np.random.RandomState(len(level) + mode)
    seeds = np.arange(n, dtype=np.uint64) + 500
    spec = level_spec(level)
    simt = reset_envs_host.SimtResetPool(spec, n, seeds, depth=6, mode=mode)
    host = reset_envs_host.ResetHostPool(spec, n, seeds, mode)
    host.reset()
    for rnd in range(4):
        for t in range(6):
            a = rng.randint(0, 7, n).astype(np.int8)
            so, sr, sd, sq, cnt = simt.step8(a)
            ho, hr, hd = host.step(a)
            assert np.array_equal(so, ho) and np.array_equal(sr.view(np.uint32), hr.view(np.uint32)), (level, rnd, t)
            assert np.array_equal(sd.astype(bool), hd.astype(bool)) and np.array_equal(sq, host.direction), (level, rnd, t)
        k = [1, 5, 17, n][rnd]                                 # ragged lists, the last one every env
        ids = rng.permutation(n)[:k].astype(np.int32)
        seeds_k = rng.randint(0, 2 ** 62, k).astype(np.uint64) * 3 if rnd % 2 == 0 else None
        obs = np.full((n, 7, 7, 3), 0xA5, np.uint8)
        dirs = np.full(n, -7, np.int8)
        obs, dirs, cnt = simt.reset_envs(ids, seeds_k, obs, dirs)
        host.reset_envs(ids, seeds_k)
        assert cnt[3] == 0 and simt.error_flag() == 0, (level, rnd)
        listed = np.zeros(n, bool)
        listed[ids] = True
        assert np.array_equal(obs[listed], host.obs[listed]) and np.array_equal(dirs[listed], host.direction[listed]), (level, rnd)
        assert (obs[~listed] == 0xA5).all() and (dirs[~listed] == -7).all(), (level, rnd, 'unlisted rows written')
        for i in range(n):
            _same_state(simt, host, i, level)
    # the listed envs were frozen or not: every env steps on after its reset
    a = rng.randint(0, 7, n).astype(np.int8)
    so, _, sd, _, _ = simt.step8(a)
    ho, _, hd = host.step(a)
    assert np.array_equal(so, ho) and np.array_equal(sd.astype(bool), hd.astype(bool))


# ------------------------------------------------------------------------------------------------------------------------
# the streaming evaluator against the reference's batch_evaluate
# ------------------------------------------------------------------------------------------------------------------------
class EmuResetTensorPool(object):
    """BabyAIVecEnv's tensor interface (what DeviceManyEnvs and vecenv.ManyEnvs use, reset_envs included) over the host
    build, CPU tensors standing in for HBM"""

    def __init__(self, level, seeds, mode=FREEZE):
        import torch
        n = len(seeds)
        self.emu = reset_envs_host.ResetHostPool(level_spec(level), n, np.asarray(seeds, dtype=np.uint64), mode)
        self.num_envs, self.device = n, torch.device('cpu')
        self.mission_tokens = torch.zeros((n, 72), dtype=torch.int16)
        self.direction = torch.zeros(n, dtype=torch.int8)

    def _tokens(self, idx):
        import torch
        for i in idx:
            self.mission_tokens[i] = torch.from_numpy(self.emu.tokens(int(i)))

    def seed(self, seeds):
        self.emu.seed(np.asarray(list(seeds), dtype=np.uint64))

    def reset(self, obs=None, direction=None):
        import torch
        obs.copy_(torch.from_numpy(self.emu.reset()))
        self.direction.copy_(torch.from_numpy(self.emu.direction))
        self._tokens(range(self.num_envs))
        return obs

    def step_learner(self, actions, obs, reward, done, direction=None):
        import torch
        o, r, d = self.emu.step(np.asarray(actions, np.int8))
        obs.copy_(torch.from_numpy(o))
        reward[...], done[...] = r, d
        self.direction.copy_(torch.from_numpy(self.emu.direction))
        if direction is not None:
            direction.copy_(self.direction)
        self._tokens(np.nonzero(d)[0])

    def reset_envs(self, env_ids, seeds=None, obs=None, direction=None):
        import torch
        ids = np.asarray(env_ids, np.int32)
        self.emu.reset_envs(ids, None if seeds is None else np.asarray(seeds, np.uint64))
        t = torch.as_tensor(ids.astype(np.int64))
        obs[t] = torch.from_numpy(self.emu.obs[ids])
        self.direction[t] = torch.from_numpy(self.emu.direction[ids])
        if direction is not None:
            direction[t] = self.direction[t]
        self._tokens(ids)
        return obs

    # host-buffer interface (vecenv.ManyEnvs)
    def reset_host(self, obs, direction):
        obs[...] = self.emu.reset()
        direction[...] = self.emu.direction

    def step_host(self, actions, obs, reward, done, direction):
        o, r, d = self.emu.step(np.asarray(actions, dtype=np.int8))
        obs[...], reward[...], done[...], direction[...] = o, r, d, self.emu.direction

    def missions(self, idx=None):
        return [detokenize(self.emu.tokens(int(i))) for i in (range(self.num_envs) if idx is None else idx)]


@pytest.mark.reference
@pytest.mark.timeout(600)
@pytest.mark.parametrize('level', ['GoToLocal', 'PickupLoc', 'BossLevel'])
def test_reference_batch_evaluate_equals_streaming_evaluator(level):
    """the reference's wave loop over 24 envs (one wave) and the streaming loop over 7 envs (24 seeds through 7 slots, resets
    at every step) on the host build: equal logs in seed order, with and without observations / actions"""
    import refenv
    refenv.setup('philox')
    import babyai.evaluate as evaluate
    from babyai_b200 import ManyEnvs
    from babyai_b200 import evaluate as bev
    episodes, seed = 24, 10 ** 9 + 7
    stock = evaluate.ManyEnvs
    evaluate.ManyEnvs = lambda envs: ManyEnvs(envs, pool=EmuResetTensorPool(level, [0] * len(envs)))
    try:
        a = evaluate.batch_evaluate(PolicyAgent(), 'BabyAI-%s-v0' % level, seed, episodes, return_obss_actions=True)
    finally:
        evaluate.ManyEnvs = stock
    b = bev.batch_evaluate(PolicyAgent(), 'BabyAI-%s-v0' % level, seed, episodes, return_obss_actions=True, num_envs=7,
                           pool=EmuResetTensorPool(level, list(range(seed, seed + 7))))
    assert len(b['seed_per_episode']) == 28 and len(a['seed_per_episode']) == 24
    k = 24                                                     # the stream's seed set is ceil(24 / 7) * 7 = 28 seeds: the first 24 are the wave's
    assert list(b['seed_per_episode'][:k]) == list(a['seed_per_episode'])
    assert [int(x) for x in b['num_frames_per_episode'][:k]] == [int(x) for x in a['num_frames_per_episode']]
    assert [np.float32(x) for x in b['return_per_episode'][:k]] == [np.float32(x) for x in a['return_per_episode']]
    assert b['actions_per_episode'][:k] == a['actions_per_episode']
    for oa, ob in zip(a['observations_per_episode'], b['observations_per_episode'][:k]):
        assert len(oa) == len(ob)
        for x, y in zip(oa, ob):
            assert np.array_equal(np.asarray(x['image']), np.asarray(y['image'])) and x['mission'] == y['mission']
    assert max(int(x) for x in a['num_frames_per_episode']) > 1


# ------------------------------------------------------------------------------------------------------------------------
# the built library
# ------------------------------------------------------------------------------------------------------------------------
def test_new_kernels_use_no_local_memory():
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
    for name, count in (('k_seed_sel', 1), ('k_gen_scan_sel', 1), ('k_pub_sel', 1), ('k_reset8', 2)):
        found = {k: v for k, v in fns.items() if re.match(r'_Z\d+' + name + r'(I|\d)', k)}
        assert len(found) == count, (name, list(found))
        for k, code in found.items():
            assert not any(re.search(r'\b(LDL|STL)\b', i) for i in code), (k, 'local memory')
