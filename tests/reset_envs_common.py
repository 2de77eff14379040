"""Shared pieces of the per-env reset tests (test_reset_envs.py, test_gpu_reset_envs.py): what a pool must do when some of
its envs start a new episode, run on the oracle (one single-env oracle pool per env, so that each env can be reseeded and
reset on its own) and on the host build (tests/hostemu/reset_envs_host.py), and a policy that is a pure function of each
env's observation, direction and mission."""
import re

import numpy as np

from babyai_b200.levels import BONUS_LEVELS, VOCAB, level_spec

AUTORESET, FREEZE = 0, 1
# one bonus level per generator kind (bonus_levels.py: bb_level_spec::bonus 1..20)
BONUS_PER_KIND = ['GoToRedBlueBall', 'OpenRedDoor', 'OpenDoor', 'GoToDoor', 'GoToObjDoor', 'ActionObjDoor', 'UnlockLocal',
                  'KeyInBox', 'UnlockPickup', 'BlockedUnlockPickup', 'UnlockToUnlock', 'PickupDist', 'PickupAbove',
                  'OpenTwoDoors', 'FindObjS5', 'KeyCorridorS3R1', '1RoomS8', 'PutNextS4N1', 'MoveTwoAcrossS5N2', 'OpenDoorsOrderN2']
_WORD = {w: i for i, w in enumerate(VOCAB) if i > 0}


def mission_code(mission):
    """the sum of the mission's token ids (what the pool's token row sums to)"""
    return sum(_WORD[w] for w in re.findall('[a-z]+', mission.lower()))


def policy(image_sum, direction, code):
    """the action of an env: a pure function of its observation (byte sum), direction and mission (token-id sum)"""
    return (np.asarray(image_sum, np.int64) * 31 + np.asarray(direction, np.int64) * 7 + np.asarray(code, np.int64) * 3) % 7


class PolicyAgent(object):
    """`act_batch` / `analyze_feedback` over the reference's obs dicts, an ObsBatch of the pool, or a list of ObsRefs"""

    def act_batch(self, many_obs):
        import torch
        if hasattr(many_obs, 'image') and hasattr(many_obs, 'tokens'):          # learner.ObsBatch: on the device
            img = many_obs.image.reshape(len(many_obs), -1).to(torch.int64).sum(1)
            a = (img * 31 + many_obs.direction.to(torch.int64) * 7 + many_obs.tokens.to(torch.int64).sum(1) * 3) % 7
            return {'action': a}
        a = [int(policy(np.asarray(o['image']).astype(np.int64).sum(), o['direction'], mission_code(o['mission']))) for o in many_obs]
        return {'action': torch.tensor(a)}

    def analyze_feedback(self, reward, done):
        pass


class OracleMirror(object):
    """The oracle for the envs `ids` of a pool: one single-env oracle pool per env.  Freeze mode: an env that has ended
    repeats its last observation, reward and direction with done = 1 until it is reset."""

    def __init__(self, level, seeds, mode, ids=None):
        import oracle as orc
        self.orc, self.level, self.freeze = orc, level, mode == FREEZE
        self.ids = np.arange(len(seeds)) if ids is None else np.asarray(ids)
        self.envs = {int(i): orc.OraclePool(level, 1, np.array([seeds[i]], np.uint64)) for i in self.ids}
        self.last = {}
        self.frozen = set()

    def _one(self, i):
        o = self.envs[i]
        return [o.obs[0].copy(), np.float32(0), np.uint8(0), np.int8(o.direction[0])]

    def reset(self):
        for i in self.envs:
            self.envs[i].reset()
            self.last[i] = self._one(i)
        self.frozen.clear()

    def step(self, actions):
        """actions for every env of the pool -> {env: [obs, reward, done, direction]}"""
        out = {}
        for i, o in self.envs.items():
            if i in self.frozen:
                out[i] = self.last[i][:2] + [np.uint8(1)] + self.last[i][3:]
                continue
            ob, r, d = o.step(np.array([actions[i]], np.int8), autoreset=not self.freeze)
            out[i] = [ob[0].copy(), np.float32(r[0]), np.uint8(d[0]), np.int8(o.direction[0])]
            if self.freeze and d[0]:
                self.frozen.add(i)
        self.last.update(out)
        return out

    def reset_envs(self, ids, seeds=None):
        """env.seed(seeds[k]) (a freshly made env) then env.reset(), for the mirrored envs among ids"""
        for k, i in enumerate(ids):
            i = int(i)
            if i not in self.envs:
                continue
            if seeds is not None:
                self.envs[i] = self.orc.OraclePool(self.level, 1, np.array([seeds[k]], np.uint64))
            self.envs[i].reset()
            self.last[i] = self._one(i)
            self.frozen.discard(i)

    def mission(self, i):
        return self.envs[int(i)].mission(0)

    def state(self, i):
        return self.envs[int(i)].state(0)


class HostMirror(object):
    """The same interface over the host build of the kernel logic (every env of the pool)"""

    def __init__(self, level, seeds, mode, ids=None):
        import reset_envs_host
        from babyai_b200.levels import detokenize
        self.detok = detokenize
        self.pool = reset_envs_host.ResetHostPool(level_spec(level), len(seeds), np.asarray(seeds, np.uint64), mode)
        self.ids = np.arange(len(seeds)) if ids is None else np.asarray(ids)
        self.last = {}

    def _rows(self, ids, rew=None, done=None):
        p = self.pool
        return {int(i): [p.obs[i].copy(), np.float32(0 if rew is None else rew[i]), np.uint8(0 if done is None else done[i]),
                         np.int8(p.direction[i])] for i in ids}

    def reset(self):
        self.pool.reset()
        self.last = self._rows(self.ids)

    def step(self, actions):
        _, r, d = self.pool.step(np.asarray(actions, np.int8))
        out = self._rows(self.ids, r, d)
        self.last.update(out)
        return out

    def reset_envs(self, ids, seeds=None):
        self.pool.reset_envs(ids, seeds)
        self.last.update(self._rows([i for i in ids if i in set(self.ids.tolist())]))

    def mission(self, i):
        return self.detok(self.pool.tokens(int(i)))

    def state(self, i):
        return self.pool.state(int(i))


def mirror_for(level, seeds, mode, ids=None):
    """the oracle for the ICLR levels, the host build for the bonus levels"""
    return (HostMirror if level in BONUS_LEVELS else OracleMirror)(level, seeds, mode, ids)


def compare_rows(got, want, what):
    """got: (obs [n, 7, 7, 3], reward [n] or None, done [n] or None, direction [n]) numpy; want: {env: [obs, r, d, dir]}"""
    obs, rew, done, dire = got
    for i, w in want.items():
        assert np.array_equal(obs[i].reshape(-1), w[0].reshape(-1)), (what, 'obs', i)
        if rew is not None:
            assert np.float32(rew[i]).view(np.uint32) == np.float32(w[1]).view(np.uint32), (what, 'reward', i, rew[i], w[1])
            assert bool(done[i]) == bool(w[2]), (what, 'done', i)
        assert int(dire[i]) == int(w[3]), (what, 'direction', i)
