"""Shared pieces of the selected-step tests (test_step_envs.py, test_gpu_step_envs.py): a mirror with one single-env pool per
env -- the oracle for the ICLR levels, the host build of the kernel logic for the bonus levels -- where only the listed envs
step, and where a fork replays the source's history on a fresh single-env pool."""
import numpy as np

from babyai_b200.levels import BONUS_LEVELS, detokenize, level_spec
from reset_envs_common import AUTORESET, FREEZE, OracleMirror, compare_rows  # noqa: F401


class _HostOne(object):
    """the host build of one env, with the single-env oracle pool's interface"""

    def __init__(self, level, seed, mode):
        import reset_envs_host
        self.p = reset_envs_host.ResetHostPool(level_spec(level), 1, np.array([seed], np.uint64), mode)

    @property
    def obs(self):
        return self.p.obs

    @property
    def direction(self):
        return self.p.direction

    def reset(self):
        self.p.reset()

    def step(self, a, autoreset=True):
        o, r, d = self.p.step(np.asarray(a, np.int8))
        return o, r, d

    def mission(self, i):
        return detokenize(self.p.tokens(i))

    def state(self, i):
        return self.p.state(i)


class SelMirror(OracleMirror):
    """OracleMirror (bonus levels: the host build) that also steps and forks the envs of an id list.  Every mirrored env keeps
    its history -- (seed or None) for a reset, an action for a step -- so that a fork is rebuilt exactly: a fresh single-env
    pool of the source's seed that replays the source's history."""

    def __init__(self, level, seeds, mode, ids=None):
        self.level, self.freeze = level, mode == FREEZE
        self.mode = mode
        self.ids = np.arange(len(seeds)) if ids is None else np.asarray(ids)
        self.seed0 = {int(i): int(seeds[i]) for i in self.ids}
        if level not in BONUS_LEVELS:
            import oracle as orc
            self.orc = orc
        self.envs = {i: self._fresh(s) for i, s in self.seed0.items()}
        self.hist = {i: [] for i in self.envs}
        self.last = {}
        self.frozen = set()

    def _fresh(self, seed):
        if self.level in BONUS_LEVELS:
            return _HostOne(self.level, seed, self.mode)
        return self.orc.OraclePool(self.level, 1, np.array([seed], np.uint64))

    def _step_one(self, i, a):
        if i in self.frozen:
            return self.last[i][:2] + [np.uint8(1)] + self.last[i][3:]
        o = self.envs[i]
        ob, r, d = o.step(np.array([a], np.int8), autoreset=not self.freeze)
        self.hist[i].append(int(a))
        if self.freeze and d[0]:
            self.frozen.add(i)
        return [ob[0].copy(), np.float32(r[0]), np.uint8(d[0]), np.int8(o.direction[0])]

    def reset(self):
        for i in self.envs:
            self.envs[i].reset()
            self.hist[i] = [None]
            self.last[i] = self._one(i)
        self.frozen.clear()

    def step(self, actions):
        out = {i: self._step_one(i, actions[i]) for i in self.envs}
        self.last.update(out)
        return out

    def step_envs(self, ids, actions):
        """action k for env ids[k], the mirrored ones among them -> {env: [obs, reward, done, direction]}"""
        out = {}
        for k, i in enumerate(ids):
            i = int(i)
            if i in self.envs:
                out[i] = self._step_one(i, actions[k])
        self.last.update(out)
        return out

    def reset_envs(self, ids, seeds=None):
        for k, i in enumerate(ids):
            i = int(i)
            if i not in self.envs:
                continue
            if seeds is not None:
                self.seed0[i] = int(seeds[k])
                self.envs[i] = self._fresh(self.seed0[i])
                self.hist[i] = []
            self.envs[i].reset()
            self.hist[i].append(None)
            self.last[i] = self._one(i)
            self.frozen.discard(i)

    def save(self, ids):
        """what a record of each env holds: {env: (seed, history, frozen, last outputs)}"""
        return {int(i): (self.seed0[int(i)], list(self.hist[int(i)]), int(i) in self.frozen, list(self.last[int(i)])) for i in ids}

    def load(self, snap, ids, srcs=None):
        """env ids[k] := the saved env srcs[k] (default: ids[k] itself), rebuilt on a fresh single-env pool"""
        for k, d in enumerate(ids):
            seed, hist, frozen, last = snap[int(d if srcs is None else srcs[k])]
            d = int(d)
            e = self._fresh(seed)
            for ev in hist:
                if ev is None:
                    e.reset()
                else:
                    e.step(np.array([ev], np.int8), autoreset=not self.freeze)
            self.envs[d], self.seed0[d], self.hist[d], self.last[d] = e, seed, list(hist), list(last)
            if frozen:
                self.frozen.add(d)
            else:
                self.frozen.discard(d)

    def copy_envs(self, src, dst):
        """env dst[k] := env src[k] as it is now (both mirrored); sources are read before any destination is written"""
        self.load(self.save(src), dst, src)
