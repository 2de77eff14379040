"""Device-resident consumer adapters (SURVEY.md 8f-1): what sits between the pool and the
reference's learner so that `BaseAlgo.collect_experiences` (rl/algos/base.py:110-232) and
`PPOAlgo.update_parameters` (rl/algos/ppo.py:34-160) run UNCHANGED while the observations
never leave HBM.

The reference moves every observation through the host three times per step: pickled out of
the worker (penv.py:11), `numpy.array([obs["image"] ...])` + a regex over the mission string
in `ObssPreprocessor.__call__` (utils/format.py:59-119), and `torch.tensor(...)` back to the
device.  Here

  DeviceParallelEnv   penv.py:18-59 surface (reset / step with auto-reset); `obs` is an
                      `ObsBatch`: a length-N sequence whose payload -- image uint8[N,7,7,3],
                      mission tokens int16[N,L], direction int8[N] -- are device tensors the
                      step kernel wrote.  Only reward / done (5 B per env) and the actions
                      (1 B per env) cross PCIe each step.
  ObssPreprocessor    utils/format.py:100-119 surface (`__call__(obss, device)`, `.vocab`,
                      `.obs_space`): `ObsBatch` -> image float[N,7,7,3], instr long[N,Lmax]
                      with two device ops; the flattened list `BaseAlgo` builds at the end of a
                      rollout (base.py:208-210: obss[i][j], env-major) -> one device gather.
  FixedVocabulary     utils/format.py:15-41 surface over the closed 32-word baby language
                      (levels.VOCAB); `save()` writes the `vocab.json` the reference reloads.
  ObsTensors          the (image, instr) pair the preprocessor returns, row-indexable; or the caller's `babyai.rl.DictList`.

Items of an `ObsBatch` are `ObsRef`s: `ref['image']` / `ref['mission']` / `ref['direction']`
materialise on the host on demand, so code that does look at single observations
(`reshape_reward`, the stock preprocessors) keeps working -- slowly, like the reference.
"""
import json
import os

import numpy as np
import torch

from .levels import VOCAB, detokenize
from .vecenv import MODE_AUTORESET, MODE_FREEZE, BabyAIVecEnv, _as_env_list, _spaces


class ObsTensors(object):
    """What `ObssPreprocessor.__call__` returns when no container class is given: the two model inputs, row-indexable
    together (`obs[rows].image`), which is all `ACModel.forward` (model.py) and `PPOAlgo.update_parameters`
    (ppo.py: `sb = exps[inds + i]`) ask of `babyai.rl.DictList`.  Pass `dictlist=babyai.rl.DictList` to get the reference's
    own type (INTEGRATION.md does)."""
    __slots__ = ('image', 'instr')

    def __init__(self, image=None, instr=None):
        self.image, self.instr = image, instr

    def __len__(self):
        return len(self.image)

    def __getitem__(self, index):
        return ObsTensors(self.image[index], self.instr[index])

    def __setitem__(self, index, other):
        self.image[index] = other.image
        self.instr[index] = other.instr


class FixedVocabulary(object):
    """Vocabulary (utils/format.py:15-41) whose ids are the pool's token ids; 0 pads."""

    def __init__(self, path=None):
        self.path = path
        self.max_size = 100                                # format.py:18; sizes the model's embedding
        self.vocab = {w: i for i, w in enumerate(VOCAB) if i > 0}

    def __getitem__(self, token):
        return self.vocab[token]                           # closed vocabulary: unknown words are an error

    def save(self, path=None):
        path = path or self.path
        if path is None:
            raise ValueError('FixedVocabulary.save() needs a path (the model directory\'s vocab.json)')
        d = os.path.dirname(path)
        if d:
            os.makedirs(d, exist_ok=True)
        with open(path, 'w') as f:
            json.dump(self.vocab, f)

    def copy_vocab_from(self, other):
        if any(self.vocab.get(k) != v for k, v in other.vocab.items()):
            raise ValueError('the other vocabulary does not use the pool\'s token ids')


_serial = [0]


class ObsBatch(object):
    """The N observations one reset() / step() produced, resident on the device."""
    __slots__ = ('image', 'tokens', 'direction', 'serial', '_host')

    def __init__(self, image, tokens, direction):
        self.image, self.tokens, self.direction = image, tokens, direction
        _serial[0] += 1
        self.serial = _serial[0]
        self._host = None

    def __len__(self):
        return self.image.shape[0]

    def __getitem__(self, j):
        if isinstance(j, slice):
            return [ObsRef(self, k) for k in range(*j.indices(len(self)))]
        if j < 0:
            j += len(self)
        if not 0 <= j < len(self):
            raise IndexError(j)
        return ObsRef(self, j)

    def __iter__(self):
        return (ObsRef(self, j) for j in range(len(self)))

    def host(self):
        """(image, tokens, direction) as numpy arrays; one device->host copy per batch, on first use."""
        if self._host is None:
            self._host = (self.image.cpu().numpy(), self.tokens.cpu().numpy(), self.direction.cpu().numpy())
        return self._host


class ObsRef(object):
    """Observation j of a batch; behaves like the reference's obs dict when somebody looks inside."""
    __slots__ = ('batch', 'j')

    def __init__(self, batch, j):
        self.batch, self.j = batch, j

    def __getitem__(self, key):
        img, tok, dire = self.batch.host()
        if key == 'image':
            return img[self.j]
        if key == 'mission':
            return detokenize(tok[self.j])
        if key == 'direction':
            return int(dire[self.j])
        raise KeyError(key)

    def keys(self):
        return ('image', 'direction', 'mission')

    def __iter__(self):
        return iter(self.keys())

    def __contains__(self, key):
        return key in self.keys()


class _Infos(object):
    """The per-env `info` dicts (always `{}` in BabyAI), made on demand: a tuple of N dicts per step would cost more
    host time than the step kernel at pool sizes."""
    __slots__ = ('n',)

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, j):
        if isinstance(j, slice):
            return [{} for _ in range(*j.indices(self.n))]
        if not -self.n <= j < self.n:
            raise IndexError(j)
        return {}

    def __iter__(self):
        return ({} for _ in range(self.n))


class DeviceParallelEnv(object):
    """babyai.rl.utils.penv.ParallelEnv surface; observations stay on the device.

    `envs` is the list `make_envs()` built (scripts/train_rl.py:53-60 shape).  `pool` is for tests only: an object
    with BabyAIVecEnv's tensor interface (the GPU-less suite passes the host build of the kernel logic).
    `fused_io` (default on; BB_LEARNER_FUSED_IO=0 switches it off) steps through bb_pool_step_learner -- actions, reward and
    done travel over mapped page-locked memory inside the one step call instead of as three separate tensor copies
    A list wrapped in RGBImgPartialObsWrapper (`make_envs(..., pixel=True)`) yields 56x56x3 pictures rendered on the device."""

    MODE = MODE_AUTORESET

    def __init__(self, envs, pool=None, fused_io=None):
        envs = _as_env_list(envs, need_seeds=(self.MODE == MODE_AUTORESET))
        self.envs = envs
        self.pixel = bool(getattr(envs, 'pixel', False))      # RGBImgPartialObsWrapper'd list: batches carry uint8[N, 56, 56, 3]
        self.observation_space, self.action_space = _spaces(self.pixel)
        self.pool = pool if pool is not None else BabyAIVecEnv(envs.level, len(envs), seeds=envs.seeds,
                                                               device=envs.device, mode=self.MODE)
        self._tokens = None
        if fused_io is None:
            fused_io = os.environ.get('BB_LEARNER_FUSED_IO', '1') != '0'
        self.fused_io = bool(fused_io) and hasattr(self.pool, 'step_learner')
        n = self.pool.num_envs
        self._rew_h, self._done_h = np.zeros(n, np.float32), np.zeros(n, np.uint8)

    def _batch(self, image, refresh_tokens):
        if refresh_tokens or self._tokens is None:         # missions change only when an episode starts
            self._tokens = self.pool.mission_tokens.clone()
        return ObsBatch(self._pix(image), self._tokens, self.pool.direction.clone())

    def _pix(self, image):
        """pixel mode: the 7x7x3 observation the step kernel wrote -> the 56x56x3 picture (one HBM-bound kernel)"""
        return self.pool.render_rgb(image) if self.pixel else image

    def _new_image(self):
        n = self.pool.num_envs
        return torch.empty((n, 7, 7, 3), dtype=torch.uint8, device=self.pool.device)

    def reset(self):
        img = self._new_image()
        self.pool.reset(obs=img)
        return self._batch(img, True)

    def step(self, actions):
        """actions: N values in 0..6 -- numpy (base.py:144), a sequence, or a torch tensor on any device (evaluate.py:124)."""
        dev = self.pool.device
        if self.fused_io:
            a = actions.cpu().numpy() if torch.is_tensor(actions) else np.asarray(actions)
            img, dire = self._new_image(), torch.empty(self.pool.num_envs, dtype=torch.int8, device=dev)
            self.pool.step_learner(a.astype(np.int8), img, self._rew_h, self._done_h, dire)
            rew_h, done_h = self._rew_h.copy(), self._done_h.astype(bool)
            if done_h.any() or self._tokens is None:
                self._tokens = self.pool.mission_tokens.clone()
            return iter((ObsBatch(self._pix(img), self._tokens, dire), rew_h, done_h, _Infos(len(done_h))))
        if torch.is_tensor(actions):
            a = actions.to(device=dev, dtype=torch.int8).contiguous()
        else:
            a = torch.as_tensor(np.ascontiguousarray(np.asarray(actions).astype(np.int8))).to(dev)
        img = self._new_image()                              # a fresh tensor per step: the batch owns it
        _, rew, done = self.pool.step(a, obs=img)
        rew_h = rew.cpu().numpy().copy()
        done_h = done.cpu().numpy().astype(bool)
        obs = self._batch(img, bool(done_h.any()))
        # penv.py:51-52 returns zip(*per_env_results): four sequences (obs, reward, done, info)
        return iter((obs, rew_h, done_h, _Infos(len(done_h))))

    def render(self):
        raise NotImplementedError                          # penv.py:54-55


class DeviceManyEnvs(DeviceParallelEnv):
    """babyai.evaluate.ManyEnvs surface (evaluate.py:58-81: seed / reset / step; finished envs freeze and repeat their last
    result) with the observations resident on the device -- `batch_evaluate` + `ModelAgent.act_batch` consume it
    unchanged when the agent's preprocessor is learner.ObssPreprocessor.  Accepts the plain gym.make list batch_evaluate
    builds, like vecenv.ManyEnvs."""
    MODE = MODE_FREEZE

    def seed(self, seeds):
        self.pool.seed(list(seeds))

    def reset_envs(self, env_ids, seeds, obs):
        """env.seed(seeds[k]) + env.reset() for envs env_ids[k] (BabyAIVecEnv.reset_envs): returns `obs` -- the batch the last
        step() returned -- with the rows of those envs replaced by their first observations and their new missions."""
        img, dire = obs.image, obs.direction.clone()
        if self.pixel:
            raw = self._new_image()
            self.pool.reset_envs(env_ids, seeds, obs=raw, direction=dire)
            idx = torch.as_tensor(np.asarray(env_ids, dtype=np.int64), device=self.pool.device)
            img = img.clone()
            img[idx] = self.pool.render_rgb(raw[idx].contiguous())
        else:
            img = img.clone()
            self.pool.reset_envs(env_ids, seeds, obs=img, direction=dire)
        self._tokens = self.pool.mission_tokens.clone()
        return ObsBatch(img, self._tokens, dire)

    def step(self, actions):
        obs, rew, done, info = super().step(actions)
        # evaluate.py:78 zips per-env result tuples; ModelAgent.analyze_feedback (utils/agent.py:76-82) tells a tuple of
        # Python bools (`if done[i]`) from a tensor (`1 - done`): hand it the tuple
        return iter((obs, tuple(float(r) for r in rew), tuple(bool(d) for d in done), info))


class ObssPreprocessor(object):
    """Drop-in for babyai.utils.format.ObssPreprocessor (format.py:100-119) over device-resident observations.

    `dictlist` is the container class to return (pass `babyai.rl.DictList` to hand the reference its own type; the default
    is ObsTensors, the image / instr pair with row indexing).  `trim=True` cuts the token tensor to the longest mission of the batch,
    as the reference pads (format.py:66-71); it costs one scalar device->host read."""

    def __init__(self, vocab_path=None, dictlist=ObsTensors, trim=True):
        self.vocab = FixedVocabulary(vocab_path)
        self.obs_space = {'image': 147, 'instr': self.vocab.max_size}       # format.py:104-107
        self.dictlist = dictlist
        self.trim = trim

    def _finish(self, image, tokens, device):
        if self.trim and tokens.shape[0]:
            width = int((tokens != 0).sum(1).max())
            tokens = tokens[:, :width]
        out = self.dictlist()
        out.image = image.to(device=device, dtype=torch.float)
        out.instr = tokens.to(device=device, dtype=torch.long)
        return out

    def __call__(self, obss, device=None):
        if isinstance(obss, ObsBatch):
            return self._finish(obss.image, obss.tokens, device)
        # a list of ObsRef in any order (base.py:208-210 builds it env-major over the T batches of a rollout)
        n = len(obss)
        if n == 0 or not isinstance(obss[0], ObsRef):
            raise TypeError('ObssPreprocessor expects the ObsBatch / ObsRef objects DeviceParallelEnv returns')
        serial = np.fromiter((r.batch.serial for r in obss), dtype=np.int64, count=n)
        env = np.fromiter((r.j for r in obss), dtype=np.int64, count=n)
        uniq, first_at = np.unique(serial, return_index=True)
        first = [obss[int(k)].batch for k in first_at]       # one representative ObsRef per distinct batch
        slot = np.searchsorted(uniq, serial)
        dev = first[0].image.device
        slot_t, env_t = torch.as_tensor(slot).to(dev), torch.as_tensor(env).to(dev)
        image = torch.stack([b.image for b in first])[slot_t, env_t]
        width = max(b.tokens.shape[1] for b in first)
        toks = torch.stack([b.tokens if b.tokens.shape[1] == width else torch.nn.functional.pad(b.tokens, (0, width - b.tokens.shape[1]))
                            for b in first])[slot_t, env_t]
        return self._finish(image, toks, device)
