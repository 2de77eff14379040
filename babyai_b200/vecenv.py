"""Host-side mirror of the reference's environment-facing interface, on top of
the C ABI (include/babyai_b200.h):

  BabyAIVecEnv      tensor API: everything stays in PyTorch-owned CUDA tensors
  ParallelEnv       drop-in for babyai.rl.utils.penv.ParallelEnv (penv.py:18-59):
                    reset() -> list of obs dicts, step(actions) -> (obs, reward, done,
                    info) sequences (zip(*results)) with auto-reset on done
  ManyEnvs          drop-in for babyai.evaluate.ManyEnvs (evaluate.py:58-81):
                    seed(seeds), reset(), step() that freezes finished envs
  make_envs         what `[gym.make(id) ...; env.seed(100*seed+i)]` builds in
                    scripts/train_rl.py:53-60, as one list-like handle
  preprocess_obss   the pool's CURRENT observation as model inputs (image float, instr long);
                    the full learner-facing adapters (per-step batches AND the flattened
                    rollout BaseAlgo builds) are babyai_b200/learner.py

PyTorch is used for device memory and streams only.
"""
import ctypes as C

import numpy as np
import torch

from . import lib as _lib
from .levels import VOCAB, LevelSpec, detokenize, level_spec

MODE_AUTORESET, MODE_FREEZE = 0, 1


class _DevArray(object):
    """A device pointer owned by the pool, exposed through the CUDA array interface."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': typestr, 'data': (int(ptr), False),
                                         'version': 2, 'strides': None}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _check(t, name, device, dtype, shape):
    """the kernels write through raw pointers: a wrong-sized, strided or foreign-device buffer would be a silent
    out-of-bounds device write"""
    if t is None:
        return
    dtypes = dtype if isinstance(dtype, tuple) else (dtype,)
    if not (torch.is_tensor(t) and t.is_cuda and t.device == device):
        raise ValueError('%s must be a CUDA tensor on %s' % (name, device))
    if t.dtype not in dtypes or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
        raise ValueError('%s must be a contiguous %s tensor of shape %s (got %s %s)' % (name, dtypes[0], tuple(shape), t.dtype, tuple(t.shape)))


def level_groups(level):
    """A level name -> None.  A dict {level_name: count} or a sequence of (level_name, count) pairs -> the list of
    (level_name, count) groups of a mixed pool, in order (a level may appear in several groups)."""
    if isinstance(level, str):
        return None
    items = list(level.items()) if isinstance(level, dict) else list(level)
    groups = []
    for item in items:
        if not (isinstance(item, (tuple, list)) and len(item) == 2 and isinstance(item[0], str)):
            raise ValueError('a mixed pool is given as (level_name, count) pairs, got %r' % (item,))
        name, count = item
        if isinstance(count, bool) or int(count) != count or count < 1:
            raise ValueError('every group needs a whole number of envs >= 1, got %r for %s' % (count, name))
        level_spec(name)                                   # unknown levels fail here, before anything is allocated
        groups.append((name, int(count)))
    if not groups:
        raise ValueError('a mixed pool needs at least one (level_name, count) group')
    if sum(c for _, c in groups) > 2 ** 31 - 1:
        raise ValueError('a pool holds at most 2**31 - 1 envs')
    return groups


class BabyAIVecEnv(object):
    """N environments of one BabyAI level living in HBM of one GPU -- or, with `level` a sequence of (level_name, count)
    pairs, a MIXED pool: group g holds envs [start, start + count) of its level (`groups`), each group stepped by its own
    level's kernels, every buffer indexed by env row as for one level (bb_pool_create_mixed)."""

    def __init__(self, level, num_envs=None, seeds=None, device=0, mode=MODE_AUTORESET):
        self.L = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError('babyai_b200 needs a CUDA device; there is no CPU fallback')
        self.level = level
        pairs = level_groups(level)
        if pairs is None:
            pairs = [(level, int(num_envs))]
        elif num_envs is not None and int(num_envs) != sum(c for _, c in pairs):
            raise ValueError('num_envs (%d) is not the sum of the group sizes (%d)' % (num_envs, sum(c for _, c in pairs)))
        self.num_envs = sum(c for _, c in pairs)
        self.device = torch.device('cuda', device)
        starts = np.cumsum([0] + [c for _, c in pairs])[:-1]
        self.groups = [(name, int(s), c) for (name, c), s in zip(pairs, starts)]
        self.mixed = len(self.groups) > 1
        self._starts = np.asarray(starts, np.int64)
        h = C.c_void_p()
        torch.cuda.set_device(self.device)
        if self.mixed:
            self.spec = None
            specs = (LevelSpec * len(pairs))(*[level_spec(name) for name, _ in pairs])
            counts = (C.c_int32 * len(pairs))(*[c for _, c in pairs])
            _lib.check(self.L.bb_pool_create_mixed(specs, counts, len(pairs), device, C.byref(h)))
        else:
            self.spec = level_spec(pairs[0][0])
            _lib.check(self.L.bb_pool_create(C.byref(self.spec), self.num_envs, device, C.byref(h)))
        self.h = h
        self.width = self.L.bb_pool_width(h)              # a mixed pool: the largest grid of its groups
        self.height = self.L.bb_pool_height(h)
        self._dims = []                                    # (width, height) of each group
        for _, s, _ in self.groups:
            w, hh = C.c_int32(), C.c_int32()
            _lib.check(self.L.bb_pool_env_dims(h, s, C.byref(w), C.byref(hh)))
            self._dims.append((w.value, hh.value))
        n = self.num_envs
        self.obs = torch.zeros((n, 7, 7, 3), dtype=torch.uint8, device=self.device)
        self.reward = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.done = torch.zeros(n, dtype=torch.uint8, device=self.device)
        self.direction = torch.zeros(n, dtype=torch.int8, device=self.device)
        tp, ml = C.c_void_p(), C.c_int32()
        _lib.check(self.L.bb_pool_mission_tokens(h, C.byref(tp), C.byref(ml)))
        self.max_tokens = ml.value
        self.mission_tokens = torch.as_tensor(_DevArray(tp.value, (n, ml.value), '<i2'), device=self.device)
        self.mode = MODE_AUTORESET
        if mode != MODE_AUTORESET:
            self.set_mode(mode)
        if seeds is not None:
            self.seed(seeds)

    def group_of(self, env_ids):
        """index into `groups` of each env id"""
        return np.searchsorted(self._starts, np.asarray(env_ids), side='right') - 1

    def level_of(self, env):
        """the level name of env `env`"""
        if not 0 <= int(env) < self.num_envs:
            raise IndexError(env)
        return self.groups[int(self.group_of(int(env)))][0]

    def _single_level(self, what):
        if self.mixed:
            raise RuntimeError('%s is not available on a mixed pool: an env record does not name its level, so a record of '
                               'one group could load silently into an env of another level' % what)

    def close(self):
        if getattr(self, 'h', None) is not None and self.h:
            self.L.bb_pool_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_mode(self, mode):
        _lib.check(self.L.bb_pool_set_mode(self.h, mode))
        self.mode = mode

    def seed(self, seeds):
        s = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64))
        assert s.shape == (self.num_envs,)
        _lib.check(self.L.bb_pool_seed(self.h, s.ctypes.data_as(C.c_void_p)))

    def reset(self, obs=None, direction=None):
        obs = self.obs if obs is None else obs
        direction = self.direction if direction is None else direction
        n = self.num_envs
        _check(obs, 'obs', self.device, torch.uint8, (n, 7, 7, 3))
        _check(direction, 'direction', self.device, torch.int8, (n,))
        _lib.check(self.L.bb_pool_reset(self.h, _ptr(obs), _ptr(direction), self._stream()))
        return obs

    def _env_ids(self, env_ids):
        """a 1-D sequence (list, numpy array or tensor) of env ids in [0, N) -> contiguous int32 numpy array"""
        return self._env_ids_like(env_ids, self.num_envs, 'env ids')

    @staticmethod
    def _env_ids_like(values, bound, name):
        if torch.is_tensor(values):
            values = values.cpu().numpy()
        a = np.asarray(values)
        if a.ndim != 1 or (a.size and a.dtype.kind not in 'iu'):
            raise ValueError('%s must be a 1-D sequence of integers' % name)
        if a.size and (a.min() < 0 or a.max() >= bound):
            raise ValueError('%s must be in [0, %d)' % (name, bound))
        return np.ascontiguousarray(a, dtype=np.int32)

    def reset_envs(self, env_ids, seeds=None, obs=None, direction=None):
        """A new episode for the listed envs only (bb_pool_reset_envs): env.seed(seeds[k]) if seeds are given, then
        env.reset(), for env env_ids[k].  Without seeds an env takes the next level of its own stream.  Only the listed rows
        of obs [N, 7, 7, 3] and direction [N] (default: the pool's own buffers) are written, and only their missions change;
        in freeze mode the listed envs step again.  Ids must not repeat.  Returns obs."""
        ids = self._env_ids(env_ids)
        if np.unique(ids).size != ids.size:
            raise ValueError('env ids must not repeat')
        s = None
        if seeds is not None:
            if torch.is_tensor(seeds):
                seeds = seeds.cpu().numpy()
            s = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64))
            if s.shape != ids.shape:
                raise ValueError('seeds must have one value per env id (%d), got shape %s' % (ids.size, s.shape))
        obs = self.obs if obs is None else obs
        direction = self.direction if direction is None else direction
        n = self.num_envs
        _check(obs, 'obs', self.device, torch.uint8, (n, 7, 7, 3))
        _check(direction, 'direction', self.device, torch.int8, (n,))
        _lib.check(self.L.bb_pool_reset_envs(self.h, ids.ctypes.data_as(C.c_void_p),
                                             s.ctypes.data_as(C.c_void_p) if s is not None else None, ids.size,
                                             _ptr(obs), _ptr(direction), self._stream()))
        return obs

    # ---- env records: save, load, fork (bb_pool_save_envs / bb_pool_load_envs) ----------------------------------------
    @property
    def record_bytes(self):
        """bytes of one env record: the row length of the tensors save_envs returns and load_envs takes"""
        self._single_level('record_bytes')
        return int(self.L.bb_pool_env_record_bytes(self.h))

    def _check_records(self, records, name, rows=None):
        if not (torch.is_tensor(records) and records.is_cuda and records.device == self.device and records.dtype == torch.uint8
                and records.is_contiguous() and records.dim() == 2 and records.shape[1] == self.record_bytes
                and (rows is None or records.shape[0] == rows) and records.data_ptr() % 16 == 0):
            raise ValueError('%s must be a contiguous, 16-byte aligned CUDA uint8 tensor [%s, %d] on %s'
                             % (name, 'n' if rows is None else rows, self.record_bytes, self.device))

    def save_envs(self, ids=None, out=None):
        """Records of the listed envs (default: every env, in order) -> uint8 [n_sel, record_bytes] on the pool's device
        (`out`, or a new tensor).  A record holds everything the env's future depends on, the levels its generator has
        already produced included, so load_envs of it continues exactly as the env would have.  The pool is unchanged; ids
        may repeat.  `torch.save(records.cpu(), path)` of the result is a checkpoint of the env side of a run."""
        self._single_level('save_envs')
        ids = None if ids is None else self._env_ids(ids)
        n_sel = self.num_envs if ids is None else ids.size
        if out is None:
            out = torch.empty((n_sel, self.record_bytes), dtype=torch.uint8, device=self.device)
        self._check_records(out, 'out', n_sel)
        _lib.check(self.L.bb_pool_save_envs(self.h, ids.ctypes.data_as(C.c_void_p) if ids is not None else None, n_sel,
                                            _ptr(out), self._stream()))
        return out

    def load_envs(self, records, ids=None, slots=None, obs=None, direction=None):
        """Env ids[k] (default: env k, every env) becomes record slots[k] (default: record k) of `records`, a tensor save_envs
        returned on a pool of the same level and ring depth.  Slots may repeat (one record into many envs), ids may not.
        Only the listed rows of obs / direction (default: the pool's own buffers) are written -- the observations of the
        loaded states -- and only the listed envs' missions change; unlisted envs are untouched.  Returns (obs, direction)."""
        self._single_level('load_envs')
        self._check_records(records, 'records')
        ids = None if ids is None else self._env_ids(ids)
        if ids is not None and np.unique(ids).size != ids.size:
            raise ValueError('env ids must not repeat')
        n_sel = self.num_envs if ids is None else ids.size
        if slots is not None:
            slots = self._env_ids_like(slots, records.shape[0], 'slots')
            if slots.size != n_sel:
                raise ValueError('slots must have one value per env id (%d), got %d' % (n_sel, slots.size))
        elif n_sel > records.shape[0]:
            raise ValueError('%d envs to load but only %d records' % (n_sel, records.shape[0]))
        obs = self.obs if obs is None else obs
        direction = self.direction if direction is None else direction
        n = self.num_envs
        _check(obs, 'obs', self.device, torch.uint8, (n, 7, 7, 3))
        _check(direction, 'direction', self.device, torch.int8, (n,))
        _lib.check(self.L.bb_pool_load_envs(self.h, ids.ctypes.data_as(C.c_void_p) if ids is not None else None,
                                            slots.ctypes.data_as(C.c_void_p) if slots is not None else None, n_sel,
                                            _ptr(records), records.shape[0], _ptr(obs), _ptr(direction), self._stream()))
        return obs, direction

    def copy_envs(self, src_ids, dst_ids, obs=None, direction=None):
        """Env dst_ids[k] becomes a copy of env src_ids[k] as it is now (copy.deepcopy of a reference env): sources may
        repeat, destinations may not, and a destination may also be a source (every source is saved before any env is
        loaded).  Returns (obs, direction) as load_envs does."""
        self._single_level('copy_envs')
        src, dst = self._env_ids(src_ids), self._env_ids(dst_ids)
        if src.shape != dst.shape:
            raise ValueError('src_ids and dst_ids must have the same length')
        if np.unique(dst).size != dst.size:
            raise ValueError('env ids must not repeat')
        uniq, slots = np.unique(src, return_inverse=True)
        return self.load_envs(self.save_envs(uniq), dst, slots.reshape(-1), obs=obs, direction=direction)

    def step(self, actions, obs=None, reward=None, done=None, direction=None):
        """actions: CUDA tensor of N int8/uint8 or int64 values."""
        n = self.num_envs
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.device == self.device and actions.is_contiguous()
                and actions.numel() == n and actions.dtype in (torch.int8, torch.uint8, torch.int64)):
            raise ValueError('actions must be a contiguous CUDA tensor of %d int8 / uint8 / int64 values on %s' % (n, self.device))
        nbytes = actions.element_size()
        obs = self.obs if obs is None else obs
        reward = self.reward if reward is None else reward
        done = self.done if done is None else done
        direction = self.direction if direction is None else direction
        self._check_step_outputs(obs, reward, done, direction, ())
        _lib.check(self.L.bb_pool_step(self.h, _ptr(actions), nbytes, _ptr(obs), _ptr(reward), _ptr(done),
                                       _ptr(direction), self._stream()))
        return obs, reward, done

    def step_envs(self, env_ids, actions, obs=None, reward=None, done=None, direction=None):
        """One step of the listed envs only (bb_pool_step_envs), every other env held still: env env_ids[k] takes action
        actions[k] -- a contiguous CUDA tensor of len(env_ids) int8 / uint8 / int64 values, what a policy evaluated on
        obs[env_ids] returns.  Only the listed rows of obs [N, 7, 7, 3], reward [N], done [N] and direction [N] (default:
        the pool's own buffers) are written, so they stay the pool's current view.  Ids must not repeat.  Returns
        (obs, reward, done)."""
        ids = self._env_ids(env_ids)
        seen = np.zeros(self.num_envs, bool)                   # linear (np.unique sorts: more host time than the launch)
        seen[ids] = True
        if np.count_nonzero(seen) != ids.size:
            raise ValueError('env ids must not repeat')
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.device == self.device and actions.is_contiguous()
                and actions.numel() == ids.size and actions.dtype in (torch.int8, torch.uint8, torch.int64)):
            raise ValueError('actions must be a contiguous CUDA tensor of %d int8 / uint8 / int64 values on %s (one per env id)'
                             % (ids.size, self.device))
        obs = self.obs if obs is None else obs
        reward = self.reward if reward is None else reward
        done = self.done if done is None else done
        direction = self.direction if direction is None else direction
        self._check_step_outputs(obs, reward, done, direction, ())
        _lib.check(self.L.bb_pool_step_envs(self.h, ids.ctypes.data_as(C.c_void_p), ids.size, _ptr(actions),
                                            actions.element_size(), _ptr(obs), _ptr(reward), _ptr(done), _ptr(direction),
                                            self._stream()))
        return obs, reward, done

    def _check_step_outputs(self, obs, reward, done, direction, lead):
        n = self.num_envs
        _check(obs, 'obs', self.device, torch.uint8, lead + (n, 7, 7, 3))
        _check(reward, 'reward', self.device, torch.float32, lead + (n,))
        _check(done, 'done', self.device, (torch.uint8, torch.bool), lead + (n,))
        _check(direction, 'direction', self.device, torch.int8, lead + (n,))

    def _check_rollout(self, actions, obs, reward, done, direction):
        if not (torch.is_tensor(actions) and actions.dim() == 2 and actions.shape[1] == self.num_envs and actions.shape[0] >= 1):
            raise ValueError('actions must have shape [T, %d]' % self.num_envs)
        _check(actions, 'actions', self.device, (torch.int8, torch.uint8), tuple(actions.shape))
        if obs is None or reward is None or done is None:
            raise ValueError('rollout needs obs, reward and done buffers')
        self._check_step_outputs(obs, reward, done, direction, (actions.shape[0],))

    def render_rgb(self, obs=None, out=None):
        """RGBImgPartialObsWrapper.observation for a batch (bb_pool_render_rgb): uint8 observations [..., 7, 7, 3] (default:
        the pool's current ones) -> uint8 images [..., 56, 56, 3] on the device; `obs` may be a whole [T, N, 7, 7, 3] rollout."""
        obs = self.obs if obs is None else obs
        if not (torch.is_tensor(obs) and obs.is_cuda and obs.device == self.device and obs.dtype == torch.uint8
                and obs.is_contiguous() and obs.dim() >= 3 and tuple(obs.shape[-3:]) == (7, 7, 3)):
            raise ValueError('obs must be a contiguous CUDA uint8 tensor [..., 7, 7, 3] on %s' % self.device)
        lead = tuple(obs.shape[:-3])
        if out is None:
            out = torch.empty(lead + (56, 56, 3), dtype=torch.uint8, device=self.device)
        _check(out, 'out', self.device, torch.uint8, lead + (56, 56, 3))
        _lib.check(self.L.bb_pool_render_rgb(self.h, _ptr(obs), _ptr(out), obs.numel() // 147, self._stream()))
        return out

    def render_grid(self, env_ids=None, tile_size=32, highlight=True, out=None):
        """MiniGridEnv.render('rgb_array', highlight=highlight, tile_size=tile_size) of the selected envs' CURRENT states
        (bb_pool_render_grid): uint8 [n_sel, H * tile_size, W * tile_size, 3] on the device.  env_ids: ids in [0, N) in any
        order, repeats allowed (default: every env in order).  On a mixed pool the selected envs must share one grid size
        (H, W: the level's own), e.g. one group per call."""
        ts = int(tile_size)
        if not 1 <= ts <= 64:
            raise ValueError('tile_size must be in 1..64 (got %r)' % (tile_size,))
        ids = None
        n_sel = self.num_envs
        if env_ids is not None:
            ids = self._env_ids(env_ids)
            n_sel = ids.size
        width, height = self._sel_dims(ids, n_sel, 'render_grid')
        shape = (n_sel, height * ts, width * ts, 3)
        if out is None:
            out = torch.empty(shape, dtype=torch.uint8, device=self.device)
        _check(out, 'out', self.device, torch.uint8, shape)
        _lib.check(self.L.bb_pool_render_grid(self.h, ids.ctypes.data_as(C.c_void_p) if ids is not None else None, n_sel, ts,
                                              1 if highlight else 0, _ptr(out), self._stream()))
        return out

    def full_obs(self, env_ids=None, out=None):
        """FullyObsWrapper.observation(obs)['image'] of the selected envs' CURRENT states (bb_pool_full_obs): grid.encode() of
        the whole grid with the agent's cell (10, 0, agent_dir), uint8 [n_sel, W, H, 3] (x-major) on the device.  env_ids: ids
        in [0, N) in any order, repeats allowed (default: every env in order).  On a mixed pool the selected envs must share one
        grid size."""
        ids = None if env_ids is None else self._env_ids(env_ids)
        n_sel = self.num_envs if ids is None else ids.size
        width, height = self._sel_dims(ids, n_sel, 'full_obs')
        shape = (n_sel, width, height, 3)
        if out is None:
            out = torch.empty(shape, dtype=torch.uint8, device=self.device)
        _check(out, 'out', self.device, torch.uint8, shape)
        _lib.check(self.L.bb_pool_full_obs(self.h, ids.ctypes.data_as(C.c_void_p) if ids is not None else None, n_sel,
                                           _ptr(out), self._stream()))
        return out

    def _sel_dims(self, ids, n_sel, what):
        """(width, height) every selected env shares; on a mixed pool a ValueError when they differ"""
        if not (self.mixed and n_sel):
            return self.width, self.height
        dims = {self._dims[g] for g in np.unique(self.group_of(np.arange(self.num_envs) if ids is None else ids))}
        if len(dims) != 1:
            raise ValueError('the envs of one %s call must share one grid size (got %s): call once per size' % (what, sorted(dims)))
        return dims.pop()

    def step_timed(self, actions):
        """bb_pool_step with CUDA events around each kernel -> (ms k_step, ms k_gen)."""
        self._single_level('step_timed')
        a, b = C.c_float(), C.c_float()
        _lib.check(self.L.bb_pool_step_timed(self.h, _ptr(actions), actions.element_size(), _ptr(self.obs),
                                             _ptr(self.reward), _ptr(self.done), _ptr(self.direction),
                                             C.byref(a), C.byref(b)))
        return a.value, b.value

    def rollout(self, actions, obs, reward, done, direction=None):
        """actions int8 [T, N] (CUDA); outputs [T, N, ...] CUDA tensors written in place."""
        self._check_rollout(actions, obs, reward, done, direction)
        T = actions.shape[0]
        _lib.check(self.L.bb_pool_rollout(self.h, _ptr(actions), T, _ptr(obs), _ptr(reward), _ptr(done),
                                          _ptr(direction), self._stream()))
        return obs, reward, done

    def rollout_timed(self, actions, obs, reward, done, direction=None):
        """rollout() with CUDA events around the stepping kernel and the level refill -> (ms, ms)."""
        self._single_level('rollout_timed')
        self._check_rollout(actions, obs, reward, done, direction)
        a, b = C.c_float(), C.c_float()
        _lib.check(self.L.bb_pool_rollout_timed(self.h, _ptr(actions), actions.shape[0], _ptr(obs), _ptr(reward), _ptr(done),
                                                _ptr(direction), C.byref(a), C.byref(b)))
        return a.value, b.value

    # ---- host-buffer path (what the reference's callers see) -----------------
    def step_host(self, actions, obs, reward, done, direction):
        a = np.ascontiguousarray(actions, dtype=np.int8)
        _lib.check(self.L.bb_pool_step_host(self.h, a.ctypes.data_as(C.c_void_p), obs.ctypes.data_as(C.c_void_p),
                                            reward.ctypes.data_as(C.c_void_p), done.ctypes.data_as(C.c_void_p),
                                            direction.ctypes.data_as(C.c_void_p)))

    def step_learner(self, actions, obs, reward, done, direction=None):
        """bb_pool_step_learner: actions int8 numpy (host) -> obs (and direction) CUDA tensors, reward float32 / done uint8
        numpy (host); synchronises the current stream."""
        a = np.ascontiguousarray(actions, dtype=np.int8)
        assert a.shape == (self.num_envs,) and reward.dtype == np.float32 and done.dtype == np.uint8
        _lib.check(self.L.bb_pool_step_learner(self.h, a.ctypes.data_as(C.c_void_p), _ptr(obs), reward.ctypes.data_as(C.c_void_p),
                                               done.ctypes.data_as(C.c_void_p), _ptr(direction), self._stream()))

    def reset_host(self, obs, direction):
        _lib.check(self.L.bb_pool_reset_host(self.h, obs.ctypes.data_as(C.c_void_p),
                                             direction.ctypes.data_as(C.c_void_p)))

    # ---- introspection ----------------------------------------------------------
    def missions(self, idx=None):
        tok = self.mission_tokens.cpu().numpy()
        idx = range(self.num_envs) if idx is None else idx
        return [detokenize(tok[i]) for i in idx]

    def state(self, i):
        """(grid uint8 [H, W] of the env's own level, hidden-state dict)"""
        width, height = self._dims[int(self.group_of(int(i)))] if 0 <= int(i) < self.num_envs else (self.width, self.height)
        grid = np.zeros((height, width), np.uint8)
        info = np.zeros(8, np.int32)
        _lib.check(self.L.bb_pool_get_state(self.h, i, grid.ctypes.data_as(C.c_void_p), info.ctypes.data_as(C.c_void_p)))
        return grid, dict(agent_x=int(info[0]), agent_y=int(info[1]), agent_dir=int(info[2]), carrying=int(info[3]),
                          step_count=int(info[4]), max_steps=int(info[5]), draws=int(info[6]), attempts=int(info[7]))

    def counters(self):
        c = np.zeros(4, np.int64)
        _lib.check(self.L.bb_pool_counters(self.h, c.ctypes.data_as(C.c_void_p)))
        return dict(steps=int(c[0]), episodes=int(c[1]), successes=int(c[2]), errors=int(c[3]))

    def launches(self):
        return int(self.L.bb_pool_launches(self.h))


# ---------------------------------------------------------------------------------
# gym-flavoured facades
# ---------------------------------------------------------------------------------
class _Space(object):
    pass


def _spaces(pixel=False, image_shape=None):
    """observation_space / action_space with the attributes the reference reads
    (utils/format.py:124-126: .spaces['image'].shape/.high; train_rl.py:96: action_space.n).  image_shape: the image of a
    fully observable list (EnvList.image_shape)."""
    img = _Space()
    img.shape = image_shape if image_shape is not None else (56, 56, 3) if pixel else (7, 7, 3)
    img.low = np.zeros(img.shape, np.uint8)
    img.high = np.full(img.shape, 255, np.uint8)
    img.dtype = np.dtype('uint8')
    obs = _Space()
    obs.spaces = {'image': img}
    act = _Space()
    act.n = 7
    return obs, act


class EnvHandle(object):
    """Stands for env i of a pool where the reference expects a list of gym envs."""

    def __init__(self, pool_spec, index):
        self.pool_spec = pool_spec
        self.index = index
        self.observation_space, self.action_space = _spaces(getattr(pool_spec, 'pixel', False), pool_spec.image_shape())


class EnvList(list):
    """What scripts/train_rl.py:53-60 builds: N seeded envs of one level -- or of several: `level` is then the list of
    (level_name, count) groups, in env order.  Two lists concatenate with `+` into the list of both groups.
    `full`: None (the 7x7 view, or its pictures with `pixel`), 'grid' (FullyObsWrapper) or 'rgb' (RGBImgObsWrapper at
    `tile_size`)."""

    def __init__(self, level, seeds, device=0, pixel=False, full=None, tile_size=8):
        self.level, self.seeds, self.device, self.pixel = level, list(seeds), device, bool(pixel)
        self.full, self.tile_size = full, int(tile_size)
        super().__init__(EnvHandle(self, i) for i in range(len(self.seeds)))

    def level_counts(self):
        """[(level_name, count), ...] in env order"""
        return level_groups(self.level) or [(self.level, len(self))]

    def wrapper(self):
        """what a batch of this list's observations is made of"""
        return (self.pixel, self.full, self.tile_size if self.full == 'rgb' else None)

    def image_shape(self):
        """obs['image'].shape of a fully observable list: FullyObsWrapper (W, H, 3); RGBImgObsWrapper (H ts, W ts, 3), the
        shape of the array MiniGridEnv.render returns (gym_minigrid declares (W ts, H ts, 3)); None for the 7x7 view"""
        if self.full is None:
            return None
        width, height = grid_dims(self.level_counts())
        return (width, height, 3) if self.full == 'grid' else (height * self.tile_size, width * self.tile_size, 3)

    def __add__(self, other):
        if not isinstance(other, EnvList):
            return list(self) + list(other)
        if other.device != self.device or other.wrapper() != self.wrapper():
            raise ValueError('only env lists on the same device and with the same observation wrapper concatenate')
        out = EnvList(self.level_counts() + other.level_counts(), self.seeds + other.seeds, self.device, self.pixel,
                      self.full, self.tile_size)
        out.image_shape()                                  # a fully observable list of two grid sizes fails here
        return out


def grid_dims(groups):
    """(width, height) of the grids of every level of [(level_name, count), ...] (RoomGrid: (room_size - 1) * num_cols + 1
    by (room_size - 1) * num_rows + 1); a ValueError when the levels' grids differ in size"""
    dims = set()
    for name, _ in groups:
        s = level_spec(name)
        dims.add(((s.room_size - 1) * s.num_cols + 1, (s.room_size - 1) * s.num_rows + 1))
    if len(dims) != 1:
        raise ValueError('a fully observable env list needs one grid size, got %s: wrap the lists of each size separately'
                         % sorted(dims))
    return dims.pop()


def make_envs(level, num_envs=None, seed=1, device=0, pixel=False):
    """`env.seed(100 * seed + i)` for env i (scripts/train_rl.py:59); pixel=True: every env wrapped in
    RGBImgPartialObsWrapper (train_rl.py:54-58, `'pixel' in args.arch`).  `level` may be a dict or a sequence of
    (level_name, count) pairs, e.g. {'GoToLocal': 64, 'BossLevel': 64}: the envs of several levels in that order (a
    multi-task list), i counting over the whole list; num_envs is then the sum of the counts or None."""
    groups = level_groups(level)
    if groups is not None:
        total = sum(c for _, c in groups)
        if num_envs is not None and int(num_envs) != total:
            raise ValueError('num_envs (%d) is not the sum of the group sizes (%d)' % (num_envs, total))
        num_envs = total
        level = groups if len(groups) > 1 else groups[0][0]
    return EnvList(level, [100 * seed + i for i in range(num_envs)], device, pixel)


def RGBImgPartialObsWrapper(envs, tile_size=8):
    """gym_minigrid.wrappers.RGBImgPartialObsWrapper for a whole env list: the pool's facades then return
    obs['image'] as uint8[56, 56, 3] pictures of the 7x7 view (tile size 8), rendered on the device by bb_pool_render_rgb."""
    if tile_size != 8:
        raise ValueError('the pool renders tile_size 8 (the size the pixel architectures consume, babyai/model.py:96-98)')
    if not isinstance(envs, EnvList):
        raise TypeError('wrap the list make_envs() built')
    return EnvList(envs.level, envs.seeds, envs.device, pixel=True)


def _wrap_full(envs, full, tile_size):
    if not isinstance(envs, EnvList):
        raise TypeError('wrap the list make_envs() built')
    if envs.wrapper() != (False, None, None):
        raise ValueError('the list is already wrapped: its envs have one observation wrapper')
    out = EnvList(envs.level, envs.seeds, envs.device, full=full, tile_size=tile_size)
    out.image_shape()                                      # one grid size
    return out


def FullyObsWrapper(envs):
    """gym_minigrid.wrappers.FullyObsWrapper for a whole env list: the pool's facades then return obs['image'] as
    grid.encode() of the whole grid, uint8[W, H, 3] with the agent's cell (10, 0, agent_dir), made on the device by
    bb_pool_full_obs, and obs dicts {'mission', 'image'}.  The levels of the list must share one grid size."""
    return _wrap_full(envs, 'grid', 8)


def RGBImgObsWrapper(envs, tile_size=8):
    """gym_minigrid.wrappers.RGBImgObsWrapper for a whole env list: obs['image'] is env.render('rgb_array', highlight=False,
    tile_size), uint8[H * tile_size, W * tile_size, 3], drawn on the device by bb_pool_render_grid (tile sizes 1..64)."""
    if isinstance(tile_size, bool) or int(tile_size) != tile_size or not 1 <= tile_size <= 64:
        raise ValueError('tile_size must be in 1..64 (got %r)' % (tile_size,))
    return _wrap_full(envs, 'rgb', int(tile_size))


def full_image(pool, full, tile_size, env_ids=None):
    """the fully observable images of a pool's envs (default: all): FullyObsWrapper ('grid') or RGBImgObsWrapper ('rgb')"""
    if full == 'grid':
        return pool.full_obs(env_ids)
    return pool.render_grid(env_ids, tile_size=tile_size, highlight=False)


def _as_env_list(envs, need_seeds):
    """An EnvList as is.  A plain list of reference envs -- what `batch_evaluate` builds with gym.make before it
    wraps them in ManyEnvs (evaluate.py:86-94) -- is accepted where the seeds arrive later through seed(): the level of
    each env is read from the reference's own class attribute (`level_name`, levelgen.py:492), and maximal runs of one
    level become the groups of a mixed pool, in list order."""
    if isinstance(envs, EnvList):
        return envs
    if need_seeds:
        raise TypeError('build the env list with babyai_b200.make_envs(): the seeds of gym envs cannot be read back')
    groups = []
    for env in envs:
        env = getattr(env, 'unwrapped', env)
        name = getattr(type(env), 'level_name', None)
        if not isinstance(name, str):
            raise TypeError('cannot tell the BabyAI level of %r; use babyai_b200.make_envs()' % (env,))
        if groups and groups[-1][0] == name:
            groups[-1][1] += 1
        else:
            groups.append([name, 1])
    groups = [tuple(g) for g in groups]
    return EnvList(groups if len(groups) > 1 else groups[0][0], [0] * len(envs))


class _HostVec(object):
    def __init__(self, envs, mode, pool=None):
        """`pool` is a test hook (an object with BabyAIVecEnv's host-buffer interface: the GPU-less suite passes the
        host build of the kernel logic); the product always builds the CUDA pool."""
        envs = _as_env_list(envs, need_seeds=(mode == MODE_AUTORESET))
        self.envs = envs
        self.pixel = bool(getattr(envs, 'pixel', False))
        self.full, self.tile_size = envs.full, envs.tile_size
        self.observation_space, self.action_space = _spaces(self.pixel, envs.image_shape())
        self.pool = pool if pool is not None else BabyAIVecEnv(envs.level, len(envs), seeds=envs.seeds, device=envs.device, mode=mode)
        n = len(envs)
        # page-locked host buffers: bb_pool_step_host DMAs straight into them
        pin = (lambda t: t.pin_memory()) if pool is None else (lambda t: t)
        self._pin = [pin(torch.zeros((n, 7, 7, 3), dtype=torch.uint8)), pin(torch.zeros(n, dtype=torch.float32)),
                     pin(torch.zeros(n, dtype=torch.uint8)), pin(torch.zeros(n, dtype=torch.int8))]
        self._obs, self._rew, self._done, self._dir = [t.numpy() for t in self._pin]
        self._missions = [''] * n

    def _obs_list(self, refresh):
        if refresh is None:
            self._missions = self.pool.missions()
        else:
            idx = np.nonzero(refresh)[0]
            if len(idx):
                for i, m in zip(idx, self.pool.missions(idx)):
                    self._missions[i] = m
        if self.full is not None:    # FullyObsWrapper / RGBImgObsWrapper.observation: {'mission', 'image'} of the current state
            img = full_image(self.pool, self.full, self.tile_size).cpu().numpy()
            return [{'image': img[i], 'mission': self._missions[i]} for i in range(len(self.envs))]
        if self.pixel:               # RGBImgPartialObsWrapper.observation: {'mission', 'image' uint8[56, 56, 3]} (no 'direction')
            dev = self.pool.device
            img = self.pool.render_rgb(torch.as_tensor(self._obs).to(dev)).cpu().numpy()
            return [{'image': img[i], 'mission': self._missions[i]} for i in range(len(self.envs))]
        img = self._obs.copy()
        return [{'image': img[i], 'direction': int(self._dir[i]), 'mission': self._missions[i]}
                for i in range(len(self.envs))]

    def render(self):
        raise NotImplementedError


class ParallelEnv(_HostVec):
    """babyai.rl.utils.penv.ParallelEnv surface (auto-reset on done)."""

    def __init__(self, envs, pool=None):
        super().__init__(envs, MODE_AUTORESET, pool)

    def reset(self):
        self.pool.reset_host(self._obs, self._dir)
        return self._obs_list(None)

    def step(self, actions):
        if torch.is_tensor(actions):
            actions = actions.cpu().numpy()
        self.pool.step_host(np.asarray(actions).astype(np.int8), self._obs, self._rew, self._done, self._dir)
        obs = self._obs_list(self._done)
        # penv.py:51-52 returns zip(*per_env_results): four sequences (obs, reward, done, info)
        return iter((tuple(obs), tuple(float(r) for r in self._rew), tuple(bool(d) for d in self._done),
                     tuple({} for _ in self.envs)))


class ManyEnvs(_HostVec):
    """babyai.evaluate.ManyEnvs surface (seed / reset / step; finished envs freeze)."""

    def __init__(self, envs, pool=None):
        super().__init__(envs, MODE_FREEZE, pool)

    def seed(self, seeds):
        self.pool.seed(list(seeds))

    def reset(self):
        self.pool.reset_host(self._obs, self._dir)
        return self._obs_list(None)

    def step(self, actions):
        if torch.is_tensor(actions):
            actions = actions.cpu().numpy()
        self.pool.step_host(np.asarray(actions).astype(np.int8), self._obs, self._rew, self._done, self._dir)
        obs = self._obs_list(np.zeros(len(self.envs), bool))
        # evaluate.py:78 returns zip(*self.results): four sequences
        return iter((tuple(obs), tuple(float(r) for r in self._rew), tuple(bool(d) for d in self._done),
                     tuple({} for _ in self.envs)))


def preprocess_obss(pool):
    """Returns a `preprocess_obss(obss, device=None)` callable that ignores its argument and hands the model the
    pool's CURRENT device tensors: image float[B,7,7,3], instr long[B,L] -- the acting half of rl/algos/base.py:134.
    BaseAlgo also preprocesses the flattened rollout (base.py:208-210,232): use learner.DeviceParallelEnv +
    learner.ObssPreprocessor for the complete contract."""
    from types import SimpleNamespace

    def fn(obss=None, device=None):
        return SimpleNamespace(image=pool.obs.float(), instr=pool.mission_tokens.long())
    fn.vocab = {w: i for i, w in enumerate(VOCAB) if i > 0}
    return fn
