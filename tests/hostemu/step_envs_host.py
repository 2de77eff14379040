"""TEST-ONLY host build of bb_pool_step_envs (step_envs_host.cpp: k_step8_sel's role with one OS thread per lane over the
ring-layout pool of simt_rollout.cpp, beside the reset / save / load host builds).  Never imported by babyai_b200/."""
import ctypes as C
import os

import numpy as np

import reset_envs_host
import save_load_host
from hostemu import HERE, ROOT, _compile, _p

SRC = os.path.join(HERE, 'step_envs_host.cpp')
OUT = os.path.join(HERE, 'libstep_envs_host.so')
DEPS = [SRC, os.path.join(ROOT, 'babyai_b200', 'csrc', 'step8_sel.cuh')] + save_load_host.DEPS
_lib = None


def lib():
    global _lib
    if _lib is None:
        if reset_envs_host._stale(OUT, DEPS):
            _compile(['g++', '-O1', '-g', '-std=c++20', '-pthread', '-Wall', '-Wno-unknown-pragmas', '-Wno-unused-function',
                      '-fno-strict-aliasing', '-ffp-contract=off', '-shared', '-fPIC', SRC], OUT)
        L = C.CDLL(OUT)
        vp, i = C.c_void_p, C.c_int
        L.r2_create.restype = vp
        L.r2_create.argtypes = [vp, i, i, vp, i]
        L.r2_destroy.argtypes = [vp]
        L.r2_step8.argtypes = [vp] + [vp] * 5 + [i, vp]
        L.r2_state.argtypes = [vp, i, vp, vp]
        L.r2_tokens.argtypes = [vp, i, vp]
        L.r2_max_tokens.argtypes = [vp]
        L.r2_error_flag.argtypes = [vp]
        L.r2_min_ring_level.argtypes = [vp]
        L.r2_seed_envs.argtypes = [vp, vp, vp, i]
        L.r2_reset_envs.argtypes = [vp, vp, i, vp, vp, vp]
        L.r2_record_bytes.restype = C.c_int64
        L.r2_record_bytes.argtypes = [vp]
        L.r2_save_envs.argtypes = [vp, vp, i, vp]
        L.r2_load_envs.argtypes = [vp, vp, vp, i] + [vp] * 4
        L.r2_dump.restype = C.c_int64
        L.r2_dump.argtypes = [vp, vp]
        L.r2_ring.argtypes = [vp, i, vp]
        L.r2_step_envs.argtypes = [vp, vp, i, vp, i] + [vp] * 5
        _lib = L
    return _lib


class StepEnvsPool(save_load_host.SaveLoadPool):
    """SaveLoadPool on the library that also steps an id list through k_step8_sel's role"""

    def __init__(self, spec, n, seeds, depth=24, mode=0):
        self.L, self.n = lib(), n
        s = np.ascontiguousarray(seeds, dtype=np.uint64)
        self.h = self.L.r2_create(C.byref(spec), n, depth, _p(s), mode)
        self.record_bytes = int(self.L.r2_record_bytes(self.h))

    def step_envs(self, ids, actions, obs=None, reward=None, done=None, dirs=None):
        """bb_pool_step_envs' device work on the host: action k for env ids[k] -> (obs [n, 7, 7, 3], reward [n], done [n],
        dirs [n], counters); only the listed rows of the outputs are written.  actions: int8 or int64 numpy, one per id"""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        a = np.ascontiguousarray(actions)
        assert a.dtype in (np.int8, np.uint8, np.int64) and a.shape == ids.shape and np.unique(ids).size == ids.size
        n = self.n
        obs = np.zeros((n, 7, 7, 3), np.uint8) if obs is None else obs
        reward = np.zeros(n, np.float32) if reward is None else reward
        done = np.zeros(n, np.uint8) if done is None else done
        dirs = np.zeros(n, np.int8) if dirs is None else dirs
        cnt = np.zeros(4, np.int64)
        self.L.r2_step_envs(self.h, _p(ids), ids.size, _p(a), a.itemsize, _p(obs), _p(reward), _p(done), _p(dirs), _p(cnt))
        return obs, reward, done, dirs, cnt
