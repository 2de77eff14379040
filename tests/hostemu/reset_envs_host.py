"""TEST-ONLY host builds of bb_pool_reset_envs: the host build of the kernel logic with a per-env seed and reset
(reset_envs_host.cpp: hostemu.cpp + he_seed_envs / he_reset_envs), and k_reset8's role with one OS thread per lane over the
ring-layout pool of simt_rollout.cpp (simt_reset.cpp).  Never imported by babyai_b200/."""
import ctypes as C
import os

import numpy as np

import hostemu
from hostemu import HERE, ROOT, _compile, _p

SRC = os.path.join(HERE, 'reset_envs_host.cpp')
OUT = os.path.join(HERE, 'libreset_envs_host.so')
DEPS = [SRC, hostemu.SRC] + hostemu.DEPS[1:]
SRC_SIMT = os.path.join(HERE, 'simt_reset.cpp')
OUT_SIMT = os.path.join(HERE, 'libsimt_reset.so')
DEPS_SIMT = [SRC_SIMT, os.path.join(ROOT, 'babyai_b200', 'csrc', 'reset8.cuh')] + hostemu.DEPS2
_lib = _lib_simt = None


def _stale(out, deps):
    return not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps))


def lib():
    global _lib
    if _lib is None:
        if _stale(OUT, DEPS):
            _compile(['g++', '-O1', '-g', '-std=c++17', '-Wall', '-Wno-unknown-pragmas', '-Wno-unused-function', '-ffp-contract=off',
                      '-shared', '-fPIC', SRC], OUT)
        L = C.CDLL(OUT)
        L.he_create.restype = C.c_void_p
        L.he_create.argtypes = [C.c_void_p, C.c_int]
        L.he_destroy.argtypes = [C.c_void_p]
        L.he_set_mode.argtypes = [C.c_void_p, C.c_int]
        L.he_seed.argtypes = [C.c_void_p, C.c_void_p]
        L.he_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.he_step.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        L.he_tokens.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.he_get_state.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.he_width.argtypes = [C.c_void_p]
        L.he_height.argtypes = [C.c_void_p]
        L.he_seed_envs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.he_reset_envs.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def lib_simt():
    global _lib_simt
    if _lib_simt is None:
        if _stale(OUT_SIMT, DEPS_SIMT):
            _compile(['g++', '-O1', '-g', '-std=c++20', '-pthread', '-Wall', '-Wno-unknown-pragmas', '-Wno-unused-function',
                      '-fno-strict-aliasing', '-ffp-contract=off', '-shared', '-fPIC', SRC_SIMT], OUT_SIMT)
        L = C.CDLL(OUT_SIMT)
        L.r2_create.restype = C.c_void_p
        L.r2_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.r2_destroy.argtypes = [C.c_void_p]
        L.r2_step8.argtypes = [C.c_void_p] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
        L.r2_state.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.r2_tokens.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.r2_max_tokens.argtypes = [C.c_void_p]
        L.r2_error_flag.argtypes = [C.c_void_p]
        L.r2_min_ring_level.argtypes = [C.c_void_p]
        L.r2_seed_envs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.r2_reset_envs.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib_simt = L
    return _lib_simt


def _ids_seeds(ids, seeds):
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    if seeds is not None:
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        assert seeds.shape == ids.shape
    return ids, seeds


class ResetHostPool(hostemu.HostEmuPool):
    """HostEmuPool on the library that also has the per-env seed and reset"""

    def __init__(self, spec, n, seeds=None, mode=0):
        self.L = lib()
        self.n = n
        self.spec = spec
        self.h = self.L.he_create(C.byref(spec), n)
        self.L.he_set_mode(self.h, mode)
        self.width = self.L.he_width(self.h)
        self.height = self.L.he_height(self.h)
        self.obs = np.zeros((n, 7, 7, 3), np.uint8)
        self.reward = np.zeros(n, np.float32)
        self.done = np.zeros(n, np.uint8)
        self.direction = np.zeros(n, np.int8)
        if seeds is not None:
            self.seed(seeds)

    def reset_envs(self, ids, seeds=None):
        """env.seed(seeds[k]) (if given) and env.reset() for envs ids[k]; writes their rows of self.obs / self.direction"""
        ids, seeds = _ids_seeds(ids, seeds)
        if seeds is not None:
            self.L.he_seed_envs(self.h, _p(ids), _p(seeds), ids.size)
        self.L.he_reset_envs(self.h, _p(ids), ids.size, _p(self.obs), _p(self.direction))
        return self.obs


class SimtResetPool(hostemu.RolloutPool):
    """RolloutPool on the library that also runs k_reset8's role (and k_step8's, for the steps between resets)"""

    def __init__(self, spec, n, seeds, depth=24, mode=0):
        self.L, self.n = lib_simt(), n
        s = np.ascontiguousarray(seeds, dtype=np.uint64)
        self.h = self.L.r2_create(C.byref(spec), n, depth, _p(s), mode)

    def reset_envs(self, ids, seeds=None, obs=None, dirs=None):
        """bb_pool_reset_envs' device work on the host -> (obs [n, 7, 7, 3], dirs [n], counters); only the listed rows of
        obs / dirs are written"""
        ids, seeds = _ids_seeds(ids, seeds)
        obs = np.zeros((self.n, 7, 7, 3), np.uint8) if obs is None else obs
        dirs = np.zeros(self.n, np.int8) if dirs is None else dirs
        cnt = np.zeros(4, np.int64)
        if seeds is not None:
            self.L.r2_seed_envs(self.h, _p(ids), _p(seeds), ids.size)
        self.L.r2_reset_envs(self.h, _p(ids), ids.size, _p(obs), _p(dirs), _p(cnt))
        return obs, dirs, cnt
