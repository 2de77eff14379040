"""TEST-ONLY host build of the fully observable observations (full_obs_host.cpp: render_grid_host.cpp + csrc/full_obs.cuh
compiled with g++): a RenderHostPool that can also return FullyObsWrapper images of its envs.  Never imported by
babyai_b200/."""
import ctypes as C
import os

import numpy as np

import render_grid_host
from hostemu import HERE, ROOT, _compile

SRC = os.path.join(HERE, 'full_obs_host.cpp')
OUT = os.path.join(HERE, 'libfull_obs_host.so')
DEPS = [SRC] + render_grid_host.DEPS + [os.path.join(ROOT, 'babyai_b200', 'csrc', 'full_obs.cuh')]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not (os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS)):
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
        L.rg_render_grid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.fo_full_obs.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _lib = L
    return _lib


class FullObsHostPool(render_grid_host.RenderHostPool):
    """RenderHostPool on the library that also holds k_full_obs's per-env source"""

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

    def full_obs_env(self, i, offset=0):
        """FullyObsWrapper image of env i through k_full_obs's per-env source, stored `offset` bytes past an aligned address"""
        buf = np.zeros(self.width * self.height * 3 + 32, np.uint8)
        base = (-buf.ctypes.data) % 16 + offset
        self.L.fo_full_obs(self.h, i, C.c_void_p(buf.ctypes.data + base))
        rest = np.concatenate([buf[:base], buf[base + self.width * self.height * 3:]])
        assert not rest.any(), 'a byte outside the frame was written'
        return buf[base:base + self.width * self.height * 3].reshape(self.width, self.height, 3)
