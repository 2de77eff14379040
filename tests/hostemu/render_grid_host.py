"""TEST-ONLY host build of the full-grid frame path (render_grid_host.cpp: hostemu.cpp + csrc/grid_render.cuh compiled with
g++): a HostEmuPool that can also render MiniGridEnv.render('rgb_array') frames of its envs, and the host rasteriser's table.
Never imported by babyai_b200/."""
import ctypes as C
import os

import numpy as np

import hostemu
from hostemu import HERE, ROOT, _compile, _p

SRC = os.path.join(HERE, 'render_grid_host.cpp')
OUT = os.path.join(HERE, 'librender_grid_host.so')
DEPS = [SRC, hostemu.SRC] + hostemu.DEPS[1:] + [os.path.join(ROOT, 'babyai_b200', 'csrc', 'grid_render.cuh'),
                                               os.path.join(ROOT, 'babyai_b200', 'csrc', 'rgb_tiles.h')]
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
        L.rg_grid_tiles.argtypes = [C.c_int, C.c_void_p]
        L.rg_grid_cell_index.argtypes = [C.c_int]
        _lib = L
    return _lib


class RenderHostPool(hostemu.HostEmuPool):
    """HostEmuPool on the library that also holds k_render_grid's per-env source"""

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

    def render_grid(self, i, tile_size=32, highlight=True):
        """MiniGridEnv.render('rgb_array') of env i's current state through k_render_grid's per-env source"""
        out = np.zeros((self.height * tile_size, self.width * tile_size, 3), np.uint8)
        self.L.rg_render_grid(self.h, i, tile_size, int(bool(highlight)), _p(out))
        return out


def grid_tiles(tile_size):
    """the host build's full-grid tile table: uint8[2, 5, 43, ts, ts, 3] (rgb_tiles.h render_grid_tiles)"""
    t = np.zeros((2, 5, 43, tile_size, tile_size, 3), np.uint8)
    lib().rg_grid_tiles(tile_size, _p(t))
    return t


def grid_cell_index(b):
    return lib().rg_grid_cell_index(b)
