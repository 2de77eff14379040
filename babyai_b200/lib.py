"""ctypes binding of libbabyai_b200.so (the C ABI in include/babyai_b200.h).

There is NO fallback: if the CUDA library has not been built, importing the
binding raises (build it with `python -m babyai_b200.build` or
`__graft_entry__.build()`); if no GPU is present, bb_pool_create fails and the
error is raised as RuntimeError."""
import ctypes as C
import os

from .levels import LevelSpec

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libbabyai_b200.so')

# every entry point include/babyai_b200.h declares
SYMBOLS = [
    'bb_pool_create', 'bb_pool_destroy', 'bb_pool_seed', 'bb_pool_set_mode', 'bb_pool_reset', 'bb_pool_reset_envs', 'bb_pool_step',
    'bb_pool_step_timed', 'bb_pool_rollout', 'bb_pool_rollout_timed', 'bb_pool_step_host', 'bb_pool_reset_host', 'bb_pool_step_learner', 'bb_pool_mission_tokens', 'bb_pool_render_rgb', 'bb_rgb_tiles', 'bb_pool_render_grid', 'bb_grid_tiles', 'bb_vocab_size',
    'bb_vocab_word', 'bb_pool_get_state', 'bb_pool_width', 'bb_pool_height', 'bb_pool_num_envs',
    'bb_pool_counters', 'bb_pool_launches', 'bb_last_error',
]

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError('%s is missing: the CUDA extension has not been built (python -m babyai_b200.build). '
                          'babyai_b200 has no CPU fallback.' % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.bb_pool_create.argtypes = [C.POINTER(LevelSpec), i32, i32, C.POINTER(vp)]
    L.bb_pool_destroy.argtypes = [vp]
    L.bb_pool_seed.argtypes = [vp, vp]
    L.bb_pool_set_mode.argtypes = [vp, i32]
    L.bb_pool_reset.argtypes = [vp, vp, vp, vp]
    L.bb_pool_reset_envs.argtypes = [vp, vp, vp, i32, vp, vp, vp]
    L.bb_pool_step.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.bb_pool_step_timed.argtypes = [vp, vp, i32, vp, vp, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.bb_pool_rollout.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.bb_pool_rollout_timed.argtypes = [vp, vp, i32, vp, vp, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.bb_pool_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    L.bb_pool_reset_host.argtypes = [vp, vp, vp]
    L.bb_pool_step_learner.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.bb_pool_render_rgb.argtypes = [vp, vp, vp, i32, vp]
    L.bb_rgb_tiles.argtypes = [vp]
    L.bb_pool_render_grid.argtypes = [vp, vp, i32, i32, i32, vp, vp]
    L.bb_grid_tiles.argtypes = [i32, vp]
    L.bb_pool_mission_tokens.argtypes = [vp, C.POINTER(vp), C.POINTER(i32)]
    L.bb_vocab_size.restype = i32
    L.bb_vocab_word.restype = C.c_char_p
    L.bb_vocab_word.argtypes = [i32]
    L.bb_pool_get_state.argtypes = [vp, i32, vp, vp]
    L.bb_pool_width.argtypes = [vp]
    L.bb_pool_height.argtypes = [vp]
    L.bb_pool_num_envs.argtypes = [vp]
    L.bb_pool_counters.argtypes = [vp, vp]
    L.bb_pool_launches.restype = i64
    L.bb_pool_launches.argtypes = [vp]
    L.bb_last_error.restype = C.c_char_p
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError('babyai_b200: ' + load().bb_last_error().decode())
