"""Shared helpers of the full-grid frame tests (MiniGridEnv.render('rgb_array'), k_render_grid): the table layout of
bb_grid_tiles, the numpy statement of a frame from an env's state and observation, the restatement of MiniGridEnv.render
for envs of the oracle shim, and the golden fixture."""
import ctypes as C
import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'rgb_grid.npz')

# the 43 cell bytes a BabyAI grid holds, in the table's cell-index order (include/babyai_b200.h, bb_grid_tiles)
CELL_BYTES = ([1] + [t | (c << 3) for t in (2, 5, 6, 7) for c in range(6)] +
              [4 | (c << 3) | (s << 6) for s in range(3) for c in range(6)])
CELL_INDEX = np.full(256, -1, np.int64)
CELL_INDEX[CELL_BYTES] = np.arange(len(CELL_BYTES))
DIR_TO_VEC = [(1, 0), (0, 1), (-1, 0), (0, -1)]

_tiles = {}


def pool_grid_tiles(ts):
    """bb_grid_tiles(ts): uint8[2 highlight, 5 agent, 43 cells, ts, ts, 3] (host rasteriser, no GPU)"""
    if ts not in _tiles:
        from babyai_b200 import lib
        t = np.zeros((2, 5, 43, ts, ts, 3), np.uint8)
        assert lib.load().bb_grid_tiles(ts, t.ctypes.data_as(C.c_void_p)) == 0
        _tiles[ts] = t
    return _tiles[ts]


def obs_highlight(obs, x, y, d, width, height):
    """the highlight mask [height, width] of a pose: the view cells of the observation with type != 0 mapped to the world
    (agent_pos + f (6 - vj) + r (vi - 3)), in-bounds cells only"""
    fx, fy = DIR_TO_VEC[d]
    rx, ry = -fy, fx
    m = np.zeros((height, width), bool)
    obs = np.asarray(obs).reshape(7, 7, 3)
    for vi in range(7):
        for vj in range(7):
            if obs[vi, vj, 0] != 0:
                wx, wy = x + fx * (6 - vj) + rx * (vi - 3), y + fy * (6 - vj) + ry * (vi - 3)
                if 0 <= wx < width and 0 <= wy < height:
                    m[wy, wx] = True
    return m


def assemble(grid, x, y, d, mask, ts, highlight=True):
    """numpy statement of a frame: grid uint8[H, W] cell bytes, agent at (x, y) facing d, mask [H, W] -> uint8[H ts, W ts, 3]"""
    H, W = grid.shape
    agent = np.zeros((H, W), np.int64)
    agent[y, x] = 1 + d
    cells = CELL_INDEX[grid]
    assert (cells >= 0).all(), 'a cell byte outside the 43 of a BabyAI grid'
    hl = mask.astype(np.int64) if highlight else np.zeros((H, W), np.int64)
    t = pool_grid_tiles(ts)[hl, agent, cells]                      # [H, W, ts, ts, 3]
    return t.transpose(0, 2, 1, 3, 4).reshape(H * ts, W * ts, 3)


def frame_of(pool, i, obs, ts, highlight=True, level=''):
    """what render_grid must return for env i of a pool (CUDA or host build): its state + the highlight of its observation.
    On PutNext*Carrying levels a state with step_count 0 still holds the object the agent starts carrying on the grid (the
    pool takes it at the first step, the reference right after reset): then the frames with one key / ball / box drawn as
    empty are returned, one of which must match."""
    grid, info = pool.state(i)
    H, W = grid.shape
    x, y, d = info['agent_x'], info['agent_y'], info['agent_dir']
    mask = obs_highlight(obs, x, y, d, W, H)
    if level.endswith('Carrying') and info['step_count'] == 0:
        out = []
        for c in np.nonzero(np.isin(grid.reshape(-1) & 7, (5, 6, 7)))[0]:
            g = grid.copy().reshape(-1)
            g[c] = 1
            out.append(assemble(g.reshape(H, W), x, y, d, mask, ts, highlight))
        return out
    return [assemble(grid, x, y, d, mask, ts, highlight)]


def matches(frame, candidates):
    return any(np.array_equal(frame, c) for c in candidates)


def shim_render(env, highlight=True, tile_size=32):
    """gym_minigrid 1.0.x MiniGridEnv.render(mode='rgb_array', highlight, tile_size), restated for an env running on the
    oracle shim (whose own render() only raises): gen_obs_grid()'s vis_mask mapped back to the world through the pose, then
    Grid.render of the whole grid with the agent on top"""
    _, vis_mask = env.gen_obs_grid()
    f_vec = env.dir_vec
    r_vec = env.right_vec
    top_left = env.agent_pos + f_vec * (env.agent_view_size - 1) - r_vec * (env.agent_view_size // 2)
    highlight_mask = np.zeros(shape=(env.width, env.height), dtype=bool)
    for vis_j in range(0, env.agent_view_size):
        for vis_i in range(0, env.agent_view_size):
            if not vis_mask[vis_i, vis_j]:
                continue
            abs_i, abs_j = top_left - (f_vec * vis_j) + (r_vec * vis_i)
            if abs_i < 0 or abs_i >= env.width:
                continue
            if abs_j < 0 or abs_j >= env.height:
                continue
            highlight_mask[abs_i, abs_j] = True
    return env.grid.render(tile_size, env.agent_pos, env.agent_dir, highlight_mask=highlight_mask if highlight else None)


def load_golden():
    """tests/golden/rgb_grid.npz (make_rgb_grid_golden.py) -> list of dict(level, seed, actions, frames=[(step, ts,
    highlight, doorway, pixels)]); step = actions applied since the first reset"""
    z = np.load(GOLD)
    levels = json.loads(str(z['levels']))
    off, px = z['offsets'], z['pixels']
    out = []
    for li, level in enumerate(levels):
        a = z['actions'][li]
        out.append(dict(level=level, seed=int(z['seeds'][li]), actions=a[a >= 0].astype(np.int8), frames=[]))
    for k, (li, step, ts, hl, door, h, w) in enumerate(z['frames']):
        out[li]['frames'].append((int(step), int(ts), bool(hl), bool(door), px[off[k]:off[k + 1]].reshape(h, w, 3)))
    return out
