"""Full-grid frames (MiniGridEnv.render('rgb_array'), scripts/manual_control.py:14) without a GPU: the full-grid tile table
(csrc/rgb_tiles.h) against the oracle shim's literal restatement of gym_minigrid's rasteriser, the kernel's per-env source
(csrc/grid_render.cuh, compiled for the host by tests/hostemu/render_grid_host.cpp) against the golden frames of the
reference's levels, and the built library's k_render_grid in sm_90a SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from render_grid_common import CELL_BYTES, CELL_INDEX, assemble, frame_of, load_golden, matches, obs_highlight, pool_grid_tiles, shim_render

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


def _shim():
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'shim'))
    from gym_minigrid.minigrid import Grid, _decode_obj
    return Grid, _decode_obj


@pytest.mark.parametrize('ts', [8, 16, 32, 7])
def test_grid_tiles_equal_shim_rasteriser(ts):
    """every tile of the table: 43 cell bytes x agent {none, 0..3} x highlight, exhaustive"""
    Grid, _decode_obj = _shim()
    tiles = pool_grid_tiles(ts)
    for k, b in enumerate(CELL_BYTES):
        t, c, s = b & 7, (b >> 3) & 7, b >> 6
        obj = _decode_obj(t, c, s) if t >= 2 else None
        for agent in range(5):
            for hl in (0, 1):
                want = Grid.render_tile(obj, agent_dir=None if agent == 0 else agent - 1, highlight=bool(hl), tile_size=ts)
                assert np.array_equal(tiles[hl, agent, k], want.astype(np.uint8)), (ts, b, agent, hl)


def test_grid_tiles_layout_and_sizes():
    from babyai_b200 import lib
    import render_grid_host as rgh
    L = lib.load()
    assert [rgh.grid_cell_index(b) for b in CELL_BYTES] == list(range(43))
    assert all(rgh.grid_cell_index(b) == 0 for b in range(256) if CELL_INDEX[b] < 0)
    for ts in (1, 64):
        t = np.zeros((2, 5, 43, ts, ts, 3), np.uint8)
        assert L.bb_grid_tiles(ts, t.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(t, rgh.grid_tiles(ts))
    buf = np.zeros(2 * 5 * 43 * 65 * 65 * 3, np.uint8)
    for ts in (0, -1, 65):
        assert L.bb_grid_tiles(ts, buf.ctypes.data_as(C.c_void_p)) != 0
    assert not buf.any()


def _host_pool(level, seed):
    from render_grid_host import RenderHostPool
    from babyai_b200.levels import level_spec
    return RenderHostPool(level_spec(level), 1, seeds=[seed])


def test_host_build_replays_golden_frames():
    """tests/golden/rgb_grid.npz (make_rgb_grid_golden.py): the reference's levels rendered by the shim after chosen steps;
    the host build replays the actions and its frames are equal, and so is the numpy assembly from the state and the
    highlight of the current observation"""
    gold = load_golden()
    n = 0
    for g in gold:
        pool = _host_pool(g['level'], g['seed'])
        obs = pool.reset().copy()
        t = 0
        for step, ts, hl, _door, want in g['frames']:
            while t < step:
                obs = pool.step(g['actions'][t:t + 1])[0].copy()
                t += 1
            got = pool.render_grid(0, ts, hl)
            assert np.array_equal(got, want), (g['level'], step, ts, hl)
            assert matches(want, frame_of(pool, 0, obs[0], ts, hl, g['level'])), (g['level'], step, ts, hl)
            n += 1
    assert n >= 60 and {f[1] for g in gold for f in g['frames']} == {7, 8, 32}
    assert any(f[3] for g in gold for f in g['frames'])


def _check_shim_env(env, pool, level, t, ts=8):
    """MiniGridEnv.render('rgb_array') on the shim == host-build frame; its highlight mask == the obs-visible cells through
    the pose"""
    want = shim_render(env, tile_size=ts)
    got = pool.render_grid(0, ts, True)
    assert np.array_equal(got, want), (level, t)
    obs = env.gen_obs()['image']
    x, y = int(env.agent_pos[0]), int(env.agent_pos[1])
    mask = obs_highlight(obs, x, y, int(env.agent_dir), env.width, env.height)
    enc = env.grid.encode().astype(np.int64)                        # [W, H, 3], empty cells as (1, 0, 0)
    grid = (enc[..., 0] | (enc[..., 1] << 3) | (enc[..., 2] << 6)).T.astype(np.uint8)
    assert np.array_equal(assemble(grid, x, y, int(env.agent_dir), mask, ts), want), (level, t)


@pytest.mark.reference
def test_reference_levels_render_like_the_host_build():
    """the reference's own levels on the shim (Philox back-end): the golden list for 150 random steps, then every served
    level for a few steps at tile size 8"""
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    import refenv
    from babyai_b200.levels import LEVELS
    refenv.setup('philox')
    rng = np.random.RandomState(3)
    golden = [g['level'] for g in load_golden()]
    for level in golden + sorted(set(LEVELS) - set(golden)):
        steps = 150 if level in golden else 6
        seed = 1000 + len(level)
        env = refenv.make_env(level, seed, 'philox')
        env.reset()
        pool = _host_pool(level, seed)
        pool.reset()
        _check_shim_env(env, pool, level, 0)
        for t in range(steps):
            a = int(rng.choice(7, p=[0.2, 0.2, 0.3, 0.08, 0.07, 0.15, 0.0]))
            _o, _r, done, _ = env.step(a)
            if done:
                env.reset()
            pool.step(np.array([a], np.int8))
            if level not in golden or t % 5 == 0:
                _check_shim_env(env, pool, level, t + 1)


def test_sass_has_k_render_grid_without_local_memory():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not available')
    from babyai_b200 import build as b
    lib = b.build()
    out = subprocess.run([exe, '-sass', '-fun', 'k_render_grid', lib], capture_output=True, text=True, timeout=300).stdout
    if 'k_render_grid' not in out:            # older cuobjdump: no -fun filtering by a partial name
        out = subprocess.run([exe, '-sass', lib], capture_output=True, text=True, timeout=300).stdout
    assert 'sm_90a' in out
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = fns.setdefault(m.group(1), []) if 'k_render_grid' in m.group(1) else None
        elif cur is not None and re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+\S', line):
            cur.append(line)
    assert len(fns) == 10, sorted(fns)             # store widths 16 / 8 / 4 / 2 / 1 x (all envs, an id list)
    for name, code in fns.items():
        assert code, name
        assert not any(re.search(r'\b(LDL|STL)\b', i) for i in code), name
        assert any('STG' in i for i in code) and any(re.search(r'\bLDG\b', i) for i in code), name
