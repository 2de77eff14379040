"""k_render_grid on the GPU (bb_pool_render_grid, BabyAIVecEnv.render_grid, SingleEnv.render('rgb_array')): the golden frames
of the reference's levels through the per-step and the rollout paths, random id lists on large pools against the numpy
assembly of state + table + observation highlight, every served level, freeze / auto-reset, a call above 4 GiB, renders
that must not disturb the stepping, stream order, and argument checks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from render_grid_common import assemble, frame_of, load_golden, matches, obs_highlight, pool_grid_tiles

pytestmark = pytest.mark.gpu

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


def _check_frames(env, ids, frames, ts, highlight, level=''):
    obs = env.obs.cpu().numpy()
    for k, i in enumerate(ids):
        assert matches(frames[k], frame_of(env, int(i), obs[i], ts, highlight, level)), (level, k, int(i), ts, highlight)


def _replay_golden(rollout, monkeypatch, kernel=None):
    import torch
    from babyai_b200 import BabyAIVecEnv
    if kernel:
        monkeypatch.setenv('BB_ROLLOUT_KERNEL', kernel)
    n_frames = 0
    for g in load_golden():
        n = 3                                                     # three envs with the trace's seed: all three must match
        env = BabyAIVecEnv(g['level'], n, seeds=np.full(n, g['seed'], np.uint64))
        env.reset()
        acts = torch.as_tensor(np.repeat(g['actions'][:, None], n, 1), device=env.device)
        T = acts.shape[0]
        obs = torch.zeros((T, n, 7, 7, 3), dtype=torch.uint8, device=env.device)
        rew = torch.zeros((T, n), device=env.device)
        done = torch.zeros((T, n), dtype=torch.uint8, device=env.device)
        t = 0
        for step, ts, hl, _door, want in g['frames']:
            if step > t:
                if rollout:                                       # chunk ends at the frame steps
                    env.rollout(acts[t:step], obs[:step - t], rew[:step - t], done[:step - t])
                else:
                    for s in range(t, step):
                        env.step(acts[s])
                t = step
            got = env.render_grid([2, 0, 1], tile_size=ts, highlight=hl).cpu().numpy()
            for k in range(n):
                assert np.array_equal(got[k], want), (g['level'], step, ts, hl, k)
            n_frames += 1
        assert env.counters()['errors'] == 0
        env.close()
    assert n_frames >= 60


def test_golden_frames_per_step(monkeypatch):
    _replay_golden(False, monkeypatch)


@pytest.mark.parametrize('kernel', ['lane', 'cta'])
def test_golden_frames_rollout(monkeypatch, kernel):
    _replay_golden(True, monkeypatch, kernel)


@pytest.mark.parametrize('level,n', [('BossLevel', 1037), ('GoToLocal', 4133)])
def test_random_id_lists(level, n):
    import torch
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64) + 17)
    env.reset()
    rng = np.random.RandomState(n)
    for t in range(25):
        env.step(torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=env.device))
    H, W = env.height, env.width
    for ts, hl, m in ((8, True, 200), (8, False, 60), (32, True, 24), (7, True, 40), (7, False, 20)):
        ids = np.r_[rng.randint(0, n, m), 0, n - 1, rng.randint(0, n, 4)]
        ids = np.r_[ids, ids[:3]]                                 # repeats, unsorted, first and last env
        out = env.render_grid(ids, tile_size=ts, highlight=hl)
        assert out.shape == (len(ids), H * ts, W * ts, 3)
        _check_frames(env, ids, out.cpu().numpy(), ts, hl, level)
    empty = env.render_grid([], tile_size=8)
    assert empty.shape == (0, H * 8, W * 8, 3)
    every = env.render_grid(None, tile_size=8)
    assert torch.equal(every, env.render_grid(np.arange(n), tile_size=8))
    assert torch.equal(every, env.render_grid(torch.arange(n), tile_size=8))
    # more ids than one launch carries (4 096)
    ids = rng.randint(0, n, 5000)
    assert torch.equal(env.render_grid(ids, tile_size=8), every[torch.as_tensor(ids, device=env.device)])
    env.close()


def test_all_levels():
    import torch
    from babyai_b200 import BabyAIVecEnv
    from babyai_b200.levels import LEVELS
    assert len(LEVELS) == 97
    rng = np.random.RandomState(4)
    for level in sorted(LEVELS):
        n = 6
        env = BabyAIVecEnv(level, n, seeds=np.arange(n, dtype=np.uint64) + 300)
        env.reset()
        _check_frames(env, range(n), env.render_grid(tile_size=8).cpu().numpy(), 8, True, level)
        for t in range(4):
            env.step(torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=env.device))
        _check_frames(env, range(n), env.render_grid(tile_size=8).cpu().numpy(), 8, True, level)
        env.close()


def test_freeze_renders_terminal_state_autoreset_renders_new_episode():
    import torch
    from babyai_b200 import BabyAIVecEnv
    from babyai_b200.vecenv import MODE_FREEZE
    n = 256
    for mode in (0, MODE_FREEZE):
        env = BabyAIVecEnv('GoToRedBall', n, seeds=np.arange(n, dtype=np.uint64), mode=mode)
        env.reset()
        rng = np.random.RandomState(2)
        ended = np.zeros(n, bool)
        frozen = {}
        for t in range(80):
            _o, _r, d = env.step(torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=env.device))
            d = d.cpu().numpy().astype(bool)
            new = d & ~ended
            ended |= d
            frames = env.render_grid(tile_size=8).cpu().numpy()
            for i in np.nonzero(new)[0][:8]:
                _g, info = env.state(int(i))
                # auto-reset: the first state of the next episode; freeze: the terminal state, kept from then on
                assert (info['step_count'] == 0) == (mode == 0)
                assert matches(frames[i], frame_of(env, int(i), env.obs[i].cpu().numpy(), 8))
                if mode == MODE_FREEZE:
                    frozen[int(i)] = frames[i]
            for i, f in frozen.items():
                assert np.array_equal(frames[i], f)
        assert ended.sum() > 20
        env.close()


def test_one_call_above_4_gib():
    import torch
    from babyai_b200 import BabyAIVecEnv
    n, ts = 800, 64
    env = BabyAIVecEnv('BossLevel', n, seeds=np.arange(n, dtype=np.uint64) + 9)
    env.reset()
    env.step(torch.full((n,), 2, dtype=torch.int8, device=env.device))
    out = env.render_grid(tile_size=ts)
    frame = out[0].numel()
    assert out.numel() > 4 * 2 ** 30
    first_above = (4 * 2 ** 30) // frame
    sample = [0, 1, first_above - 1, first_above, first_above + 1, n - 1]
    _check_frames(env, sample, out[sample].cpu().numpy(), ts, True)
    del out
    env.close()


def test_renders_leave_stepping_unchanged():
    import torch
    from babyai_b200 import BabyAIVecEnv
    n = 512
    a = BabyAIVecEnv('GoTo', n, seeds=np.arange(n, dtype=np.uint64))
    b = BabyAIVecEnv('GoTo', n, seeds=np.arange(n, dtype=np.uint64))
    a.reset(), b.reset()
    rng = np.random.RandomState(8)
    for t in range(60):
        act = torch.as_tensor(rng.randint(0, 7, n), dtype=torch.int8, device=a.device)
        oa, ra, da = [x.clone() for x in a.step(act)]
        a.render_grid(rng.randint(0, n, 37), tile_size=(8, 32, 5)[t % 3], highlight=bool(t & 1))
        ob, rb, db = b.step(act)
        assert torch.equal(oa, ob) and torch.equal(ra.view(torch.int32), rb.view(torch.int32)) and torch.equal(da, db), t
        assert torch.equal(a.direction, b.direction), t
    assert a.counters() == b.counters()
    a.close(), b.close()


def test_stream_ordered_on_a_side_stream():
    import torch
    from babyai_b200 import BabyAIVecEnv
    n = 2048
    env = BabyAIVecEnv('BossLevel', n, seeds=np.arange(n, dtype=np.uint64) + 3)
    s = torch.cuda.Stream()
    rng = np.random.RandomState(6)
    acts = torch.as_tensor(rng.randint(0, 7, (30, n)), dtype=torch.int8, device=env.device)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        env.reset()
        for t in range(30):
            env.step(acts[t])
        out = env.render_grid(tile_size=16)              # queued behind the steps on s, no synchronisation in between
    s.synchronize()
    ids = np.r_[0, n - 1, rng.randint(0, n, 30)]
    _check_frames(env, ids, out.cpu().numpy()[ids], 16, True)
    env.close()


def test_bad_arguments_raise_without_a_launch():
    import torch
    from babyai_b200 import BabyAIVecEnv, lib
    n = 64
    env = BabyAIVecEnv('GoToLocal', n)
    env.reset()
    env.render_grid(tile_size=8)                         # tables of the sizes used below are built
    L0 = env.launches()
    H, W = env.height, env.width
    for kw in (dict(env_ids=[0, n]), dict(env_ids=[-1]), dict(env_ids=[[0, 1]]), dict(tile_size=0), dict(tile_size=65)):
        with pytest.raises(ValueError):
            env.render_grid(**kw)
    good = (2, H * 8, W * 8, 3)
    for out in (torch.empty((3,) + good[1:], dtype=torch.uint8, device='cuda'), torch.empty(good, dtype=torch.int16, device='cuda'),
                torch.empty(good, dtype=torch.uint8), torch.empty((2, H * 8, W * 8 * 2, 3), dtype=torch.uint8, device='cuda')[:, :, ::2]):
        with pytest.raises(ValueError):
            env.render_grid([0, 1], tile_size=8, out=out)
    # the C ABI checks on its own
    L = lib.load()
    buf = torch.empty((n,) + good[1:], dtype=torch.uint8, device='cuda')
    ptr = C.c_void_p(buf.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ids = np.array([0, n], np.int32)
    assert L.bb_pool_render_grid(env.h, ids.ctypes.data_as(C.c_void_p), 2, 8, 1, ptr, st) != 0
    ids = np.array([-1, 0], np.int32)
    assert L.bb_pool_render_grid(env.h, ids.ctypes.data_as(C.c_void_p), 2, 8, 1, ptr, st) != 0
    assert L.bb_pool_render_grid(env.h, None, n - 1, 8, 1, ptr, st) != 0
    for ts in (0, 65):
        assert L.bb_pool_render_grid(env.h, None, n, ts, 1, ptr, st) != 0
    assert L.bb_pool_render_grid(env.h, None, n, 8, 1, C.c_void_p(buf.data_ptr() + 1), st) != 0
    assert env.launches() == L0
    out = env.render_grid([0, 1], tile_size=8)
    assert env.launches() == L0 + 1
    _check_frames(env, [0, 1], out.cpu().numpy(), 8, True)
    env.close()


def test_single_env_render_equals_shim_grid_render():
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'shim'))
    from gym_minigrid.minigrid import Grid, _decode_obj
    from babyai_b200 import gymapi
    env = gymapi.make('BabyAI-KeyCorridorS3R3-v0', seed=5)
    assert env.metadata['render.modes'] == ['rgb_array']
    obs = env.reset()
    rng = np.random.RandomState(0)
    steps = 0
    for t in range(40):
        grid, info = env._vec.pool.state(0)
        assert env.step_count == steps == info['step_count']
        assert tuple(env.agent_pos) == (info['agent_x'], info['agent_y']) and env.agent_dir == info['agent_dir']
        H, W = grid.shape
        g = Grid(W, H)
        for y in range(H):
            for x in range(W):
                b = int(grid[y, x])
                g.set(x, y, _decode_obj(b & 7, (b >> 3) & 7, b >> 6) if (b & 7) >= 2 else None)
        mask = obs_highlight(obs['image'], info['agent_x'], info['agent_y'], info['agent_dir'], W, H).T     # [x, y]
        for ts, hl in ((8, True), (5, False)):
            want = g.render(ts, np.array((info['agent_x'], info['agent_y'])), info['agent_dir'], highlight_mask=mask if hl else None)
            assert np.array_equal(env.render('rgb_array', highlight=hl, tile_size=ts), want), (t, ts)
        obs, _r, done, _ = env.step(int(rng.randint(0, 6)))
        steps += 1
        if done:
            obs = env.reset()
            steps = 0
    with pytest.raises(NotImplementedError):
        env.render()
    assert env.render(close=True) is None
    env.close()


def test_table_of_each_size_is_the_host_table():
    """the device table is bb_grid_tiles: a frame of every cell at tile sizes 1 and 64 through the kernel"""
    from babyai_b200 import BabyAIVecEnv
    env = BabyAIVecEnv('GoToLocal', 4, seeds=np.arange(4, dtype=np.uint64))
    env.reset()
    for ts in (1, 3, 12, 64):
        _check_frames(env, range(4), env.render_grid(tile_size=ts).cpu().numpy(), ts, True)
    assert pool_grid_tiles(1).shape == (2, 5, 43, 1, 1, 3)
    env.close()
