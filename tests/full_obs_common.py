"""Shared helpers of the fully observable observation tests (bb_pool_full_obs, FullyObsWrapper / RGBImgObsWrapper): the two
gym_minigrid 1.0.x wrappers restated over the oracle shim's gym, the numpy statement of a full observation from a pool's state,
a CPU-tensor pool over the host build for the facades, and the golden fixture."""
import json
import os

import numpy as np
import torch

# in a directory of its own: the top level of tests/golden holds one trace file per level (common.GOLDEN_LEVELS)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'full_obs', 'full_obs.npz')

# 7 ICLR levels (doors open / closed / locked, Unlock's untracked carry) and 5 bonus levels, two of them on non-square grids
ICLR_LEVELS = ['GoToLocal', 'BossLevel', 'Unlock', 'Open', 'GoToImpUnlock', 'PickupLoc', 'SynthSeq']
BONUS_LEVELS = ['PutNextS5N2Carrying', 'KeyCorridorS3R1', 'MoveTwoAcrossS5N2', 'KeyInBox', 'OpenDoorsOrderN4']
P_RANDOM = [0.2, 0.2, 0.3, 0.08, 0.07, 0.15, 0.0]


def wrappers():
    """gym_minigrid 1.0.x FullyObsWrapper and RGBImgObsWrapper (wrappers.py), restated over whichever `gym` is importable (the
    oracle shim's in these tests)"""
    import gym
    from gym import spaces

    class FullyObsWrapper(gym.ObservationWrapper):
        def __init__(self, env):
            super().__init__(env)
            self.observation_space.spaces['image'] = spaces.Box(
                low=0, high=255, shape=(self.env.width, self.env.height, 3), dtype='uint8')

        def observation(self, obs):
            env = self.unwrapped
            full_grid = env.grid.encode()
            full_grid[env.agent_pos[0]][env.agent_pos[1]] = np.array([10, 0, env.agent_dir])   # 'agent', 'red', agent_dir
            return {'mission': obs['mission'], 'image': full_grid}

    class RGBImgObsWrapper(gym.ObservationWrapper):
        def __init__(self, env, tile_size=8):
            super().__init__(env)
            self.tile_size = tile_size
            self.observation_space.spaces['image'] = spaces.Box(
                low=0, high=255, shape=(self.env.width * tile_size, self.env.height * tile_size, 3), dtype='uint8')

        def observation(self, obs):
            env = self.unwrapped
            rgb_img = env.render(mode='rgb_array', highlight=False, tile_size=self.tile_size)
            return {'mission': obs['mission'], 'image': rgb_img}

    return FullyObsWrapper, RGBImgObsWrapper


def shim_renderable(env):
    """a reference env on the shim, given MiniGridEnv.render('rgb_array') (render_grid_common.shim_render; the shim's raises)"""
    from render_grid_common import shim_render
    u = env.unwrapped
    u.render = lambda mode='human', close=False, highlight=True, tile_size=32: shim_render(u, highlight, tile_size)
    return env


def encode(grid, x, y, d):
    """numpy statement: cell bytes [H, W] with the agent at (x, y) facing d -> FullyObsWrapper image uint8[W, H, 3]"""
    g = np.asarray(grid).T
    img = np.stack([g & 7, (g >> 3) & 7, g >> 6], -1).astype(np.uint8)
    img[x, y] = (10, 0, d)
    return img


def expected(pool, i, level=''):
    """what full_obs must return for env i of a pool with a state() (oracle, host build, CUDA pool).  On PutNext*Carrying
    levels a state at step 0 still holds the object the agent starts carrying on the grid: then the images with one key /
    ball / box read as empty are returned, one of which must match."""
    grid, s = pool.state(i)
    x, y, d = s['agent_x'], s['agent_y'], s['agent_dir']
    if level.endswith('Carrying') and s['step_count'] == 0:
        out = []
        for c in np.nonzero(np.isin(grid.reshape(-1) & 7, (5, 6, 7)))[0]:
            g = grid.copy().reshape(-1)
            g[c] = 1
            out.append(encode(g.reshape(grid.shape), x, y, d))
        return out
    return [encode(grid, x, y, d)]


def matches(img, candidates):
    return any(np.array_equal(img, c) for c in candidates)


class FullTensorPool(object):
    """BabyAIVecEnv's tensor and host-buffer interfaces over the host build (tests/hostemu/full_obs_host.py), CPU tensors
    standing in for device memory: what the facades need in every observation mode"""

    def __init__(self, level, seeds, mode=0):
        from babyai_b200.levels import level_spec
        from full_obs_host import FullObsHostPool
        n = len(seeds)
        self.emu = FullObsHostPool(level_spec(level), n, np.asarray(seeds, dtype=np.uint64), mode)
        self.num_envs, self.width, self.height = n, self.emu.width, self.emu.height
        self.device = torch.device('cpu')
        self.mission_tokens = torch.zeros((n, 72), dtype=torch.int16)
        self.direction = torch.zeros(n, dtype=torch.int8)

    def _tokens(self, idx):
        for i in idx:
            self.mission_tokens[i] = torch.from_numpy(self.emu.tokens(int(i)))

    def seed(self, seeds):
        self.emu.seed(np.asarray(list(seeds), dtype=np.uint64))

    def reset(self, obs=None, direction=None):
        obs.copy_(torch.from_numpy(self.emu.reset()))
        self.direction.copy_(torch.from_numpy(self.emu.direction))
        self._tokens(range(self.num_envs))
        return obs

    def step(self, actions, obs=None, reward=None, done=None, direction=None):
        o, r, d = self.emu.step(actions.numpy())
        obs.copy_(torch.from_numpy(o))
        self.direction.copy_(torch.from_numpy(self.emu.direction))
        self._tokens(np.nonzero(d)[0])
        return obs, torch.from_numpy(r.copy()), torch.from_numpy(d.copy())

    def step_learner(self, actions, obs, reward, done, direction=None):
        o, r, d = self.emu.step(actions)
        obs.copy_(torch.from_numpy(o))
        reward[...], done[...] = r, d
        self.direction.copy_(torch.from_numpy(self.emu.direction))
        if direction is not None:
            direction.copy_(self.direction)
        self._tokens(np.nonzero(d)[0])

    def reset_host(self, obs, direction):
        obs[...] = self.emu.reset()
        direction[...] = self.emu.direction

    def step_host(self, actions, obs, reward, done, direction):
        o, r, d = self.emu.step(np.asarray(actions, dtype=np.int8))
        obs[...], reward[...], done[...], direction[...] = o, r, d, self.emu.direction

    def missions(self, idx=None):
        from babyai_b200.levels import detokenize
        return [detokenize(self.emu.tokens(int(i))) for i in (range(self.num_envs) if idx is None else idx)]

    def state(self, i):
        return self.emu.state(i)

    def full_obs(self, env_ids=None):
        ids = range(self.num_envs) if env_ids is None else env_ids
        return torch.from_numpy(np.stack([self.emu.full_obs_env(int(i), int(i) % 4) for i in ids]))

    def render_grid(self, env_ids=None, tile_size=32, highlight=True):
        ids = range(self.num_envs) if env_ids is None else env_ids
        return torch.from_numpy(np.stack([self.emu.render_grid(int(i), tile_size, highlight) for i in ids]))


def load_golden():
    """tests/golden/full_obs/full_obs.npz (make_full_obs_golden.py) -> list of dict(level, seed, actions, images [T + 1, W, H, 3]);
    images[t] is the FullyObsWrapper image after t actions (an episode that ends is reset at once, as ParallelEnv does)"""
    z = np.load(GOLD)
    levels = json.loads(str(z['levels']))
    out = []
    for li, level in enumerate(levels):
        a = z['actions'][li]
        a = a[a >= 0].astype(np.int8)
        w, h = (int(v) for v in z['dims'][li])
        img = z['images'][z['offsets'][li]:z['offsets'][li + 1]].reshape(len(a) + 1, w, h, 3)
        out.append(dict(level=level, seed=int(z['seeds'][li]), actions=a, images=img))
    return out
