"""The per-environment `gym.Env` surface of the reference (SURVEY.md 8b, row "Per-env gym.Env"):
`gym.make('BabyAI-GoToLocal-v0')`, `env.seed(int)`, `reset()`, `step(action)`, `.observation_space`,
`.action_space`, `.actions` -- what `imitation.py:84,114`, `scripts/enjoy.py:35-44,86` and
`scripts/manual_control.py:52-73` hold on to.  One environment is a pool of one: the same kernels, the same
level stream for a seed as env i of a big pool seeded with it.  It exists for API completeness (scripts that
look at a single env); throughput comes from the pooled facades in vecenv.py / learner.py.

    env = babyai_b200.gymapi.make('BabyAI-GoToLocal-v0'); env.seed(7); obs = env.reset()
    obs, reward, done, info = env.step(env.actions.forward)

`register_levels()` registers the served `BabyAI-<Level>-v0` ids (levelgen.py:481-486) with whatever `gym` is
importable, entry points pointing here, so `gym.make(id)` returns these objects.
"""
import os
from enum import IntEnum

import numpy as np

from .levels import LEVELS
from .vecenv import EnvList, ManyEnvs, _spaces, grid_dims


class Actions(IntEnum):
    """MiniGridEnv.Actions (scripts/enjoy.py:35-44, utils/agent.py:89)"""
    left = 0
    right = 1
    forward = 2
    pickup = 3
    drop = 4
    toggle = 5
    done = 6


class Grid(object):
    """MiniGridEnv.grid as far as gym_minigrid's FullyObsWrapper reads it (wrappers.py): `encode()` of the env's current
    state, made on the device by bb_pool_full_obs."""

    def __init__(self, env):
        self._env = env
        self.width, self.height = env.width, env.height

    def encode(self, vis_mask=None):
        """Grid.encode(): uint8[W, H, 3] of (type, color, state) per cell, x-major; the agent is not part of the grid"""
        if vis_mask is not None:
            raise NotImplementedError('Grid.encode(vis_mask): the pool encodes whole grids')
        pool = self._env._vec.pool
        img = pool.full_obs([0])[0].cpu().numpy()
        grid, s = pool.state(0)
        x, y = s['agent_x'], s['agent_y']
        b = int(grid[y, x])                               # what the agent stands on: empty, or an open door
        img[x, y] = (b & 7, (b >> 3) & 7, b >> 6)
        return img


def _level_of(name):
    if name.startswith('BabyAI-') and name.endswith('-v0'):
        name = name[len('BabyAI-'):-len('-v0')]
    if name not in LEVELS:
        raise KeyError('level %r is not served by the pool' % name)
    return name


class SingleEnv(object):
    """gym.Env-shaped view of a one-environment pool.  Like a gym env it does NOT reset itself: after `done`
    further steps repeat the terminal result until reset() (the pool's freeze mode, evaluate.py:72-78)."""
    Actions = Actions
    metadata = {'render.modes': ['rgb_array']}
    reward_range = (0, 1)

    def __init__(self, level, seed=None, device=0, pool=None):
        self.level_name = _level_of(level)
        self.gym_id = 'BabyAI-%s-v0' % self.level_name           # levelgen.py:481,492-493
        self.actions = Actions
        self.observation_space, self.action_space = _spaces()
        self.spec = None
        if seed is None:                                          # gym seeding with None: entropy from the OS
            seed = int.from_bytes(os.urandom(4), 'little')
        self._vec = ManyEnvs(EnvList(self.level_name, [seed], device), pool=pool)
        self.mission = None
        self.width, self.height = grid_dims([(self.level_name, 1)])     # MiniGridEnv.width / height
        self.grid = Grid(self)

    @property
    def unwrapped(self):
        return self

    def seed(self, seed=None):
        if seed is None:
            seed = int.from_bytes(os.urandom(4), 'little')
        self._vec.seed([int(seed)])
        return [int(seed)]

    def reset(self):
        obs = self._vec.reset()[0]
        self.mission = obs['mission']
        return obs

    def step(self, action):
        obs, reward, done, info = self._vec.step([int(action)])
        return obs[0], reward[0], done[0], info[0]

    def render(self, mode='human', close=False, highlight=True, tile_size=32):
        """MiniGridEnv.render: 'rgb_array' returns the full grid as numpy uint8[H * tile_size, W * tile_size, 3] (drawn on the
        device by bb_pool_render_grid); there is no window, so 'human' raises."""
        if close:
            return None
        if mode != 'rgb_array':
            raise NotImplementedError("render(%r): the pool has no window; use render('rgb_array')" % (mode,))
        pool = self._vec.pool
        if not hasattr(pool, 'render_grid'):
            raise NotImplementedError('this pool cannot render')
        return pool.render_grid(None, tile_size=tile_size, highlight=highlight)[0].cpu().numpy()

    def _state(self):
        return self._vec.pool.state(0)[1]

    @property
    def step_count(self):
        """steps taken in the current episode (MiniGridEnv.step_count)"""
        return self._state()['step_count']

    @property
    def agent_pos(self):
        s = self._state()
        return np.array((s['agent_x'], s['agent_y']))

    @property
    def agent_dir(self):
        return self._state()['agent_dir']

    def close(self):
        self._vec.pool.close() if hasattr(self._vec.pool, 'close') else None


def make(name, **kwargs):
    """gym.make for the served ids: 'BabyAI-GoToLocal-v0' or 'GoToLocal'."""
    return SingleEnv(name, **kwargs)


def register_levels(gym=None):
    """Register every served level as BabyAI-<Level>-v0 with `gym` (default: the importable one).  Returns the ids."""
    if gym is None:
        import gym
    import functools
    ids = []
    for level in sorted(LEVELS):
        gid = 'BabyAI-%s-v0' % level
        gym.envs.registration.register(id=gid, entry_point=functools.partial(SingleEnv, level))
        ids.append(gid)
    return ids
