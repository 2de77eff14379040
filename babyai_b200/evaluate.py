"""`batch_evaluate` (babyai/evaluate.py:85-140) as a stream: one pool of `num_envs` envs in freeze mode, and every env that
finishes an episode starts the next unused seed at once (BabyAIVecEnv.reset_envs) instead of idling until the slowest episode
of its wave has ended.

The seed set, the logs and their order are the reference's: `ceil(episodes / num_envs) * num_envs` seeds from `seed`, one
entry per seed in seed order.  For an agent whose action for an env depends only on that env's observations since its reset
(ModelAgent: `analyze_feedback` zeroes an env's memory row when it reports done), the logs equal a wave evaluation of the same
seeds.  Rebinding `babyai.evaluate.batch_evaluate = babyai_b200.evaluate.batch_evaluate` is all a caller changes
(INTEGRATION.md section 2).
"""
import numpy as np

from .learner import DeviceManyEnvs
from .vecenv import EnvList


def batch_evaluate(agent, env_name, seed, episodes, return_obss_actions=False, pixel=False, num_envs=256, pool=None):
    """agent: `act_batch(many_obs)['action']` and `analyze_feedback(reward, done)`, as the reference calls them.
    env_name: 'BabyAI-<Level>-v0' or '<Level>'.  `pool` is a test hook (an object with BabyAIVecEnv's tensor interface,
    reset_envs included, in freeze mode); the product builds the CUDA pool."""
    level = env_name[len('BabyAI-'):-len('-v0')] if env_name.startswith('BabyAI-') and env_name.endswith('-v0') else env_name
    num_envs = min(num_envs, episodes)
    n_seeds = (episodes + num_envs - 1) // num_envs * num_envs
    env = DeviceManyEnvs(EnvList(level, range(seed, seed + num_envs), pixel=pixel), pool=pool)
    many_obs = env.reset()

    frames = np.zeros(n_seeds, dtype='int64')              # per seed (index: seed - `seed`)
    returns = np.zeros(n_seeds)
    obss = [[] for _ in range(n_seeds)] if return_obss_actions else None
    actions = [[] for _ in range(n_seeds)] if return_obss_actions else None
    episode = np.arange(num_envs)                          # the seed index each env is playing
    steps = np.zeros(num_envs, dtype='int64')              # its steps in that episode
    active = np.ones(num_envs, dtype='bool')
    next_seed = num_envs
    while active.any():
        action = agent.act_batch(many_obs)['action']
        if return_obss_actions:
            for i in np.nonzero(active)[0]:
                obss[episode[i]].append(many_obs[i])
                actions[episode[i]].append(action[i].item())
        many_obs, reward, done, _ = env.step(action)
        agent.analyze_feedback(reward, done)
        done = np.array(done, dtype='bool')
        steps[active] += 1
        just_done = np.nonzero(done & active)[0]
        if len(just_done) == 0:
            continue
        frames[episode[just_done]] = steps[just_done]
        returns[episode[just_done]] = np.asarray(reward, dtype='float64')[just_done]
        active[just_done] = False
        # the envs that just finished take the next seeds, in env order; once the seeds run out they stay frozen
        k = min(len(just_done), n_seeds - next_seed)
        if k > 0:
            ids = just_done[:k]
            many_obs = env.reset_envs(ids, [seed + s for s in range(next_seed, next_seed + k)], many_obs)
            episode[ids] = np.arange(next_seed, next_seed + k)
            steps[ids] = 0
            active[ids] = True
            next_seed += k

    logs = {
        "num_frames_per_episode": list(frames),
        "return_per_episode": list(returns),
        "observations_per_episode": obss if return_obss_actions else [],
        "actions_per_episode": actions if return_obss_actions else [],
        "seed_per_episode": list(range(seed, seed + n_seeds)),
    }
    return logs
