"""tests/golden/full_obs/full_obs.npz: fully observable observations (gym_minigrid 1.0.x FullyObsWrapper, restated in
tests/full_obs_common.py over the oracle shim's gym) of the reference's own levels, run with the Philox back-end: per level one
seed, one random action stream and the image after every action (an episode that ends is reset at once, as ParallelEnv
does).  The levels include the non-square KeyCorridorS3R1 and MoveTwoAcrossS5N2 and PutNextS5N2Carrying, whose episodes start
carrying.  Build container only (needs the reference tree).

usage: python tests/golden/make_full_obs_golden.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..', 'oracle'))
sys.path.insert(0, os.path.join(HERE, '..'))
import refenv  # noqa: E402
from full_obs_common import P_RANDOM, wrappers  # noqa: E402

LEVELS = [('GoToLocal', 13, 120), ('BossLevel', 23, 150), ('Unlock', 33, 150), ('KeyCorridorS3R1', 43, 120),
          ('MoveTwoAcrossS5N2', 53, 120), ('PutNextS5N2Carrying', 63, 120), ('OpenDoorsOrderN4', 73, 120)]


def main():
    refenv.setup('philox')
    FullyObsWrapper, _ = wrappers()
    rng = np.random.RandomState(9)
    actions, images, dims = [], [], []
    for level, seed, T in LEVELS:
        env = FullyObsWrapper(refenv.make_env(level, seed, 'philox'))
        imgs = [env.reset()['image'].copy()]
        acts = []
        for _ in range(T):
            a = int(rng.choice(7, p=P_RANDOM))
            acts.append(a)
            obs, _r, done, _ = env.step(a)
            if done:
                obs = env.reset()
            imgs.append(obs['image'].copy())
        actions.append(acts)
        images.append(np.stack(imgs))
        dims.append(imgs[0].shape[:2])
    A = np.full((len(LEVELS), max(len(a) for a in actions)), -1, np.int8)
    for i, a in enumerate(actions):
        A[i, :len(a)] = a
    sizes = [im.size for im in images]
    out = os.path.join(HERE, 'full_obs', 'full_obs.npz')
    np.savez_compressed(out, levels=json.dumps([l[0] for l in LEVELS]), seeds=np.array([l[1] for l in LEVELS], np.uint64),
                        actions=A, dims=np.array(dims, np.int32), offsets=np.concatenate([[0], np.cumsum(sizes)]),
                        images=np.concatenate([im.reshape(-1) for im in images]))
    print('%d images of %d levels -> %s (%d KB)' % (sum(len(im) for im in images), len(LEVELS), out, os.path.getsize(out) // 1024))


if __name__ == '__main__':
    main()
