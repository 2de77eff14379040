"""tests/golden/rgb_grid.npz: full-grid frames (MiniGridEnv.render('rgb_array') of gym_minigrid 1.0.x, restated in
tests/render_grid_common.py over the oracle shim's Grid.render) of the reference's own levels, run with the Philox back-end: per level one seed and one action stream, and the frame
of the env's state after chosen steps (step 0 = after reset; an episode that ends is reset at once, as the pool's auto-reset
does).  Every frame is stored at tile size 8, some also at 32 and at 7; highlight on and off; all four headings; the agent
standing in an open doorway.  Build container only (needs /root/reference).

usage: python tests/golden/make_rgb_grid_golden.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..', 'oracle'))
sys.path.insert(0, os.path.join(HERE, '..'))
import refenv  # noqa: E402
from render_grid_common import shim_render  # noqa: E402

# (level, seed, steps, drive with the reference bot): the bot walks through doorways; it hangs on KeyInBox, so the levels
# it is not needed on get random actions (toggle-heavy: doors open and close)
LEVELS = [('GoToLocal', 31, 60, False), ('BossLevel', 41, 220, True), ('Unlock', 51, 160, True), ('KeyInBox', 61, 80, False),
          ('PutNextS6N3Carrying', 71, 60, False), ('OpenDoorsOrderN4', 81, 120, False), ('KeyCorridorS3R3', 91, 120, False)]
EVERY = 20                    # a frame every EVERY steps, plus the first step the agent stands in an open doorway
P_RANDOM = [0.2, 0.2, 0.3, 0.08, 0.07, 0.15, 0.0]


def main():
    gym = refenv.setup('philox')
    from babyai.bot import Bot
    actions, frames, recs = [], [], []
    headings, doorway = set(), 0
    rng = np.random.RandomState(5)
    for li, (level, seed, T, use_bot) in enumerate(LEVELS):
        env = refenv.make_env(level, seed, 'philox')
        env.reset()
        bot, last = (Bot(env) if use_bot else None), None
        acts = []
        in_door = False

        def snap(t, door):
            k = len(recs)
            sizes = [8] + ([32] if k % 5 == 1 else []) + ([7] if k % 5 == 3 else [])
            for ts in sizes:
                hl = not (k % 3 == 2 and ts == 8)
                f = shim_render(env, highlight=hl, tile_size=ts)
                frames.append(f.copy())
                recs.append([li, t, ts, int(hl), int(door), f.shape[0], f.shape[1]])
            headings.add(int(env.agent_dir))

        snap(0, False)
        for t in range(1, T + 1):
            a = None
            if bot is not None and rng.rand() < 0.85:
                try:
                    a = int(bot.replan(last))
                except Exception:
                    bot = None
            if a is None:
                a = int(rng.choice(7, p=P_RANDOM))
                bot = None
            last = a
            acts.append(a)
            _obs, _r, done, _ = env.step(a)
            if done:
                env.reset()
                bot, last = (Bot(env) if use_bot else None), None
            cell = env.grid.get(*env.agent_pos)
            door = cell is not None and cell.type == 'door'
            if door and not in_door and doorway < 6:
                doorway += 1
                snap(t, True)
            elif t % EVERY == 0:
                snap(t, door)
            in_door = door
        actions.append(acts)
    assert headings == {0, 1, 2, 3}, headings
    assert doorway >= 1
    r = np.array(recs, np.int32)
    assert set(r[:, 2]) == {7, 8, 32} and set(r[:, 3]) == {0, 1}
    T = max(len(a) for a in actions)
    A = np.full((len(LEVELS), T), -1, np.int8)
    for i, a in enumerate(actions):
        A[i, :len(a)] = a
    sizes = np.array([f.size for f in frames], np.int64)
    out = os.path.join(HERE, 'rgb_grid.npz')
    np.savez_compressed(out, levels=json.dumps([l[0] for l in LEVELS]), seeds=np.array([l[1] for l in LEVELS], np.uint64),
                        actions=A, frames=r, offsets=np.concatenate([[0], np.cumsum(sizes)]),
                        pixels=np.concatenate([f.reshape(-1) for f in frames]))
    print('%d frames (%d in a doorway), headings %s -> %s (%d KB)' % (len(frames), int(r[:, 4].sum()), sorted(headings), out,
                                                                   os.path.getsize(out) // 1024))


if __name__ == '__main__':
    main()
