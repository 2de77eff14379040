/*
 * babyai_b200.h -- C ABI of the GPU-native (H100) batched BabyAI environment pool.
 *
 * The reference (mila-iqia/babyai) has no FFI: its "plugin interface" for the
 * environment path is the duck-typed Python surface that babyai/rl and
 * babyai/imitation.py consume.  Each entry point below names the reference
 * interface it replaces (paths relative to the reference tree).  The Python
 * host side (babyai_b200/vecenv.py) mirrors that surface on top of this ABI;
 * INTEGRATION.md shows the ctypes binding a maintainer adds.
 *
 * Conventions: plain pointers and sizes only (no torch types).  `*_dev`
 * pointers are CUDA device pointers on the pool's device (typically the
 * data_ptr() of PyTorch-owned tensors); `*_host` pointers are host memory.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Any call may use any stream, and the pool orders its own state between
 * them: a call on a stream other than the previous call's waits for the pool
 * work enqueued so far (the internal-stream calls -- *_host, *_timed -- too).
 * The caller orders its own buffers, as in PyTorch: a buffer written on one
 * stream and read by a call on another needs the caller's own event.  A
 * stream handed to the pool must stay valid until the pool's next call.
 * Every function returns 0 on success, non-zero on error; bb_last_error()
 * returns a thread-local message.  A pool is used by one host thread at a
 * time, one outstanding step at a time (penv.py has the same contract).
 */
#ifndef BABYAI_B200_H
#define BABYAI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BB_OBS_BYTES 147          /* uint8[7][7][3], index (vi*7+vj)*3+c   */
#define BB_MAX_OBJ 32             /* describable objects per env (doors incl.) */
#define BB_MAX_TOKENS 72          /* longest BossLevel mission, in words    */

/* level families (which gen_mission the generator kernel runs) */
#define BB_KIND_REDBALL 0         /* iclr19_levels.py:10-72   GoToRedBall*          */
#define BB_KIND_OBJ 1             /* iclr19_levels.py:75-301,360-415,477-491 GoToObj/GoToLocal/PutNextLocal/GoTo/Pickup/UnblockPickup/Open/PutNext */
#define BB_KIND_LEVELGEN 2        /* levelgen.py:256-460 LevelGen (PickupLoc .. BossLevel) */
#define BB_KIND_IMPUNLOCK 3       /* iclr19_levels.py:304-355 GoToImpUnlock; num_dists = distractors per unlocked room */
#define BB_KIND_UNLOCK 4          /* iclr19_levels.py:418-474 Unlock;        num_dists = distractors per unlocked room */
#define BB_KIND_BONUS 5           /* bonus_levels.py: the family is bb_level_spec::bonus (BB_BN_*), its constructor arguments bonus_a / bonus_b */
/* instruction / action kinds (verifier.py) */
#define BB_I_GOTO 0
#define BB_I_PICKUP 1
#define BB_I_OPEN 2
#define BB_I_PUTNEXT 3
/* rand_instr kinds (levelgen.py:407) */
#define BB_K_ACTION 0
#define BB_K_AND 1
#define BB_K_SEQ 2

/* Constructor arguments of the reference level classes
 * (RoomGridLevel.__init__ levelgen.py:25-33, LevelGen.__init__ :262-291,
 *  Level_* in iclr19_levels.py). */
typedef struct bb_level_spec {
    int32_t kind;
    int32_t room_size, num_rows, num_cols, num_dists;
    int32_t instr;              /* BB_KIND_OBJ: BB_I_GOTO / BB_I_PICKUP / BB_I_OPEN / BB_I_PUTNEXT */
    int32_t doors_open;         /* Level_GoTo(doors_open=...)                 */
    int32_t grey_dists;         /* Level_GoToRedBallGrey                      */
    double  locked_room_prob;   /* LevelGen(...) from here on                 */
    int32_t locations, unblocking, implicit_unlock;
    int32_t n_action_kinds; int32_t action_kinds[4];
    int32_t n_instr_kinds;  int32_t instr_kinds[3];
    int32_t all_unique;         /* BB_KIND_OBJ: add_distractors(all_unique=...) (Level_PutNextLocal)        */
    int32_t require_unreachable;/* BB_KIND_OBJ: Level_UnblockPickup rejects levels whose objects are all reachable */
    /* verifier modes (babyai/levels/verifier.py) */
    int32_t strict_mask;        /* bit l: leaf instruction l is built with strict=True (:255, :323, :369); bit 4: the Before / After root is (:430) */
    int32_t done_actions;       /* verifier.use_done_actions (BABYAI_DONE_ACTIONS, :15-17): instructions report through the `done` action */
    /* BB_KIND_BONUS (babyai/levels/bonus_levels.py): 1 GoToRedBlueBall :7, 2 OpenRedDoor :43, 3 OpenDoor :65 (a: 0 / 1 color / 2 loc),
     * 4 GoToDoor :150, 5 GoToObjDoor :174, 6 ActionObjDoor :200, 7 UnlockLocal :237 (a: distractors), 8 KeyInBox :267,
     * 9 UnlockPickup :290 (a: distractors), 10 BlockedUnlockPickup :332, 11 UnlockToUnlock :364, 12 PickupDist :401, 13 PickupAbove :447,
     * 14 OpenTwoDoors :472 (a, b: first / second colour + 1, 0 = random), 15 FindObj :565, 16 KeyCorridor :614 (a: object type),
     * 17 1Room :707, 18 PutNext :766 (a: objs_per_room, b: start_carrying), 19 MoveTwoAcross :907 (a: objs_per_room),
     * 20 OpenDoorsOrder :974 (a: num_doors) */
    int32_t bonus, bonus_a, bonus_b;
} bb_level_spec;

typedef struct bb_pool bb_pool;

/* step-mode: what happens to an environment whose episode ended */
#define BB_MODE_AUTORESET 0       /* babyai/rl/utils/penv.py:7-11,48-50 (ParallelEnv) */
#define BB_MODE_FREEZE 1          /* babyai/evaluate.py:72-78 (ManyEnvs)              */

/* Replaces: `envs = [gym.make(id) for _ in range(N)]` + `ParallelEnv(envs)` /
 * `ManyEnvs(envs)` construction (scripts/train_rl.py:53-60, rl/algos/base.py:54,
 * evaluate.py:86-94).  Allocates the struct-of-arrays state of n_envs
 * environments in device memory of CUDA device `device`. */
int bb_pool_create(const bb_level_spec *spec, int32_t n_envs, int32_t device, bb_pool **out);
int bb_pool_destroy(bb_pool *pool);

/* Replaces: a list of gym envs of SEVERAL levels handed to ParallelEnv(envs) / ManyEnvs(envs) (penv.py:18-59,
 * evaluate.py:58-81; the multi_env list of imitation.py:83-84,163-165,326-338; multi-task and curriculum training).  A MIXED
 * pool of n_groups contiguous groups: group g holds envs [start_g, start_g + counts[g]) (start_0 = 0, in list order) of level
 * specs[g]; a spec may appear in several groups.  Each group is an ordinary pool of its level -- its own state layout, level
 * ring, generation schedule and kernels -- whose rows of every buffer are [start_g, start_g + counts[g]), so a mixed pool
 * computes exactly what its groups compute as separate pools with the same seeds (default seeds: 0 .. counts[g] - 1 in each
 * group).  The handle is a bb_pool: every entry point below takes it (the exceptions are listed there).  The mission tokens of
 * all groups are one int16 [N][L] array, L the largest max_tokens of the groups (shorter missions are zero-padded).  Rollout
 * and step outputs keep the UBLKCP bulk-store path where a group's rows start on a multiple of 16 envs and (rollout) N is
 * one too: group sizes that are multiples of 32 keep it everywhere, other sizes are correct through plain stores.
 * Counts >= 1, N <= INT32_MAX; n_groups = 1 is bb_pool_create. */
int bb_pool_create_mixed(const bb_level_spec *specs, const int32_t *counts, int32_t n_groups, int32_t device, bb_pool **out);
/* 1 for a pool of one level; group g's first env, env count and level spec (any pointer may be NULL). */
int32_t bb_pool_num_groups(const bb_pool *pool);
int bb_pool_group(const bb_pool *pool, int32_t g, int32_t *start, int32_t *count, bb_level_spec *spec_out);
/* grid width / height of env `env` (on a mixed pool they differ between groups) */
int bb_pool_env_dims(const bb_pool *pool, int32_t env, int32_t *w, int32_t *h);

/* Replaces: env.seed(seed) per env (scripts/train_rl.py:59; ManyEnvs.seed
 * evaluate.py:64-65).  seeds_host[n_envs]; restarts each env's random stream. */
int bb_pool_seed(bb_pool *pool, const uint64_t *seeds_host);

int bb_pool_set_mode(bb_pool *pool, int32_t mode);

/* Replaces: ParallelEnv.reset (penv.py:39-43) / ManyEnvs.reset (evaluate.py:67-70)
 * -> RoomGridLevel.reset (levelgen.py:35-47).  Generates a new level for every
 * env and writes the first observation.  obs_dev: uint8[n_envs][147];
 * dir_dev: int8[n_envs] or NULL. */
int bb_pool_reset(bb_pool *pool, uint8_t *obs_dev, int8_t *dir_dev, void *stream);

/* Replaces: env.seed(seeds_host[k]) (if seeds_host != NULL) then env.reset() for the envs env_ids_host[0..n_sel) only
 * (RoomGridLevel.reset, levelgen.py:35-47; make_agent_demos.py:93, evaluate.py:64-70 per env).  Each listed env starts a
 * new episode: with seeds, the first level of seed seeds_host[k] (its state is then that of a pool that bb_pool_seed gave
 * that seed, followed by bb_pool_reset: generation draws and attempts included); without, the next level of the env's own
 * stream (what its next auto-reset would have taken).  In freeze mode the env steps again from the next call.  Envs not
 * listed keep their state, level rings and streams.  obs_dev: uint8[n_envs][147], dir_dev: int8[n_envs] or NULL: only the
 * rows of the listed envs are written; their mission tokens are rewritten.  Counters are unchanged (a reset ends no counted
 * episode).  Ids must lie in [0, n_envs) without repeats; arguments are checked before anything is enqueued, and n_sel = 0
 * enqueues nothing.  Asynchronous and stream-ordered on `stream`; the host arrays are consumed before the call returns.
 * Device work scales with n_sel; in auto-reset mode a reseeded env's ring is refilled serially (D levels per env). */
int bb_pool_reset_envs(bb_pool *pool, const int32_t *env_ids_host, const uint64_t *seeds_host, int32_t n_sel,
                       uint8_t *obs_dev, int8_t *dir_dev, void *stream);

/* Replaces: copy.deepcopy(env) of a reference env (fork a state, rewind to it), and what a reference user cannot do at all:
 * keep the env side of a training run in a checkpoint.  A RECORD is one env's whole future as bytes: its live level (pose,
 * step count, frozen flag, objects, instruction state, mission, grid), its random stream, locked_room, attempts, last reward,
 * and the levels its generator has already produced (the stream position is the one AFTER those levels, so they travel with
 * it).  An env loaded from a record continues exactly as the saved env would have: every later observation, reward, done
 * and level.  bb_pool_env_record_bytes: the size and stride of one record (a multiple of 16; header + (1 + ring depth) levels,
 * of which only the levels in use are read or written).  A record is valid for the pool that wrote it and for every pool
 * created with the same level spec and ring depth (a checkpoint survives a process restart); a record with another layout
 * tag leaves its env untouched and adds one to the error counter.
 * bb_pool_save_envs: record k of records_dev (16-byte aligned, n_sel records) := env env_ids_host[k]; NULL ids = every env in
 * order (n_sel must be n_envs); ids may repeat.  The pool is unchanged.
 * bb_pool_load_envs: env env_ids_host[k] := record slots_host[k] of the n_records at records_dev (NULL slots: record k; NULL
 * ids: env k, n_sel must be n_envs).  Slots may repeat (one record into many envs: a fork); ids must lie in [0, n_envs)
 * without repeats.  Rows env_ids_host[k] of obs_dev uint8[n_envs][147] / dir_dev int8[n_envs] (either may be NULL) receive
 * the observation of the env's state after the call; no other row is written; the loaded envs' mission tokens are
 * rewritten.  Envs not listed keep their state, level rings and streams.  Counters are unchanged.
 * Both: arguments are checked before anything is enqueued, n_sel = 0 enqueues nothing; asynchronous and stream-ordered on
 * `stream` (the caller orders records_dev between streams); the host arrays are consumed before the call returns.
 * Not on a mixed pool (an error, nothing enqueued; bb_pool_env_record_bytes returns 0): a record's layout tag is made of the
 * grid size, token width and ring depth, not of the level, so a record of one group's level would load silently into an env
 * of another level with the same layout. */
int64_t bb_pool_env_record_bytes(const bb_pool *pool);
int bb_pool_save_envs(bb_pool *pool, const int32_t *env_ids_host, int32_t n_sel, uint8_t *records_dev, void *stream);
int bb_pool_load_envs(bb_pool *pool, const int32_t *env_ids_host, const int32_t *slots_host, int32_t n_sel,
                      const uint8_t *records_dev, int32_t n_records, uint8_t *obs_dev, int8_t *dir_dev, void *stream);

/* Replaces: ParallelEnv.step (penv.py:45-52) / ManyEnvs.step (evaluate.py:72-78)
 * -> RoomGridLevel.step (levelgen.py:49-66) -> MiniGridEnv.step/gen_obs.
 * actions_dev: n_envs actions, action_bytes = 1 (int8/uint8) or 8 (int64, what
 * torch's dist.sample() yields, rl/algos/base.py:142).  Outputs: obs uint8
 * [n_envs][147]; reward float32[n_envs]; done uint8[n_envs]; dir int8[n_envs]
 * (may be NULL).  In AUTORESET mode a finished env returns the terminal
 * reward/done together with the first observation of its next episode. */
int bb_pool_step(bb_pool *pool, const void *actions_dev, int32_t action_bytes,
                 uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev, void *stream);

/* Replaces: ManyEnvs.step (babyai/evaluate.py:72-78), which steps only the envs that are not done -- here any id list: one
 * step of the listed envs, every other env held still.  The result equals bb_pool_step restricted to the listed envs: env
 * env_ids_host[k] applies action k of actions_dev (indexed by LIST POSITION, like seeds_host of bb_pool_reset_envs: what a
 * policy evaluated on obs[ids] returns) and writes ROW env_ids_host[k] of obs_dev uint8 [n_envs][147], reward_dev float32
 * [n_envs], done_dev uint8 [n_envs] and dir_dev int8 [n_envs] (may be NULL) -- only the listed rows.  action_bytes: 1
 * (int8 / uint8) or 8 (int64).  In auto-reset mode a listed env whose episode ends takes the next level of its ring and
 * returns the terminal reward and done with the new episode's first observation (its mission tokens change); in freeze mode
 * a listed frozen env replays its last reward with done = 1, as in bb_pool_step.  Unlisted envs do not move: their state,
 * stream, step count, output rows and mission tokens stay as they were (a generation pass that falls due may top their
 * rings up with the next levels of their own streams, as during any call).  The counters change as bb_pool_step would change
 * them for the listed envs.  Ids lie in [0, n_envs) without repeats; every argument is checked before anything is enqueued,
 * and n_sel = 0 enqueues nothing and is not a step.  Stream-ordered on `stream` like bb_pool_step, no synchronisation; the
 * host id array is consumed before the call returns.  Device work scales with n_sel: one launch per 4 096 ids. */
int bb_pool_step_envs(bb_pool *pool, const int32_t *env_ids_host, int32_t n_sel, const void *actions_dev, int32_t action_bytes,
                      uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev, void *stream);

/* bb_pool_step on the pool's internal stream with CUDA events around each of its
 * two kernels (measurement hook for bench.py's roofline line; synchronises).  Not on a mixed pool (one pair of times per
 * level). */
int bb_pool_step_timed(bb_pool *pool, const void *actions_dev, int32_t action_bytes,
                       uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev,
                       float *ms_step_kernel, float *ms_gen_kernel);

/* T consecutive steps with pre-recorded actions (the "random action" rollout
 * of BASELINE.json configs, and the shape of BaseAlgo.collect_experiences'
 * [frames_per_proc][procs] buffers, rl/algos/base.py:110-188): actions int8
 * [T][n_envs]; outputs [T][n_envs]...  Results are identical to T calls of
 * bb_pool_step.  Grids up to 22 x 22 with a ring of pre-generated levels deep enough
 * (>= 3 T): ONE persistent kernel keeps the env state in shared memory for the T steps
 * (single-room levels: level generation runs inside it too); otherwise one CUDA graph
 * of T step launches.  Mixed pool: each group runs on an internal stream of its own, forked from `stream` and joined back
 * into it, so the groups' kernels share the GPU; every buffer keeps the row stride N between steps. */
int bb_pool_rollout(bb_pool *pool, const int8_t *actions_dev, int32_t T,
                    uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev, void *stream);

/* bb_pool_rollout on the pool's internal stream with CUDA events around the stepping kernel and around the
 * level refill (measurement hook for bench.py's roofline line; synchronises).  Times are 0 when the call
 * took the per-step-graph path.  Not on a mixed pool. */
int bb_pool_rollout_timed(bb_pool *pool, const int8_t *actions_dev, int32_t T,
                          uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev,
                          float *ms_rollout_kernel, float *ms_refill);

/* Same as bb_pool_step but with HOST buffers (what ParallelEnv.step hands
 * back to BaseAlgo.collect_experiences, rl/algos/base.py:144): copies actions
 * host->device, steps, copies obs/reward/done/dir device->host, synchronises
 * (a mixed pool: every group is enqueued first, then one synchronisation). */
int bb_pool_step_host(bb_pool *pool, const int8_t *actions_host,
                      uint8_t *obs_host, float *reward_host, uint8_t *done_host, int8_t *dir_host);
int bb_pool_reset_host(bb_pool *pool, uint8_t *obs_host, int8_t *dir_host);

/* The learner's step (BaseAlgo.collect_experiences, rl/algos/base.py:131-188, with the observations resident on the
 * device): actions from a HOST buffer (base.py:144 hands numpy), observation (and optionally direction) into DEVICE
 * buffers on `stream`, reward / done into HOST buffers (base.py:158-179 reads them there); synchronises `stream` (once, after
 * every group of a mixed pool). */
int bb_pool_step_learner(bb_pool *pool, const int8_t *actions_host, uint8_t *obs_dev, float *reward_host,
                         uint8_t *done_host, int8_t *dir_dev, void *stream);

/* Replaces: gym_minigrid.wrappers.RGBImgPartialObsWrapper.observation -> MiniGridEnv.get_obs_render (tile_size 8), the
 * wrapper the reference puts around every env when 'pixel' is in the architecture name (scripts/train_rl.py:54-58,
 * babyai/evaluate.py:91-92; consumed by the 8x8 / stride-8 first convolution, babyai/model.py:96-98).  The image is a pure
 * function of the 7x7x3 observation: obs_dev uint8 [n_obs][147] (what bb_pool_step / bb_pool_reset / bb_pool_rollout wrote;
 * n_obs may be T * n_envs) -> rgb_dev uint8 [n_obs][56][56][3], 16-byte aligned.  One HBM-bound kernel (9 408 B written
 * per 147 B read); the 513 tiles it copies are rasterised once per pool exactly as the reference package draws them. */
int bb_pool_render_rgb(bb_pool *pool, const uint8_t *obs_dev, uint8_t *rgb_dev, int32_t n_obs, void *stream);
/* The tile table itself (host): uint8 [513][8][8][3]; id = cell byte (type | color << 3 | state << 6) for a visible cell,
 * 256 for an unseen cell, 257 + cell byte for the agent's own cell.  For parity tests. */
int bb_rgb_tiles(uint8_t *tiles_host);

/* Replaces: MiniGridEnv.render('rgb_array', highlight=highlight, tile_size=tile_size) (gym_minigrid 1.0.x), what
 * scripts/manual_control.py:14 draws and what video logging of agents needs: the full grid of each selected env's CURRENT
 * state (after an auto-reset step: the first state of the new episode; in freeze mode: the terminal state).  Cell (x, y) is
 * Grid.render_tile(cell, agent_dir if the agent stands there, highlight = the cell is visible in the agent's 7x7 view);
 * the carried object and box contents are not drawn.  env_ids_host: n_sel ids in [0, n_envs), any order, repeats allowed;
 * NULL = every env in order (n_sel must then be n_envs).  tile_size 1..64.  rgb_dev: uint8 [n_sel][H*ts][W*ts][3],
 * 16-byte aligned.  Stream-ordered after the work already on `stream`, no synchronisation (the table of a tile size is
 * rasterised on the host and uploaded the first time that size is rendered); arguments are checked before anything is
 * launched.  On a mixed pool the selected envs must share one grid size (H, W of bb_pool_env_dims); an error otherwise. */
int bb_pool_render_grid(bb_pool *pool, const int32_t *env_ids_host, int32_t n_sel, int32_t tile_size, int32_t highlight,
                        uint8_t *rgb_dev, void *stream);
/* The full-grid tile table of one tile size (host, no GPU): uint8 [2][5][43][ts][ts][3] indexed by highlight, agent (0 none,
 * 1 + direction) and the cell index of a grid cell byte (0 empty, 1 + 6 k + color for k = wall / key / ball / box,
 * 25 + 6 state + color for doors).  For parity tests. */
int bb_grid_tiles(int32_t tile_size, uint8_t *tiles_host);

/* Replaces: gym_minigrid 1.0.x FullyObsWrapper.observation(obs)['image']: grid.encode() of each selected env's CURRENT
 * state, uint8 [n_sel][W][H][3] in x-major order (row k of out_dev is env env_ids_host[k]), each cell (type, color, state) of
 * OBJECT_TO_IDX / COLOR_TO_IDX / STATE_TO_IDX, an empty cell (1, 0, 0), and the agent's cell (10 = 'agent', 0 = 'red',
 * agent_dir).  The carried object is not in the grid.  env_ids_host: n_sel ids in [0, n_envs), any order, repeats allowed;
 * NULL = every env in order (n_sel must then be n_envs).  Any alignment of out_dev.  Stream-ordered after the work already on
 * `stream`, no synchronisation; arguments are checked before anything is launched.  On a mixed pool the selected envs must
 * share one grid size (W, H of bb_pool_env_dims); an error otherwise, with nothing launched. */
int bb_pool_full_obs(bb_pool *pool, const int32_t *env_ids_host, int32_t n_sel, uint8_t *out_dev, void *stream);

/* Replaces: obs['mission'] + InstructionsPreprocessor (utils/format.py:59-75).
 * Device pointer to int16 [n_envs][max_len] token ids of the current missions
 * (0 = pad, ids index bb_vocab_word); rewritten whenever an env is reset. */
int bb_pool_mission_tokens(bb_pool *pool, const int16_t **tokens_dev, int32_t *max_len);
int32_t bb_vocab_size(void);
const char *bb_vocab_word(int32_t id);   /* id 1..bb_vocab_size(); 0 = pad -> "" */

/* Introspection for parity tests: one env's hidden state copied to host.
 * grid_host: uint8[height*width] of the env's own grid (bb_pool_env_dims), cell = type | color<<3 | state<<6 (empty 0x01);
 * info_host: int32[8] = agent_x, agent_y, agent_dir, carrying cell byte (0 none),
 * step_count, max_steps, rng draws (low 31 bits), generation attempts. */
int bb_pool_get_state(bb_pool *pool, int32_t env, uint8_t *grid_host, int32_t *info_host);
int32_t bb_pool_width(const bb_pool *pool);      /* a mixed pool: the largest of its groups */
int32_t bb_pool_height(const bb_pool *pool);
int32_t bb_pool_num_envs(const bb_pool *pool);

/* Counters since creation, summed on the device (and over the groups of a mixed pool): [0] env-steps, [1] episodes
 * ended, [2] episodes ended in success, [3] internal errors (must stay 0).
 * (Multi-GPU runs all-gather these -- the only collective on this path.) */
int bb_pool_counters(bb_pool *pool, int64_t *out4_host);

/* Number of kernel launches issued by this pool since creation. */
int64_t bb_pool_launches(const bb_pool *pool);

const char *bb_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
