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

/* Replaces: ParallelEnv.step (penv.py:45-52) / ManyEnvs.step (evaluate.py:72-78)
 * -> RoomGridLevel.step (levelgen.py:49-66) -> MiniGridEnv.step/gen_obs.
 * actions_dev: n_envs actions, action_bytes = 1 (int8/uint8) or 8 (int64, what
 * torch's dist.sample() yields, rl/algos/base.py:142).  Outputs: obs uint8
 * [n_envs][147]; reward float32[n_envs]; done uint8[n_envs]; dir int8[n_envs]
 * (may be NULL).  In AUTORESET mode a finished env returns the terminal
 * reward/done together with the first observation of its next episode. */
int bb_pool_step(bb_pool *pool, const void *actions_dev, int32_t action_bytes,
                 uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev, void *stream);

/* bb_pool_step on the pool's internal stream with CUDA events around each of its
 * two kernels (measurement hook for bench.py's roofline line; synchronises). */
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
 * of T step launches. */
int bb_pool_rollout(bb_pool *pool, const int8_t *actions_dev, int32_t T,
                    uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev, void *stream);

/* bb_pool_rollout on the pool's internal stream with CUDA events around the stepping kernel and around the
 * level refill (measurement hook for bench.py's roofline line; synchronises).  Times are 0 when the call
 * took the per-step-graph path. */
int bb_pool_rollout_timed(bb_pool *pool, const int8_t *actions_dev, int32_t T,
                          uint8_t *obs_dev, float *reward_dev, uint8_t *done_dev, int8_t *dir_dev,
                          float *ms_rollout_kernel, float *ms_refill);

/* Same as bb_pool_step but with HOST buffers (what ParallelEnv.step hands
 * back to BaseAlgo.collect_experiences, rl/algos/base.py:144): copies actions
 * host->device, steps, copies obs/reward/done/dir device->host, synchronises. */
int bb_pool_step_host(bb_pool *pool, const int8_t *actions_host,
                      uint8_t *obs_host, float *reward_host, uint8_t *done_host, int8_t *dir_host);
int bb_pool_reset_host(bb_pool *pool, uint8_t *obs_host, int8_t *dir_host);

/* The learner's step (BaseAlgo.collect_experiences, rl/algos/base.py:131-188, with the observations resident on the
 * device): actions from a HOST buffer (base.py:144 hands numpy), observation (and optionally direction) into DEVICE
 * buffers on `stream`, reward / done into HOST buffers (base.py:158-179 reads them there); synchronises `stream`. */
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
 * launched. */
int bb_pool_render_grid(bb_pool *pool, const int32_t *env_ids_host, int32_t n_sel, int32_t tile_size, int32_t highlight,
                        uint8_t *rgb_dev, void *stream);
/* The full-grid tile table of one tile size (host, no GPU): uint8 [2][5][43][ts][ts][3] indexed by highlight, agent (0 none,
 * 1 + direction) and the cell index of a grid cell byte (0 empty, 1 + 6 k + color for k = wall / key / ball / box,
 * 25 + 6 state + color for doors).  For parity tests. */
int bb_grid_tiles(int32_t tile_size, uint8_t *tiles_host);

/* Replaces: obs['mission'] + InstructionsPreprocessor (utils/format.py:59-75).
 * Device pointer to int16 [n_envs][max_len] token ids of the current missions
 * (0 = pad, ids index bb_vocab_word); rewritten whenever an env is reset. */
int bb_pool_mission_tokens(bb_pool *pool, const int16_t **tokens_dev, int32_t *max_len);
int32_t bb_vocab_size(void);
const char *bb_vocab_word(int32_t id);   /* id 1..bb_vocab_size(); 0 = pad -> "" */

/* Introspection for parity tests: one env's hidden state copied to host.
 * grid_host: uint8[height*width], cell = type | color<<3 | state<<6 (empty 0x01);
 * info_host: int32[8] = agent_x, agent_y, agent_dir, carrying cell byte (0 none),
 * step_count, max_steps, rng draws (low 31 bits), generation attempts. */
int bb_pool_get_state(bb_pool *pool, int32_t env, uint8_t *grid_host, int32_t *info_host);
int32_t bb_pool_width(const bb_pool *pool);
int32_t bb_pool_height(const bb_pool *pool);
int32_t bb_pool_num_envs(const bb_pool *pool);

/* Counters since creation, summed on the device: [0] env-steps, [1] episodes
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
