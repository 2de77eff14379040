// pool.cu -- kernels and C ABI of the batched BabyAI environment pool (sm_90a).
//
//   k_rollout     bb_pool_rollout (and bb_pool_step on single-room levels, T = 1): persistent over T steps, per CTA
//                 two stepping warps (one lane per environment, state resident in shared memory) and, in fused
//                 launches, one generator warp that refills the level rings of the CTA's environments.
//   k_step8       bb_pool_step on multi-room levels: eight lanes per environment (one per view column).
//   k_gen_scan, k_gen_small  level generation for single-room levels as separate passes (reset, per-step API, rooms
//                 smaller than 6x6): one lane per environment, the warp in lock-step through one attempt per round.
//   k_gen         level generation for every other level: one warp per level (generate_level).
//   k_seed        env.seed().
//   k_seed_sel, k_gen_scan_sel, k_pub_sel, k_reset8  bb_pool_reset_envs: seed, refill and reset the envs of an id list only.
//   k_render_rgb, k_render_grid  pictures: the partial view of an observation, and the full grid of an env's current state.
// Levels depend only on the env's random stream, never on actions, so generating episodes k+1 .. k+D while episode k
// is being played is equivalent to generating them at reset time: every env owns a ring of D pre-generated levels.
// The per-environment logic (step, verifier, observation, generators) is env_logic.cuh; DESIGN.md section 4 has the
// measurements behind each choice.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include <new>
#include <vector>
#include <algorithm>
#include <stdlib.h>

#include "../../include/babyai_b200.h"
#include "env_logic.cuh"
#include "level_params.h"
#include "simt.cuh"
#include "gen_round.cuh"
#include "rollout_lane.cuh"
#include "rollout_cta.cuh"
#include "step8.cuh"
#include "reset8.cuh"
#include <type_traits>
#include "rgb_tiles.h"
#include "grid_render.cuh"

using namespace bb;

// ---------------------------------------------------------------------------------
struct PoolPtrs {
    // live state of every environment
    uint8_t *grid; EnvHot *hot; ObjTab *obj; InstrRec *ins; int16_t *tok;
    // ring of pre-generated levels: arrays [depth][n]; env e has consumed head[e] and k_gen has produced
    // tail[e] levels since the last seed(); level number L lives in slot L % depth
    uint8_t *rgrid; EnvHot *rhot; ObjTab *robj; InstrRec *rins; int16_t *rtok;
    uint32_t *head, *tail;
    // no fences: k_gen works from head_snap (copied from head after the step it was forked from finished)
    // and k_step trusts tail_pub (copied from tail only after a k_gen has completed)
    uint32_t *head_snap, *tail_pub;
    RngRec *rng; uint8_t *locked_room; uint32_t *attempts;
    float *last_reward;
    uint32_t *gen_ticket;      // work-ticket counter of k_gen / k_gen_small
    uint32_t *gen_count; int32_t *gen_list;                          // k_gen_scan: four lists (by missing levels) of envs whose ring is not full
    unsigned long long *warp_counters;   // [num_warps][4]: steps, episodes, successes, errors
    int *err_flag;                       // mapped page-locked word: set by a kernel that found a ring dry; the host fails the next call
    int32_t depth, n;
};

constexpr int GEN_THREADS = 64;                    // 2 warps per block; one warp generates one level at a time
constexpr int GEN_BLOCKS_PER_SM = 14;            // k_gen: 64 threads x 72 registers per block: 14 blocks fill an SM's register file

__device__ __forceinline__ LevelOut ring_slot(const LevelParams &lp, const PoolPtrs &P, int env, int slot)
{
    const size_t idx = (size_t)slot * P.n + env;
    LevelOut o;
    o.grid = P.rgrid + idx * lp.cells_pad; o.hot = P.rhot + idx; o.obj = P.robj + idx; o.ins = P.rins + idx;
    o.tok = P.rtok + idx * lp.max_tokens;
    return o;
}

// ---- k_step8: EIGHT LANES PER ENVIRONMENT, the one-launch-per-step kernel of the multi-room levels (step8.cuh has the role
// function and the design notes; it also runs in tests/hostemu with one OS thread per lane)
// UNTR: KIND_UNLOCK pools (objects without a table entry, env_logic.cuh CARRY_UNTRACKED); every other level runs the
// UNTR = false instantiations
template <int ACT_BYTES, bool UNTR = false>
__global__ void __launch_bounds__(S8_THREADS)
k_step8(const LevelParams lp, const PoolPtrs P, const void *__restrict__ actions, uint8_t *__restrict__ obs,
        float *__restrict__ reward, uint8_t *__restrict__ done, int8_t *__restrict__ dirs, const int n,
        const int mode, const int force_reset)
{
    extern __shared__ __align__(16) uint8_t smem8[];               // [16 envs][cells_pad + 144] then the tiles
    step8_role<PoolPtrs, ACT_BYTES, UNTR>(lp, P, actions, obs, reward, done, dirs, n, mode, force_reset, smem8,
                                          threadIdx.x & 31, threadIdx.x >> 5, blockIdx.x);
}

// Level generation for small single-room levels: ONE LANE PER ENVIRONMENT, THE WARP IN LOCK-STEP THROUGH THE PHASES
// OF ONE ATTEMPT PER ROUND (env_logic.cuh: small_attempt_begin / small_place_try / small_flood_* / small_pick /
// small_desc_try / emit_small_level).
//   k_gen_scan   compacts the environments whose ring is not full into four work lists by the number of levels they
//                miss (>= 4, 3, 2, 1): levels of one env are serial (one random stream), so the longest chains start first;
//   k_gen_small  a lane takes an env from the lists (warp-aggregated atomic) and produces its missing levels one
//                attempt per round.  Inside a round every lane of the warp is in the same phase: placement tries
//                (lanes that are done wait), flood fill, descriptor, and the level is written straight from
//                registers.  Philox is converged too: a lane's next 64 draws sit in a shared-memory ring that is
//                topped up for the whole warp whenever one lane runs low (DrawRing).
// Round 1's version ran a per-lane state machine instead (each lane in its own phase): ncu showed 9.8 active
// lanes per instruction and IPC 0.7.  A rejected attempt costs one round of that lane;
// the env's records (stream position, ring tail) are consistent after every round, so the per-launch round budget
// of bb_pool_rollout's in-stream refill needs no saved generator state.
constexpr int GS_THREADS = 128;

// gen_small_round: one round of the small-level generator for the 32 lanes of a warp -- gen_round.cuh (also compiled for
// the host, with the warp vote emulated by threads, in tests/hostemu)

__global__ void k_gen_scan(const PoolPtrs P, const int n, const int target, const int snap_heads)
{
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int b = -1;
    if (env < n) {
        uint32_t hd;
        if (snap_heads) { hd = P.head[env]; P.head_snap[env] = hd; }      // in-stream refill: the snapshot is taken here
        else hd = P.head_snap[env];
        const int missing = target - (int)(P.tail[env] - hd);
        if (missing > 0) b = missing >= 4 ? 3 : missing - 1;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, b == k);
        if (m) {
            int base = 0;
            if (lane == 0) base = (int)atomicAdd(P.gen_count + k, (uint32_t)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            if (b == k) P.gen_list[(size_t)k * n + base + __popc(m & ((1u << lane) - 1u))] = env;
        }
    }
}

__global__ void __launch_bounds__(GS_THREADS)
k_gen_small(const LevelParams lp, const PoolPtrs P, const int target, const int max_rounds, const int min_active, const int min_keep)
{
    __shared__ uint32_t s_ring[DrawRing::RING_WORDS][GS_THREADS];         // the lanes' draw rings: word j of thread t at [j][t]
    const unsigned FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, tid = threadIdx.x;
    const uint32_t c3 = P.gen_count[3], c2 = P.gen_count[2], c1 = P.gen_count[1], c0 = P.gen_count[0];
    const uint32_t count = c0 + c1 + c2 + c3;
    const uint32_t D = (uint32_t)P.depth;
    DrawRing ds;
    ds.init(&s_ring[0][tid], GS_THREADS, 0, 0);
    int env = -1, left = 0, rounds = 0;
    uint32_t tl = 0;
    bool exhausted = false;
    for (;;) {
        // ---- idle lanes take the next work item (one atomic per warp), longest chains first -----------
        const bool need = left == 0 && !exhausted;
        const uint32_t mneed = __ballot_sync(FULL, need);
        if (mneed) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(P.gen_ticket, (uint32_t)__popc(mneed));
            base = __shfl_sync(FULL, base, 0);
            if (need) {
                uint32_t idx = base + (uint32_t)__popc(mneed & ((1u << lane) - 1u));
                if (idx < count) {
                    int b = 3;
                    if (idx >= c3) { idx -= c3; b = 2; if (idx >= c2) { idx -= c2; b = 1; if (idx >= c1) { idx -= c1; b = 0; } } }
                    env = P.gen_list[(size_t)b * P.n + idx];
                    tl = P.tail[env];
                    left = target - (int)(tl - P.head_snap[env]);
                    const RngRec r = P.rng[env];
                    ds.init(&s_ring[0][tid], GS_THREADS, r.seed, r.draws);
                } else exhausted = true;
            }
        }
        const bool active = left > 0;
        const uint32_t mact = __ballot_sync(FULL, active);
        if (!mact) break;
        // budget spent: the envs keep their deficit -- unless a ring holds fewer than `min_keep` levels (what the launches
        // up to the next refill pass can consume): then the pass goes on until that ring is safe (must-complete rule)
        const bool low = __any_sync(FULL, active && target - left < min_keep);
        if (max_rounds > 0 && rounds >= max_rounds && !low) break;
        // bounded refill (bb_pool_rollout): a round costs the same whether 32 lanes work or 2 (deficits > 1 and
        // rejected attempts leave sparse warps behind), so a sparse warp stops after its first round and leaves the
        // rest to the next pass -- unless a ring is more than half empty
        if (min_active > 0 && rounds >= 1 && __popc(mact) < min_active && !low && !__any_sync(FULL, active && left > (int)(D / 2))) break;
        rounds++;
        gen_small_round<DrawRing, false>(lp, P, ds, active, env, tl, left, D);
    }
}

// ---- persistent rollout kernel: T steps per launch, state resident in shared memory --------------
// bb_pool_rollout's kernel.  Every per-step kernel above reloads ~290 bytes of env state per step through
// a chain of dependent DRAM round trips and is latency-bound at 11-14 warps per SM.  Here a warp loads the
// records of its 32 envs ONCE (coalesced), then runs T steps on them out of shared memory -- per step it
// only reads 32 action bytes and writes the 32 observations / rewards / dones -- and stores the state
// back at the end.  Finished envs take their next level from the ring: >= T levels per env are there before
// the launch, and whoever refills (the CTA's own generator warp, a refill pass between launches, or k_gen on the
// side stream from a head snapshot taken before the launch) never touches a slot this launch can consume.
constexpr int R_WARPS = 2;                    // stepping warps per CTA
constexpr int R_THREADS = 32 * R_WARPS;       // ... and the launch adds one generator warp in fused mode (R_THREADS_FUSED)
constexpr int R_THREADS_FUSED = R_THREADS + 32;
// Generator warp of a fused launch (single-room levels, ParallelEnv mode): while the two stepping warps of the CTA
// run their T steps (k_rollout issues ~48 % of the SM's slots: latency-bound), a third warp refills the rings of the
// CTA's 64 envs with the same round function as k_gen_small -- in issue slots that are idle anyway, with no
// refill pass between launches.  Its shared-memory area: draw rings of 8 Philox blocks per lane, the work list.
// RolloutRing, RG_RING_WORDS, RG_AREA_WORDS: gen_round.cuh

struct SmemOnlyMem {            // lane-private records in shared memory (byte addressable; odd word strides)
    const LevelParams &lp; uint8_t *g, *o, *i;
    __device__ __forceinline__ SmemOnlyMem(const LevelParams &lp_, uint8_t *g_, uint8_t *o_, uint8_t *i_) : lp(lp_), g(g_), o(o_), i(i_) {}
    __device__ __forceinline__ int cell(int x, int y) const { return g[y * lp.rs_g + x]; }
    __device__ __forceinline__ void set_cell(int x, int y, int v) { bb::set_cell(lp, g, x, y, v); }
    __device__ __forceinline__ uint32_t word_at(int off) const { return *reinterpret_cast<const uint32_t *>(g + off); }
    __device__ __forceinline__ int ox(int k) const { return o[k]; }
    __device__ __forceinline__ int oy(int k) const { return o[MAXOBJ + k]; }
    __device__ __forceinline__ int otc(int k) const { return o[2 * MAXOBJ + k]; }
    __device__ __forceinline__ uint32_t oxw(int i) const { return reinterpret_cast<const uint32_t *>(o)[i]; }
    __device__ __forceinline__ uint32_t oyw(int i) const { return reinterpret_cast<const uint32_t *>(o)[MAXOBJ / 4 + i]; }
    __device__ __forceinline__ void set_oxy(int k, int x, int y) { o[k] = (uint8_t)x; o[MAXOBJ + k] = (uint8_t)y; }
    __device__ __forceinline__ uint32_t desc_mask(int d) const { return reinterpret_cast<const uint32_t *>(i)[d]; }
    __device__ __forceinline__ int leaf_kind(int l) const { return i[32 + l]; }
    __device__ __forceinline__ int leaf_pre(int l) const { return i[36 + l]; }
    __device__ __forceinline__ void set_leaf_pre(int l, int v) { i[36 + l] = (uint8_t)v; }
    __device__ __forceinline__ int root_kind() const { return i[40]; }
    __device__ __forceinline__ int side_and() const { return i[41]; }
    __device__ __forceinline__ void set_side_and(int v) { i[41] = (uint8_t)v; }
    __device__ __forceinline__ int flags() const { return i[42]; }
    __device__ __forceinline__ void set_flags(int v) { i[42] = (uint8_t)v; }
    __device__ __forceinline__ int start_carry() const { return i[43]; }
};

template <int K>
struct SmemRoomKindMem : SmemOnlyMem {           // env_logic.cuh mem_spec: single-room levels with one instruction kind K
    static constexpr int spec_room_kinds = K;
    __device__ __forceinline__ SmemRoomKindMem(const LevelParams &lp_, uint8_t *g_, uint8_t *o_, uint8_t *i_) : SmemOnlyMem(lp_, g_, o_, i_) {}
};

template <int ACT_BYTES, bool UNTR = false, int ROOM_KINDS = 0>
__global__ void __launch_bounds__(R_THREADS_FUSED, 7)
k_rollout(const LevelParams lp, const PoolPtrs P, const void *__restrict__ actions_v, uint8_t *__restrict__ obs,
          float *__restrict__ reward, uint8_t *__restrict__ done, int8_t *__restrict__ dirs, const int n, const int T,
          const int mode, const int force_reset, const int gen_rounds, const int gen_min_active)
{
    extern __shared__ __align__(16) uint32_t smr[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int warp_words = rl_warp_words(lp);
    const bool fused = gen_rounds > 0;                  // launched with R_THREADS_FUSED threads and RG_AREA_WORDS more shared memory
    uint32_t *g_area = smr + R_WARPS * warp_words;
    volatile int *s_done = reinterpret_cast<volatile int *>(g_area + RG_AREA_WORDS - 4);
    if (warp == R_WARPS) {
        // generator warp (fused launches only): gen_round.cuh
        rollout_gen_warp(lp, P, g_area, s_done, n, T, blockIdx.x * R_WARPS * 32, gen_rounds, gen_min_active, lane, R_WARPS);
        return;
    }
    // stepping warps: rollout_lane.cuh (also compiled, with the warp primitives emulated by threads, in tests/hostemu)
    rollout_lane_step_warp<PoolPtrs, typename std::conditional<ROOM_KINDS != 0, SmemRoomKindMem<ROOM_KINDS>, SmemOnlyMem>::type, ACT_BYTES, UNTR>(lp, P, actions_v, obs, reward, done, dirs, n, T, mode, force_reset, fused,
                                                                   smr + warp * warp_words, lane, blockIdx.x * R_WARPS + warp, s_done);
}

// k_rollout_cta -- bb_pool_rollout on MULTI-ROOM levels: 32 envs per CTA, a lane-per-env step phase and a 4-lanes-per-env
// observation phase per step, row-major grid only in shared memory (rollout_cta.cuh has the design and the numbers).
template <bool UNTR>
__global__ void __launch_bounds__(RC_THREADS, 7)
k_rollout_cta(const LevelParams lp, const PoolPtrs P, const int8_t *__restrict__ actions, uint8_t *__restrict__ obs,
              float *__restrict__ reward, uint8_t *__restrict__ done, int8_t *__restrict__ dirs, const int n, const int T, const int mode)
{
    extern __shared__ __align__(16) uint32_t smc[];
    rollout_cta_role<PoolPtrs, UNTR>(lp, P, actions, obs, reward, done, dirs, n, T, mode, smc, threadIdx.x, blockIdx.x);
}
// Level generation, decoupled from the step: tops every environment's ring up to `target` levels.
//
// ONE WARP PER ENVIRONMENT.  Generation is a long, branchy, data-dependent rejection-sampling program;
// with one lane per env the 32 lanes of a warp run 32 different paths serially (measured in round 1:
// 3.0 active lanes per instruction).  Instead every lane of the warp runs the same env with identical
// control flow: no divergence, the Philox blocks are computed 32 at a time across the lanes into a shared-memory buffer of 128
// draws (struct Rng), the lanes split the grid rendering, object matching and row initialisation, and lane 0 commits the
// scalar records.  DESIGN.md 4.4 has the list of what round 2 did to this kernel and the measurements.
// Work distribution: k_gen_scan lists the envs whose ring is not full, longest chains first; a warp takes ONE env per
// ticket from a global counter (the slowest generations are a geometric tail of rejected attempts, so static
// assignment would wait for them).
// IMPUNLOCK: the instantiation that serves GoToImpUnlock, Unlock and the bonus families (implicit-unlock placement, untracked
// objects, the bonus_levels.py generators); every other level runs k_gen<false>.
#if BB_GEN_COOP
template <bool IMPUNLOCK>
__global__ void __launch_bounds__(GEN_THREADS)
k_gen(const LevelParams lp, const PoolPtrs P, const int n, const int target, const int lanes_per_warp, const int chain_cap)
{
    __shared__ typename GenMemFor<IMPUNLOCK>::type gen_mem[GEN_THREADS / 32];     // GenMemX (untracked objects) for k_gen<true>
    GenMem *mem = &gen_mem[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const uint32_t c3 = P.gen_count[3], c2 = P.gen_count[2], c1 = P.gen_count[1], c0 = P.gen_count[0];
    const uint32_t count = c0 + c1 + c2 + c3;
    const uint32_t D = (uint32_t)P.depth;
    for (;;) {
        uint32_t idx = 0;
        if (lane == 0) idx = atomicAdd(P.gen_ticket, 1u);
        idx = __shfl_sync(0xFFFFFFFFu, idx, 0);
        if (idx >= count) break;
        int b = 3;
        if (idx >= c3) { idx -= c3; b = 2; if (idx >= c2) { idx -= c2; b = 1; if (idx >= c1) { idx -= c1; b = 0; } } }
        const int env = P.gen_list[(size_t)b * n + idx];
        const uint32_t t0 = P.tail[env];
        const int have = (int)(t0 - P.head_snap[env]);            // consumption as of the step this pass was forked from
        int m = target - have;
        // chain cap (concurrent / periodic passes of bb_pool_rollout): a ring that is still at least half full gets at most
        // `chain_cap` levels per pass -- the levels of one env are serial, and an env that ended ten episodes since the last
        // pass (missions solved at reset) would otherwise set the duration of the whole pass; its deficit is worked off over the next passes, a ring below half is always filled up
        if (chain_cap > 0 && m > chain_cap && have >= (int)(D / 2)) m = chain_cap;
        RngRec r = P.rng[env];
        uint8_t lr = P.locked_room[env];
        int att = 0;
        for (int i = 0; i < m; i++) {
            const LevelOut o = ring_slot(lp, P, env, (int)((t0 + (uint32_t)i) % D));
            att += generate_level_t<IMPUNLOCK>(lp, o, &r, &lr, mem);
            __syncwarp();
            if (lane == 0) P.tail[env] = t0 + (uint32_t)i + 1u;
        }
        if (lane == 0) { P.rng[env] = r; P.locked_room[env] = lr; P.attempts[env] += (uint32_t)att; }
        __syncwarp();
    }
}
#else
// ONE LANE PER LEVEL: a lane takes an env from k_gen_scan's lists (one env per ticket, longest chains first) and generates
// its missing levels with the scalar generator -- the very code of the host build -- its working arrays (GenMem, ~1.3 KB)
// in local memory.  `lanes_per_warp` of the 32 lanes work (the others exit): the lanes of a warp run different levels, so
// the warp executes the union of their control flow; fewer working lanes per warp = shorter latency per level, more =
// more levels per issued instruction (BB_GEN_LANES).
template <bool IMPUNLOCK>
__global__ void __launch_bounds__(GEN_THREADS)
k_gen(const LevelParams lp, const PoolPtrs P, const int n, const int target, const int lanes_per_warp, const int chain_cap)
{
    if ((int)(threadIdx.x & 31) >= lanes_per_warp) return;
    typename GenMemFor<IMPUNLOCK>::type mem;
    const uint32_t c3 = P.gen_count[3], c2 = P.gen_count[2], c1 = P.gen_count[1], c0 = P.gen_count[0];
    const uint32_t count = c0 + c1 + c2 + c3;
    const uint32_t D = (uint32_t)P.depth;
    for (;;) {
        uint32_t idx = atomicAdd(P.gen_ticket, 1u);
        if (idx >= count) break;
        int b = 3;
        if (idx >= c3) { idx -= c3; b = 2; if (idx >= c2) { idx -= c2; b = 1; if (idx >= c1) { idx -= c1; b = 0; } } }
        const int env = P.gen_list[(size_t)b * n + idx];
        const uint32_t t0 = P.tail[env];
        const int have = (int)(t0 - P.head_snap[env]);
        int m = target - have;
        if (chain_cap > 0 && m > chain_cap && have >= (int)(D / 2)) m = chain_cap;
        RngRec r = P.rng[env];
        uint8_t lr = P.locked_room[env];
        int att = 0;
        for (int i = 0; i < m; i++) {
            const LevelOut o = ring_slot(lp, P, env, (int)((t0 + (uint32_t)i) % D));
            att += generate_level_t<IMPUNLOCK>(lp, o, &r, &lr, &mem);
            P.tail[env] = t0 + (uint32_t)i + 1u;
        }
        P.rng[env] = r; P.locked_room[env] = lr; P.attempts[env] += (uint32_t)att;
    }
}
#endif

// k_render_rgb -- RGBImgPartialObsWrapper.observation for a batch: uint8[n][7][7][3] observations -> uint8[n][56][56][3]
// images (tile size 8).  The image is a pure function of the observation: every view cell selects one of 513 pre-rendered
// 192-byte tiles (rgb_tiles.h).  This is the one output of the path that is genuinely HBM bound: 9 408 bytes written per
// 147 bytes read (616 MB per step of 65 536 envs).  One warp per environment at a time: the 49 tile ids go to shared
// memory, then the warp streams the image out as 588 coalesced 16-byte stores; each store is two 8-byte pieces of tile
// rows (a pixel row is 7 tiles x 24 bytes, so 8-byte pieces never straddle a tile) fetched from the L1-resident table.
// Which tile piece a lane needs in iteration k does not depend on the environment: the (cell, offset inside the tile) pairs
// are computed once per CTA into shared memory.
constexpr int RGB_THREADS = 256, RGB_IMG_BYTES = 56 * 56 * 3, RGB_VEC = RGB_IMG_BYTES / 16, RGB_ITERS = (RGB_VEC + 31) / 32;   // 9408 B, 588, 19

__global__ void __launch_bounds__(RGB_THREADS, 4)
k_render_rgb(const uint8_t *__restrict__ obs, uint8_t *__restrict__ rgb, const uint8_t *__restrict__ lut, const int n)
{
    __shared__ uint16_t s_ids[RGB_THREADS / 32][64];
    __shared__ uint32_t s_where[RGB_ITERS][32];  // two (cell index | offset in tile << 8) pairs per 16-byte vector, per lane
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nwarps = gridDim.x * (RGB_THREADS / 32);
    // piece h (8 bytes) of the image: pixel row h / 21, 8-byte column h % 21 -> tile column vi = (h % 21) / 3, part (h % 21) % 3
    for (int idx = threadIdx.x; idx < RGB_ITERS * 32; idx += RGB_THREADS) {
        uint32_t w = 0;
        for (int half = 0; half < 2; half++) {
            const int h = 2 * ((idx & 31) + 32 * (idx >> 5)) + half;
            const int row = h / 21, c8 = h - row * 21, vi = c8 / 3, part = c8 - vi * 3;
            const int vj = (row >> 3) % 7, ty = row & 7;           // (% 7: the padding vectors past 588 stay inside the id table)
            const uint32_t v = (uint32_t)(vi * 7 + vj) | ((uint32_t)(ty * 24 + part * 8) << 8);
            w |= v << (16 * half);
        }
        s_where[idx >> 5][idx & 31] = w;
    }
    __syncthreads();
    uint16_t *ids = s_ids[warp];
    for (int env = blockIdx.x * (RGB_THREADS / 32) + warp; env < n; env += nwarps) {
        const uint8_t *o = obs + (size_t)env * OBS_BYTES;
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const int cell = lane + 32 * r;
            if (cell < 49) {
                const uint32_t t = o[3 * cell], c = o[3 * cell + 1], st = o[3 * cell + 2];
                const uint32_t b = t | (c << 3) | (st << 6);
                ids[cell] = (uint16_t)(t == 0 ? bb_rgb::ID_UNSEEN : (cell == 27 ? bb_rgb::ID_AGENT0 + b : b));   // cell 27 = view (3, 6): the agent
            }
        }
        __syncwarp();
        uint4 *dst = reinterpret_cast<uint4 *>(rgb + (size_t)env * RGB_IMG_BYTES);
#pragma unroll 4
        for (int k = 0; k < RGB_ITERS; k++) {
            const int i = lane + 32 * k;
            if (i < RGB_VEC) {
                const uint32_t w = s_where[k][lane];
                const uint2 a = __ldg(reinterpret_cast<const uint2 *>(lut + (size_t)ids[w & 0xFF] * bb_rgb::TILE_BYTES + ((w >> 8) & 0xFF)));
                const uint2 b = __ldg(reinterpret_cast<const uint2 *>(lut + (size_t)ids[(w >> 16) & 0xFF] * bb_rgb::TILE_BYTES + (w >> 24)));
                __stcs(dst + i, make_uint4(a.x, a.y, b.x, b.y));           // streaming store: the image is not read again here
            }
        }
        __syncwarp();                              // ids are rewritten for the next env
    }
}

// k_render_grid -- MiniGridEnv.render('rgb_array', highlight, tile_size) for selected envs: uint8[n_sel][H ts][W ts][3].
// A frame is a pure function of the env's current state in HBM (grid bytes, pose) and of the table of 430 tiles
// (rgb_tiles.h, render_grid_tiles) for the tile size: up to 484 grid bytes in, up to 5.9 MB (22 x 22 cells at 64 px) out,
// so the kernel is bound by its stores.  One CTA per frame at a time (grid-stride over the selection):
//   1. thread 0 reads the pose and computes the view's visibility (grid_render.cuh: col_load / col_see / vis_rows);
//   2. every thread turns cells into tile offsets in shared memory (grid_tile_id, <= 484 cells; grid_hidden_cell: the object a
//      PutNext*Carrying episode starts carrying is off the grid in the reference's state after reset);
//   3. the CTA streams the frame out as V-byte pieces of tile rows: consecutive threads write consecutive pieces (coalesced
//      streaming stores), each piece one load from the L2-resident table.  V = min(16, lowest set bit of ts) divides the tile
//      row (3 ts bytes) and hence the frame, so a piece never straddles a tile and every frame of the 16-byte-aligned output
//      starts V-aligned: 16-byte stores at ts 16 / 32 / 48 / 64, 8 at ts 8, single bytes at odd sizes (exact for every ts).
// Where a piece comes from: the (tile column, offset in the tile row) of piece j of a pixel row is the same for every row and
// env (s_pos, once per CTA); each thread walks its pieces with a fixed stride, so the pixel row / tile row it is in is
// advanced by additions -- the loop has no division.
constexpr int RG_THREADS = 256, RG_BLOCKS_PER_SM = 8, RG_IDS = 4096;

// which envs a launch renders: frame k of the launch is env first + k (all envs, in order) or id[k] (a list of up to RG_IDS,
// passed by value in the launch parameters: no device buffer, so calls on different streams share nothing)
struct RgRange { int32_t first; __device__ __forceinline__ int env(int k) const { return first + k; } };
struct RgList { int32_t id[RG_IDS]; __device__ __forceinline__ int env(int k) const { return id[k]; } };

template <int V> struct RgVec;
template <> struct RgVec<16> { typedef uint4 T; };
template <> struct RgVec<8> { typedef uint2 T; };
template <> struct RgVec<4> { typedef unsigned int T; };
template <> struct RgVec<2> { typedef unsigned short T; };
template <> struct RgVec<1> { typedef unsigned char T; };

template <int V, class Sel>
__global__ void __launch_bounds__(RG_THREADS)
k_render_grid(const LevelParams lp, const PoolPtrs P, const Sel sel, const int n_sel, uint8_t *__restrict__ out,
              const uint8_t *__restrict__ lut, const int ts, const int highlight)
{
    typedef typename RgVec<V>::T VT;
    extern __shared__ __align__(16) uint32_t s_rg[];
    __shared__ uint64_t s_vis;
    __shared__ int s_pose, s_hidden;
    const int W = lp.W, HW = lp.H * lp.W;
    const int tile_row = 3 * ts, tile_bytes = tile_row * ts;
    const int ppr = W * tile_row / V;                                  // pieces per pixel row
    const uint32_t total = (uint32_t)(lp.H * ts) * (uint32_t)ppr;      // pieces per frame
    const size_t frame_bytes = (size_t)total * V;
    uint32_t *s_off = s_rg;                                            // [HW] table byte offset of each cell's tile
    uint16_t *s_pos = reinterpret_cast<uint16_t *>(s_rg + HW);         // [ppr] tile column | byte offset in the tile row << 8
    for (int j = threadIdx.x; j < ppr; j += RG_THREADS) {
        const int c = j * V, tx = c / tile_row;
        s_pos[j] = (uint16_t)(tx | ((c - tx * tile_row) << 8));
    }
    // this thread's first piece (pixel row r0 = tile row cy0, row ty0 inside it; piece j0) and the stride in the same terms
    const int r0 = threadIdx.x / ppr, j0 = threadIdx.x - r0 * ppr;
    const int cy0 = r0 / ts, ty0 = r0 - cy0 * ts;
    const int dR = RG_THREADS / ppr, dJ = RG_THREADS - dR * ppr;
    const int dCy = dR / ts, dTy = dR - dCy * ts;
    for (int k = blockIdx.x; k < n_sel; k += gridDim.x) {
        const int env = sel.env(k);
        const uint8_t *grid = P.grid + (size_t)env * lp.cells_pad;
        if (threadIdx.x == 0) {
            const EnvHot h = P.hot[env];
            const int dir = h.dirflags & 3;
            s_pose = h.x | (h.y << 8) | (dir << 16);
            s_vis = grid_view_vis(lp, GridWords{ grid }, h.x, h.y, dir);
            s_hidden = lp.bonus == BN_PUTNEXT ? grid_hidden_cell(lp, h, P.obj[env], P.ins[env]) : -1;
        }
        __syncthreads();                          // (also: every thread is done with the previous frame's s_off)
        const int pose = s_pose, ax = pose & 0xFF, ay = (pose >> 8) & 0xFF, dir = pose >> 16;
        const uint64_t vis = s_vis;
        const int hidden = s_hidden;
        for (int c = threadIdx.x; c < HW; c += RG_THREADS) {
            const int y = c / W, x = c - y * W;
            const int cell = c == hidden ? CELL_EMPTY : grid[y * lp.rs_g + x];
            s_off[c] = (uint32_t)grid_tile_id(cell, x, y, ax, ay, dir, vis, highlight != 0) * (uint32_t)tile_bytes;
        }
        __syncthreads();                          // (also: thread 0 may overwrite s_vis / s_pose for the next frame)
        uint8_t *dst = out + (size_t)k * frame_bytes;
        int j = j0, ty = ty0, cyw = cy0 * W;
        for (uint32_t i = threadIdx.x; i < total; i += RG_THREADS) {
            const uint32_t pos = s_pos[j];
            const uint32_t src = s_off[cyw + (pos & 0xFF)] + (uint32_t)(ty * tile_row) + (pos >> 8);
            __stcs(reinterpret_cast<VT *>(dst + (size_t)i * V), __ldg(reinterpret_cast<const VT *>(lut + src)));
            j += dJ; ty += dTy; cyw += dCy * W;
            if (j >= ppr) { j -= ppr; ty++; }
            if (ty >= ts) { ty -= ts; cyw += W; }
        }
    }
}

__global__ void k_seed(const PoolPtrs P, const uint64_t *seeds, const int n)
{
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= n) return;
    RngRec r; r.seed = seeds[env]; r.draws = 0;
    P.rng[env] = r;
    P.locked_room[env] = 0xFF;
    P.tail[env] = P.head[env];                                 // empty ring: old levels belong to the old stream
    P.tail_pub[env] = P.head[env];
    P.attempts[env] = 0;
}

// ---- bb_pool_reset_envs: a new episode for the envs of an id list -----------------------------------------------------
// The ids (and the seeds) travel by value in the launch parameters, in chunks, as k_render_grid's do: calls on different
// streams share no device buffer.  Every kernel here touches the listed envs only, so a call costs O(n_sel), not O(n_envs).
constexpr int RS_IDS = 4096, RS_SEEDS = 2048;
struct RsList { int32_t id[RS_IDS]; };
struct RsSeeds { int32_t id[RS_SEEDS]; uint64_t seed[RS_SEEDS]; };

// k_seed for the listed envs
__global__ void k_seed_sel(const PoolPtrs P, const __grid_constant__ RsSeeds sel, const int n_sel)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_sel) return;
    const int env = sel.id[k];
    RngRec r; r.seed = sel.seed[k]; r.draws = 0;
    P.rng[env] = r;
    P.locked_room[env] = 0xFF;
    P.tail[env] = P.head[env];
    P.tail_pub[env] = P.head[env];
    P.attempts[env] = 0;
}

// k_gen_scan for the listed envs: the head snapshot of these envs only, onto the same four work lists (gen_count must be
// cleared before the first chunk; the chunks of one call append)
__global__ void k_gen_scan_sel(const PoolPtrs P, const __grid_constant__ RsList sel, const int n_sel, const int target)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int b = -1, env = 0;
    if (k < n_sel) {
        env = sel.id[k];
        const uint32_t hd = P.head[env];
        P.head_snap[env] = hd;
        const int missing = target - (int)(P.tail[env] - hd);
        if (missing > 0) b = missing >= 4 ? 3 : missing - 1;
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, b == q);
        if (m) {
            int base = 0;
            if (lane == 0) base = (int)atomicAdd(P.gen_count + q, (uint32_t)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            if (b == q) P.gen_list[(size_t)q * P.n + base + __popc(m & ((1u << lane) - 1u))] = env;
        }
    }
}

// publishes tail_pub for the listed envs, after the generation pass that wrote their rings has completed
__global__ void k_pub_sel(const PoolPtrs P, const __grid_constant__ RsList sel, const int n_sel)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n_sel) { const int env = sel.id[k]; P.tail_pub[env] = P.tail[env]; }
}

// the reset itself: reset8.cuh (also compiled, with the warp primitives emulated by threads, in tests/hostemu)
template <bool UNTR>
__global__ void __launch_bounds__(S8_THREADS)
k_reset8(const LevelParams lp, const PoolPtrs P, const __grid_constant__ RsList sel, const int n_sel, uint8_t *__restrict__ obs,
         int8_t *__restrict__ dirs)
{
    extern __shared__ __align__(16) uint8_t smem8[];
    reset8_role<PoolPtrs, UNTR>(lp, P, sel.id, n_sel, obs, dirs, smem8, threadIdx.x & 31, threadIdx.x >> 5, blockIdx.x);
}

// ====================================== host side ======================================
static thread_local char g_err[512] = "";
static int fail(const char *fmt, const char *a = "")
{
    snprintf(g_err, sizeof g_err, fmt, a);
    return 1;
}
#define CU(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return fail("CUDA error: %s", cudaGetErrorString(_e)); } while (0)

struct bb_pool;
static int ring_dry(const bb_pool *p);
#define BB_CHECK_RINGS(p) do { if (ring_dry(p)) return fail("a level ring ran dry (level generation fell behind the rollouts: counters()['errors'] > 0); the pool's episodes are no longer valid -- seed() it again, and use a deeper ring (BB_RING_DEPTH) or a shorter rollout"); } while (0)

struct GraphKey { const void *a, *o, *r, *d, *q; int T; int mode; };
constexpr int MAX_GEN_EVENTS = 40;

struct bb_pool {
    LevelParams lp;
    PoolPtrs P;
    int n, device, mode, num_warps, gen_blocks, gen_blocks_beside, gen_lanes, sm_count;
    // level supply schedule: ring depth D; k_gen is enqueued on gen_stream after every G-th step and
    // step s (counted from the last point at which a finished k_gen launched >= -G existed) waits for the
    // k_gen launched at >= s - D (see DESIGN.md section 4)
    int D, G, nev;
    bool gen_generic; int gen_fused; int gen_small_blocks, gen_budget, gen_min_active, refill_every; long long rollouts;   // BB_GEN_GENERIC=1: warp-per-level k_gen even for small levels
    bool no_persistent, after_rollout, gen_concurrent; int persist_max_cells;   // BB_NO_PERSISTENT=1: bb_pool_rollout always uses the per-step graph
    int room_kinds;                // level_spec_room_kinds(lp): bb_pool_rollout uses the specialised k_rollout instantiation (BB_ROLLOUT_SPEC=0: never)
    bool rollout_cta;              // bb_pool_rollout through k_rollout_cta (default on multi-room levels; BB_ROLLOUT_KERNEL=lane|cta)
    bool step_cols;                // BB_STEP_KERNEL=cols: k_step8 for every level (default: k_rollout with T = 1 on single-room grids)
    long long rel;
    cudaStream_t stream;           // internal stream: host-buffer API, seeding, graph capture origin
    cudaStream_t gen_stream;       // level generation runs here, concurrently with the steps
    cudaStream_t last_stream;      // the stream the previous call enqueued pool work on (order_after_last)
    cudaEvent_t ev_last;           // recorded on last_stream when a call arrives on another stream
    cudaEvent_t ev_fork, ev_join;
    cudaEvent_t gen_ev[MAX_GEN_EVENTS];
    long long gens_enqueued;       // k index of the next k_gen in the current epoch
    bool gen_outstanding;
    std::vector<void *> allocs;
    // host-buffer API staging
    int8_t *h_act; uint8_t *h_obs; float *h_rew; uint8_t *h_done; int8_t *h_dir;      // pinned
    uint8_t *d_rgb_lut;            // the 513 RGB tiles (rgb_tiles.h), rendered on first use
    uint8_t *d_grid_lut[bb_rgb::MAX_TILE_SIZE + 1];   // full-grid tile tables by tile size (rgb_tiles.h render_grid_tiles), rendered on first use
    int *h_err;                    // mapped: PoolPtrs::err_flag (a kernel found a level ring dry)
    int chain_cap;                 // BB_GEN_CHAIN_CAP: levels per env and pass of k_gen while the ring is at least half full (0 = no cap)
    int last_T, refill_cap;        // rollout length of the previous bb_pool_rollout call; BB_REFILL_EVERY as a cap for concurrent passes
    int fused_T;                   // longest T a fused rollout launch has guaranteed levels for (see bb_pool_rollout)
    int zerocopy, zc_level; const void *chk_rew, *chk_done, *chk_dir; bool chk_pinned; int8_t *zc_act; float *zc_rew; uint8_t *zc_done; int8_t *zc_dir; uint8_t *zc_obs;   // BB_HOST_ZEROCOPY
    int8_t *d_act; uint8_t *d_obs; float *d_rew; uint8_t *d_done; int8_t *d_dir;
    uint64_t *d_seeds;
    long long launches;
    cudaGraphExec_t graph; GraphKey gkey;
    cudaEvent_t ev[3];
    cudaEvent_t tev[4]; bool time_rollout, tev_kernel, tev_refill;
    const void *chk_obs; bool direct;            // bb_pool_step_host: caller buffers are page-locked       // bb_pool_rollout_timed
    int lz_state; int8_t *lz_act; float *lz_rew; uint8_t *lz_done;   // bb_pool_step_learner: 0 = not probed, 1 = mapped staging, 2 = copies
};

static int ring_dry(const bb_pool *p) { return p->h_err && *reinterpret_cast<volatile const int *>(p->h_err) != 0; }

template <typename T>
static int dalloc(bb_pool *p, T **out, size_t count)
{
    void *ptr = nullptr;
    size_t bytes = count * sizeof(T);
    if (bytes == 0) bytes = 16;
    CU(cudaMalloc(&ptr, bytes));
    CU(cudaMemset(ptr, 0, bytes));
    p->allocs.push_back(ptr);
    *out = reinterpret_cast<T *>(ptr);
    return 0;
}

static int make_params(const bb_level_spec *s, LevelParams *lp)
{
    const char *e = make_level_params(s, lp);
    return e ? fail("%s", e) : 0;
}

// the generator kernel of a pass, on the work lists a scan has built.  sel_envs > 0 (bb_pool_reset_envs): the lists hold at
// most that many envs, and the grid is no wider than they need
static void launch_gen_work(bb_pool *p, int target, cudaStream_t st, int max_rounds, int min_active, int min_keep, bool beside,
                            int chain_cap, int sel_envs = 0)
{
    if (p->lp.small && !p->gen_generic) {
        int blocks = p->gen_small_blocks;
        if (sel_envs > 0 && (sel_envs + GS_THREADS - 1) / GS_THREADS < blocks) blocks = (sel_envs + GS_THREADS - 1) / GS_THREADS;
        k_gen_small<<<blocks, GS_THREADS, 0, st>>>(p->lp, p->P, target, max_rounds, min_active, min_keep);
    } else {
        // blocks of a pass that runs BESIDE the rollout kernel (BB_GEN_BESIDE_BLOCKS_PER_SM, default = the full width): its
        // resident blocks delay the next rollout launch's CTAs, but a
        // narrower pass takes longer than the launches it overlaps and the join waits for it
        int blocks = beside && p->gen_blocks_beside < p->gen_blocks ? p->gen_blocks_beside : p->gen_blocks;
        if (sel_envs > 0 && (sel_envs + GEN_THREADS / 32 - 1) / (GEN_THREADS / 32) < blocks) blocks = (sel_envs + GEN_THREADS / 32 - 1) / (GEN_THREADS / 32);
        if (p->lp.kind == KIND_IMPUNLOCK || p->lp.kind == KIND_UNLOCK || p->lp.kind == KIND_BONUS) k_gen<true><<<blocks, GEN_THREADS, 0, st>>>(p->lp, p->P, p->n, target, p->gen_lanes, chain_cap);
        else k_gen<false><<<blocks, GEN_THREADS, 0, st>>>(p->lp, p->P, p->n, target, p->gen_lanes, chain_cap);
    }
}

static void launch_gen_kernel(bb_pool *p, int target, cudaStream_t st, int max_rounds = 0, int min_active = 0, bool snap_heads = false, int min_keep = 0, bool beside = false, int chain_cap = 0)
{
    cudaMemsetAsync(p->P.gen_count, 0, 8 * sizeof(uint32_t), st);      // list counters + work ticket
    k_gen_scan<<<(p->n + 255) / 256, 256, 0, st>>>(p->P, p->n, target, snap_heads ? 1 : 0);
    p->launches++;
    launch_gen_work(p, target, st, max_rounds, min_active, min_keep, beside, chain_cap);
}

// A SELECTED generation pass (bb_pool_reset_envs): tops the rings of the listed envs up to `target` levels -- their head
// snapshot (k_gen_scan_sel), the generator kernel launch_gen_kernel would pick, then their tail_pub.  Nothing else is read or
// written, so it costs what the listed envs need, whatever the pool size.
static void launch_gen_sel(bb_pool *p, const int32_t *ids, int32_t n_sel, int target, cudaStream_t st)
{
    cudaMemsetAsync(p->P.gen_count, 0, 8 * sizeof(uint32_t), st);
    RsList l;
    for (int32_t k0 = 0; k0 < n_sel; k0 += RS_IDS) {
        const int m = n_sel - k0 < RS_IDS ? n_sel - k0 : RS_IDS;
        memcpy(l.id, ids + k0, (size_t)m * sizeof(int32_t));
        k_gen_scan_sel<<<(m + 255) / 256, 256, 0, st>>>(p->P, l, m, target);
        p->launches++;
    }
    launch_gen_work(p, target, st, 0, 0, 0, false, 0, n_sel);
    p->launches++;
    for (int32_t k0 = 0; k0 < n_sel; k0 += RS_IDS) {
        const int m = n_sel - k0 < RS_IDS ? n_sel - k0 : RS_IDS;
        memcpy(l.id, ids + k0, (size_t)m * sizeof(int32_t));
        k_pub_sel<<<(m + 255) / 256, 256, 0, st>>>(p->P, l, m);
        p->launches++;
    }
}

// One generation pass on stream `st`: snapshot the consumption counters, reset the work-ticket counter,
// run k_gen, then publish the production counters.  The two small device-to-device copies replace
// __threadfence() pairs in the kernels (a gpu-scope fence invalidates the SM's whole L1).
static void launch_gen(bb_pool *p, cudaStream_t st)
{
    const int target = p->mode == BB_MODE_AUTORESET ? p->D : 1;
    const size_t nb = (size_t)p->n * sizeof(uint32_t);
    cudaMemcpyAsync(p->P.head_snap, p->P.head, nb, cudaMemcpyDeviceToDevice, st);
    launch_gen_kernel(p, target, st);
    cudaMemcpyAsync(p->P.tail_pub, p->P.tail, nb, cudaMemcpyDeviceToDevice, st);
    p->launches++;
}

static void launch_step(bb_pool *p, const void *actions, int action_bytes, uint8_t *obs, float *rew, uint8_t *done,
                        int8_t *dirs, int force_reset, cudaStream_t st)
{
    // single-room grids (<= 128 bytes of cells): the persistent kernel with T = 1 (coalesced state load / store);
    // everything else, and KIND_UNLOCK: k_step8, eight lanes per environment.  BB_STEP_KERNEL=cols forces k_step8.
    const bool cols = p->step_cols || p->lp.cells_pad > 128 || p->lp.kind == KIND_UNLOCK;
    if (!cols) {
        const size_t smem = (size_t)R_WARPS * rl_warp_words(p->lp) * 4;
        const int blocks = (p->n + 32 * R_WARPS - 1) / (32 * R_WARPS);
        if (action_bytes == 8) k_rollout<8><<<blocks, R_THREADS, smem, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, 1, p->mode, force_reset, 0, 0);
        else k_rollout<1><<<blocks, R_THREADS, smem, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, 1, p->mode, force_reset, 0, 0);
        p->launches++;
        return;
    }
    const int blocks8 = (p->n + 4 * S8_WARPS - 1) / (4 * S8_WARPS);
    const size_t sm8 = (size_t)S8_WARPS * 4 * (p->lp.cells_pad + S8_REC_FIXED) + (size_t)S8_WARPS * (S8_TILE_WORDS + 1) * 4;
    if (p->lp.kind == KIND_UNLOCK) {
        if (action_bytes == 8) k_step8<8, true><<<blocks8, S8_THREADS, sm8, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, p->mode, force_reset);
        else k_step8<1, true><<<blocks8, S8_THREADS, sm8, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, p->mode, force_reset);
    }
    else if (action_bytes == 8) k_step8<8><<<blocks8, S8_THREADS, sm8, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, p->mode, force_reset);
    else k_step8<1><<<blocks8, S8_THREADS, sm8, st>>>(p->lp, p->P, actions, obs, rew, done, dirs, p->n, p->mode, force_reset);
    p->launches++;
}

// ---- level-supply schedule ---------------------------------------------------------------------
// Invariant at a "sync point" (rel = 0): every k_gen enqueued so far is ordered before the next step
// and the most recent one was enqueued at relative step >= -G, i.e. every ring held >= D - G + ... levels.
// A k_gen that ran to completion after step t leaves every ring full with respect to the heads it saw,
// and one env consumes at most one level per step, so step s is safe once a k_gen enqueued at t >= s - D
// has finished.
static int sched_before_step(bb_pool *p, long long s, cudaStream_t st)
{
    if (p->mode != BB_MODE_AUTORESET) return 0;
    const long long need = s - p->D;                 // a finished k_gen enqueued at >= need is required
    if (need <= -(long long)p->G) return 0;          // the sync-point state suffices
    const long long k = need <= 0 ? 0 : (need + p->G - 1) / p->G;
    CU(cudaStreamWaitEvent(st, p->gen_ev[k % p->nev], 0));
    return 0;
}
static int sched_after_step(bb_pool *p, long long s, cudaStream_t st)
{
    if (p->mode != BB_MODE_AUTORESET) return 0;
    if (s % p->G != 0) return 0;
    const long long k = s / p->G;
    CU(cudaEventRecord(p->ev_fork, st));
    CU(cudaStreamWaitEvent(p->gen_stream, p->ev_fork, 0));
    launch_gen(p, p->gen_stream);
    CU(cudaEventRecord(p->gen_ev[k % p->nev], p->gen_stream));
    p->gen_outstanding = true;
    return 0;
}
// make `st` wait for every k_gen enqueued so far; afterwards rel = 0 is a sync point again
static int sched_join(bb_pool *p, cudaStream_t st)
{
    if (p->gen_outstanding) {
        CU(cudaEventRecord(p->ev_join, p->gen_stream));
        CU(cudaStreamWaitEvent(st, p->ev_join, 0));
        p->gen_outstanding = false;
    }
    p->rel = 0;
    return 0;
}

// The pool orders its own state between streams; the caller orders its own buffers.  Every entry point that enqueues work on
// the pool's state calls this first with the stream it enqueues on: when that differs from the stream of the previous such
// call, `st` waits for everything enqueued on the previous stream so far.  On the same stream it enqueues nothing.
static int order_after_last(bb_pool *p, cudaStream_t st)
{
    if (st == p->last_stream) return 0;
    CU(cudaEventRecord(p->ev_last, p->last_stream));
    CU(cudaStreamWaitEvent(st, p->ev_last, 0));
    p->last_stream = st;
    return 0;
}

// leaving rollout mode: the rings only hold >= D - T levels; make this a proper sync point again
static int sched_leave_rollout(bb_pool *p, cudaStream_t st)
{
    if (!p->after_rollout) return 0;
    p->rollouts = 0; p->fused_T = 0;
    if (sched_join(p, st)) return 1;
    if (p->mode == BB_MODE_AUTORESET) launch_gen(p, st);
    p->after_rollout = false;
    return 0;
}

// a tile table rasterised on the host, uploaded through the pool's internal stream (which only the pool's synchronous entry
// points use) and kept until bb_pool_destroy.  The copy has landed when this returns, so a kernel on any stream may read the
// table (a cudaMemcpy from pageable memory returns once the data is staged, and a non-blocking stream is not ordered after it).
static int upload_table(bb_pool *p, const std::vector<uint8_t> &h, uint8_t **out)
{
    void *d = nullptr;
    CU(cudaMalloc(&d, h.size()));
    p->allocs.push_back(d);
    CU(cudaMemcpyAsync(d, h.data(), h.size(), cudaMemcpyHostToDevice, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    *out = (uint8_t *)d;
    return 0;
}

// the device table of one tile size, rendered on first use
static int grid_table(bb_pool *p, int ts, const uint8_t **lut)
{
    if (!p->d_grid_lut[ts]) {
        std::vector<uint8_t> h((size_t)bb_rgb::GRID_TILES * ts * ts * 3);
        bb_rgb::render_grid_tiles(ts, h.data());
        if (upload_table(p, h, &p->d_grid_lut[ts])) return 1;
    }
    *lut = p->d_grid_lut[ts];
    return 0;
}

template <int V>
static void launch_render_grid(bb_pool *p, const int32_t *ids, int32_t n_sel, int ts, int highlight, uint8_t *rgb, cudaStream_t st,
                               const uint8_t *lut)
{
    const LevelParams &lp = p->lp;
    const size_t frame = (size_t)lp.H * lp.W * ts * ts * 3;
    const size_t smem = (size_t)lp.H * lp.W * 4 + (size_t)(lp.W * 3 * ts / V) * 2;
    const int cap = p->sm_count * RG_BLOCKS_PER_SM;
    if (!ids) {
        const RgRange r = { 0 };
        k_render_grid<V, RgRange><<<n_sel < cap ? n_sel : cap, RG_THREADS, smem, st>>>(lp, p->P, r, n_sel, rgb, lut, ts, highlight);
        p->launches++;
        return;
    }
    RgList l;
    for (int32_t k0 = 0; k0 < n_sel; k0 += RG_IDS) {
        const int m = n_sel - k0 < RG_IDS ? n_sel - k0 : RG_IDS;
        memcpy(l.id, ids + k0, (size_t)m * sizeof(int32_t));
        k_render_grid<V, RgList><<<m < cap ? m : cap, RG_THREADS, smem, st>>>(lp, p->P, l, m, rgb + (size_t)k0 * frame, lut, ts, highlight);
        p->launches++;
    }
}

extern "C" {

const char *bb_last_error(void) { return g_err; }

// inside bb_pool_create: a failing CUDA call releases everything allocated so far
#define CUP(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { fail("CUDA error: %s", cudaGetErrorString(_e)); bb_pool_destroy(p); return 1; } } while (0)
int bb_pool_create(const bb_level_spec *spec, int32_t n_envs, int32_t device, bb_pool **out)
{
    if (!spec || !out || n_envs < 1) return fail("bad arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail("no CUDA device available (the pool has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail("bad device index");
    CU(cudaSetDevice(device));
    bb_pool *p = new (std::nothrow) bb_pool();
    if (!p) return fail("out of memory");
    if (make_params(spec, &p->lp)) { delete p; return 1; }
    p->n = n_envs; p->device = device; p->mode = BB_MODE_AUTORESET;
    p->num_warps = (n_envs + 3) / 4 + 4;          // counter slots: the 8-lanes-per-env kernel has the most warps
    {
        cudaDeviceProp prop;
        CUP(cudaGetDeviceProperties(&prop, device));
        p->sm_count = prop.multiProcessorCount;
        int want = (n_envs + GEN_THREADS / 32 - 1) / (GEN_THREADS / 32);      // one warp per env at most
        int gen_per_sm = GEN_BLOCKS_PER_SM;
        if (const char *e = getenv("BB_GEN_BLOCKS_PER_SM")) { int v = atoi(e); if (v >= 1 && v <= 16) gen_per_sm = v; }
        int cap = prop.multiProcessorCount * gen_per_sm;             // a multiple of the SM count
        p->gen_blocks = want < cap ? want : cap;
        p->gen_lanes = 8;                                   // working lanes per warp of the lane-per-level k_gen
        if (const char *e = getenv("BB_GEN_LANES")) { int v = atoi(e); if (v >= 1 && v <= 32) p->gen_lanes = v; }
        int beside = GEN_BLOCKS_PER_SM;
        if (const char *e = getenv("BB_GEN_BESIDE_BLOCKS_PER_SM")) { int v = atoi(e); if (v >= 1 && v <= 16) beside = v; }
        p->gen_blocks_beside = prop.multiProcessorCount * beside;
        int per_sm = 4;
        if (const char *e = getenv("BB_GEN_SMALL_BLOCKS_PER_SM")) { int v = atoi(e); if (v >= 1 && v <= 16) per_sm = v; }
        p->gen_small_blocks = prop.multiProcessorCount * per_sm;
    }
    p->gen_generic = getenv("BB_GEN_GENERIC") != nullptr;
    p->gen_budget = 8;                                     // k_gen_small rounds (attempts per lane) per refill pass of bb_pool_rollout
    if (const char *e = getenv("BB_GEN_BUDGET")) p->gen_budget = atoi(e);
    p->lz_state = 0;
    p->zerocopy = 1; p->zc_level = 0; p->chk_rew = nullptr;
    if (const char *e = getenv("BB_HOST_ZEROCOPY")) p->zerocopy = atoi(e);
    p->gen_fused = 1;                                      // bb_pool_rollout on single-room levels: generator warp inside k_rollout (see bb_pool_rollout)
    if (const char *e = getenv("BB_GEN_FUSED")) p->gen_fused = atoi(e);
    p->gen_min_active = 16;                                // ... and a warp with fewer working lanes than this stops after its first round
    if (const char *e = getenv("BB_GEN_MIN_ACTIVE")) p->gen_min_active = atoi(e);
    p->refill_every = 2; p->rollouts = 0;                  // a refill pass every 2nd rollout launch: more envs per pass, more lanes busy
    p->refill_cap = 0; p->last_T = 0;
    p->chain_cap = 0;
    if (const char *e = getenv("BB_GEN_CHAIN_CAP")) { int v = atoi(e); if (v >= 0 && v <= 1024) p->chain_cap = v; }
    if (const char *e = getenv("BB_REFILL_EVERY")) { int v = atoi(e); if (v >= 1 && v <= 8) { p->refill_every = v; p->refill_cap = v; } }
    // ring depth: short single-room episodes (max_steps 64..128) end often and level generation has a long
    // rejection tail, so they get a deep ring; multi-room episodes last hundreds of steps
    // >= 3 x the 40-step rollout of bb_pool_rollout (one refill pass per two launches); for the per-step API one
    // generation pass per 32 steps (many levels per pass: a multi-room level is ~20-40 us of serial work for one warp)
    // multi-room levels (generation passes run BESIDE the rollouts on a side stream): twice the depth, so that one pass may
    // overlap several launches (bb_pool_rollout: a pass is joined D / 2T launches after it was forked)
    p->D = 128;
    if (p->lp.cells_pad > 256) {
        // 512 levels deep where the rings fit in a fifth of the free device memory (23 GB for 32 768 BossLevel envs), else 256 / 128:
        // a pass then has six (three, one) 40-step launches to finish in, and an env that ends ten episodes during a pass
        // (missions that are solved at reset) does not hold the next launch up
        size_t free_b = 0, total_b = 0;
        const size_t per_level = (size_t)p->lp.cells_pad + sizeof(EnvHot) + sizeof(ObjTab) + sizeof(InstrRec) + 2 * (size_t)p->lp.max_tokens;
        if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
        const size_t ring512 = (size_t)n_envs * 512 * per_level;
        p->D = ring512 <= free_b / 5 ? 512 : (ring512 / 2 <= free_b / 3 ? 256 : 128);
    }
    if (const char *e = getenv("BB_RING_DEPTH")) { int d = atoi(e); if (d >= 1 && d <= 1024) p->D = d; }
    p->G = p->D >= 64 ? 32 : (p->D >= 8 ? p->D / 4 : 1);
    if (const char *e = getenv("BB_GEN_PERIOD")) { int g = atoi(e); if (g >= 1 && g <= p->D) p->G = g; }
    p->nev = p->D / p->G + 3;
    if (p->nev > MAX_GEN_EVENTS) { p->nev = 0; bb_pool_destroy(p); return fail("ring depth / generation period too large"); }
    p->rel = 0; p->gens_enqueued = 0; p->gen_outstanding = false;
    p->step_cols = false;
    p->rollout_cta = p->lp.num_rows * p->lp.num_cols > 1;
    p->room_kinds = level_spec_room_kinds(p->lp);
    if (const char *e = getenv("BB_ROLLOUT_SPEC")) if (atoi(e) == 0) p->room_kinds = 0;
    if (const char *e = getenv("BB_ROLLOUT_KERNEL")) p->rollout_cta = !strcmp(e, "cta");
    p->no_persistent = getenv("BB_NO_PERSISTENT") != nullptr; p->after_rollout = false;
    p->persist_max_cells = 1152;                           // k_rollout stages up to 22 x 22 grids (2 x 43 KB of shared memory per CTA)
    if (const char *e = getenv("BB_PERSIST_MAX_CELLS")) p->persist_max_cells = atoi(e);
    p->gen_concurrent = p->lp.cells_pad > 256;
    if (const char *e = getenv("BB_GEN_CONCURRENT")) p->gen_concurrent = atoi(e) != 0;
    if (const char *e = getenv("BB_STEP_KERNEL")) p->step_cols = !strcmp(e, "cols");
    p->launches = 0; p->graph = nullptr; p->ev[0] = p->ev[1] = p->ev[2] = nullptr; p->tev[0] = p->tev[1] = p->tev[2] = p->tev[3] = nullptr; p->time_rollout = false; p->chk_obs = nullptr; p->direct = false;
    const LevelParams &lp = p->lp;
    const size_t n = (size_t)n_envs, D = (size_t)p->D;
    PoolPtrs &P = p->P;
    P.depth = p->D; P.n = n_envs;
    if (dalloc(p, &P.grid, n * lp.cells_pad) || dalloc(p, &P.hot, n) || dalloc(p, &P.obj, n) || dalloc(p, &P.ins, n) ||
        dalloc(p, &P.tok, n * lp.max_tokens) || dalloc(p, &P.rgrid, D * n * lp.cells_pad) || dalloc(p, &P.rhot, D * n) ||
        dalloc(p, &P.robj, D * n) || dalloc(p, &P.rins, D * n) || dalloc(p, &P.rtok, D * n * lp.max_tokens) ||
        dalloc(p, &P.head, n) || dalloc(p, &P.tail, n) || dalloc(p, &P.head_snap, n) || dalloc(p, &P.tail_pub, n) ||
        dalloc(p, &P.rng, n) || dalloc(p, &P.locked_room, n) || dalloc(p, &P.attempts, n) || dalloc(p, &P.last_reward, n) ||
        dalloc(p, &P.gen_count, 8) || dalloc(p, &P.gen_list, 4 * n) ||
        dalloc(p, &P.warp_counters, (size_t)p->num_warps * 4) ||
        dalloc(p, &p->d_act, n) || dalloc(p, &p->d_obs, n * OBS_BYTES) || dalloc(p, &p->d_rew, n) || dalloc(p, &p->d_done, n) ||
        dalloc(p, &p->d_dir, n) || dalloc(p, &p->d_seeds, n)) {
        bb_pool_destroy(p);
        return 1;
    }
    P.gen_ticket = P.gen_count + 4;                      // one memset clears the list counters and the work ticket
    CUP(cudaMemset(P.locked_room, 0xFF, n));
    CUP(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    {
        int lo = 0, hi = 0;
        CUP(cudaDeviceGetStreamPriorityRange(&lo, &hi));                  // lo = lowest priority
        CUP(cudaStreamCreateWithPriority(&p->gen_stream, cudaStreamNonBlocking, lo));
    }
    CUP(cudaFuncSetAttribute(k_rollout<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout<1, false, 1 << I_GOTO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout<1, false, 1 << I_GOTO>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_rollout<1, false, 1 << I_PICKUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout<1, false, 1 << I_PICKUP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_rollout_cta<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout_cta<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    CUP(cudaFuncSetAttribute(k_rollout_cta<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_rollout_cta<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    // kernels that run concurrently must ask for the SAME L1/shared-memory split: an SM drains before it changes
    // its carve-out, which serialised k_rollout and k_gen_small
    CUP(cudaFuncSetAttribute(k_rollout<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_rollout<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_gen_small, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_gen_scan, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_gen<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_gen<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_step8<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_step8<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_rollout<1, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_step8<1, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaFuncSetAttribute(k_step8<8, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUP(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
    CUP(cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming));
    CUP(cudaEventCreateWithFlags(&p->ev_last, cudaEventDisableTiming));
    p->last_stream = p->stream;
    for (int i = 0; i < p->nev; i++) CUP(cudaEventCreateWithFlags(&p->gen_ev[i], cudaEventDisableTiming));
    CUP(cudaMallocHost((void **)&p->h_act, n));
    CUP(cudaMallocHost((void **)&p->h_obs, n * OBS_BYTES));
    CUP(cudaMallocHost((void **)&p->h_rew, n * sizeof(float)));
    CUP(cudaMallocHost((void **)&p->h_done, n));
    CUP(cudaMallocHost((void **)&p->h_dir, n));
    CUP(cudaHostAlloc((void **)&p->h_err, sizeof(int), cudaHostAllocMapped));
    *p->h_err = 0;
    { void *d = nullptr; CUP(cudaHostGetDevicePointer(&d, p->h_err, 0)); P.err_flag = (int *)d; }
    // default seeds 0..n-1 so that an unseeded pool is still deterministic
    std::vector<uint64_t> seeds(n);
    for (size_t i = 0; i < n; i++) seeds[i] = i;
    if (bb_pool_seed(p, seeds.data())) { bb_pool_destroy(p); return 1; }
    *out = p;
    return 0;
}

#undef CUP

int bb_pool_destroy(bb_pool *p)
{
    if (!p) return 0;
    cudaSetDevice(p->device);
    cudaDeviceSynchronize();
    if (p->graph) cudaGraphExecDestroy(p->graph);
    for (int i = 0; i < 3; i++) if (p->ev[i]) cudaEventDestroy(p->ev[i]);
    for (int i = 0; i < 4; i++) if (p->tev[i]) cudaEventDestroy(p->tev[i]);
    for (int i = 0; i < p->nev; i++) if (p->gen_ev[i]) cudaEventDestroy(p->gen_ev[i]);
    if (p->ev_fork) cudaEventDestroy(p->ev_fork);
    if (p->ev_join) cudaEventDestroy(p->ev_join);
    if (p->ev_last) cudaEventDestroy(p->ev_last);
    for (void *a : p->allocs) cudaFree(a);
    if (p->h_act) cudaFreeHost(p->h_act);
    if (p->h_obs) cudaFreeHost(p->h_obs);
    if (p->h_rew) cudaFreeHost(p->h_rew);
    if (p->h_done) cudaFreeHost(p->h_done);
    if (p->h_dir) cudaFreeHost(p->h_dir);
    if (p->h_err) cudaFreeHost(p->h_err);
    if (p->stream) cudaStreamDestroy(p->stream);
    if (p->gen_stream) cudaStreamDestroy(p->gen_stream);
    delete p;
    return 0;
}

int bb_pool_seed(bb_pool *p, const uint64_t *seeds_host)
{
    if (!p || !seeds_host) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    CU(cudaDeviceSynchronize());
    p->gen_outstanding = false; p->rel = 0; p->after_rollout = false; p->fused_T = 0;
    p->last_stream = p->stream;                        // synchronous: nothing earlier is left to order after
    if (p->h_err) *p->h_err = 0;
    // stream-ordered copy: a synchronous cudaMemcpy from pageable memory may return before its last
    // chunk has landed, and p->stream (non-blocking) is not ordered after the legacy stream
    CU(cudaMemcpyAsync(p->d_seeds, seeds_host, (size_t)p->n * sizeof(uint64_t), cudaMemcpyHostToDevice, p->stream));
    k_seed<<<(p->n + 255) / 256, 256, 0, p->stream>>>(p->P, p->d_seeds, p->n);
    p->launches++;
    if (p->mode == BB_MODE_AUTORESET) launch_gen(p, p->stream);
    CU(cudaStreamSynchronize(p->stream));
    CU(cudaGetLastError());
    return 0;
}

int bb_pool_set_mode(bb_pool *p, int32_t mode)
{
    if (!p || (mode != BB_MODE_AUTORESET && mode != BB_MODE_FREEZE)) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    CU(cudaDeviceSynchronize());
    p->gen_outstanding = false; p->rel = 0; p->after_rollout = false;
    p->last_stream = p->stream;
    p->mode = mode;
    if (mode == BB_MODE_AUTORESET) { launch_gen(p, p->stream); CU(cudaStreamSynchronize(p->stream)); }
    if (p->graph) { cudaGraphExecDestroy(p->graph); p->graph = nullptr; }
    return 0;
}

int bb_pool_reset(bb_pool *p, uint8_t *obs_dev, int8_t *dir_dev, void *stream)
{
    if (!p || !obs_dev) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (order_after_last(p, st)) return 1;
    if (sched_join(p, st)) return 1;
    p->after_rollout = false; p->rollouts = 0;
    launch_gen(p, st);                                 // make sure every ring holds a level
    launch_step(p, nullptr, 1, obs_dev, nullptr, nullptr, dir_dev, 1, st);
    if (p->mode == BB_MODE_AUTORESET) launch_gen(p, st);      // rings full again: a sync point
    CU(cudaGetLastError());
    return 0;
}

// A new episode for the listed envs only (DESIGN.md section 4.8).  After the join no generation pass writes a ring; the listed
// envs are (re)seeded, a selected pass gives each listed ring its next level (freeze mode: 1, auto-reset: D), k_reset8 takes
// it, and in auto-reset mode a second selected pass tops the listed rings back up to D -- so every ring is as deep as the
// per-step schedule and the rollout paths assume (the unlisted ones are exactly as they were).
int bb_pool_reset_envs(bb_pool *p, const int32_t *env_ids_host, const uint64_t *seeds_host, int32_t n_sel, uint8_t *obs_dev,
                       int8_t *dir_dev, void *stream)
{
    if (!p || !obs_dev || n_sel < 0 || (n_sel > 0 && !env_ids_host)) return fail("bad arguments");
    if (n_sel > p->n) return fail("more env ids than envs: an id is repeated");
    for (int32_t k = 0; k < n_sel; k++)
        if (env_ids_host[k] < 0 || env_ids_host[k] >= p->n) return fail("env id out of range [0, n_envs)");
    {
        std::vector<int32_t> s(env_ids_host, env_ids_host + n_sel);
        std::sort(s.begin(), s.end());
        if (std::adjacent_find(s.begin(), s.end()) != s.end()) return fail("env ids must not repeat");
    }
    BB_CHECK_RINGS(p);
    CU(cudaSetDevice(p->device));
    if (n_sel == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (order_after_last(p, st)) return 1;
    if (sched_join(p, st)) return 1;                   // no generation pass is still writing rings on the side stream
    if (seeds_host) {
        RsSeeds s;
        for (int32_t k0 = 0; k0 < n_sel; k0 += RS_SEEDS) {
            const int m = n_sel - k0 < RS_SEEDS ? n_sel - k0 : RS_SEEDS;
            memcpy(s.id, env_ids_host + k0, (size_t)m * sizeof(int32_t));
            memcpy(s.seed, seeds_host + k0, (size_t)m * sizeof(uint64_t));
            k_seed_sel<<<(m + 255) / 256, 256, 0, st>>>(p->P, s, m);
            p->launches++;
        }
    }
    const int target = p->mode == BB_MODE_AUTORESET ? p->D : 1;
    launch_gen_sel(p, env_ids_host, n_sel, target, st);
    const size_t sm8 = (size_t)S8_WARPS * 4 * (p->lp.cells_pad + S8_REC_FIXED) + (size_t)S8_WARPS * (S8_TILE_WORDS + 1) * 4;
    RsList l;
    for (int32_t k0 = 0; k0 < n_sel; k0 += RS_IDS) {
        const int m = n_sel - k0 < RS_IDS ? n_sel - k0 : RS_IDS;
        memcpy(l.id, env_ids_host + k0, (size_t)m * sizeof(int32_t));
        const int blocks = (m + 4 * S8_WARPS - 1) / (4 * S8_WARPS);
        if (p->lp.kind == KIND_UNLOCK) k_reset8<true><<<blocks, S8_THREADS, sm8, st>>>(p->lp, p->P, l, m, obs_dev, dir_dev);
        else k_reset8<false><<<blocks, S8_THREADS, sm8, st>>>(p->lp, p->P, l, m, obs_dev, dir_dev);
        p->launches++;
    }
    if (p->mode == BB_MODE_AUTORESET) launch_gen_sel(p, env_ids_host, n_sel, p->D, st);
    CU(cudaGetLastError());
    return 0;
}

int bb_pool_step(bb_pool *p, const void *actions_dev, int32_t action_bytes, uint8_t *obs_dev, float *reward_dev,
                 uint8_t *done_dev, int8_t *dir_dev, void *stream)
{
    if (!p || !actions_dev || !obs_dev || !reward_dev || !done_dev) return fail("bad arguments");
    if (action_bytes != 1 && action_bytes != 8) return fail("action_bytes must be 1 or 8");
    BB_CHECK_RINGS(p);
    CU(cudaSetDevice(p->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (order_after_last(p, st)) return 1;
    if (sched_leave_rollout(p, st)) return 1;
    if (sched_before_step(p, p->rel, st)) return 1;
    launch_step(p, actions_dev, action_bytes, obs_dev, reward_dev, done_dev, dir_dev, 0, st);
    if (sched_after_step(p, p->rel, st)) return 1;
    p->rel++;
    CU(cudaGetLastError());
    return 0;
}

int bb_pool_step_timed(bb_pool *p, const void *actions_dev, int32_t action_bytes, uint8_t *obs_dev, float *reward_dev,
                       uint8_t *done_dev, int8_t *dir_dev, float *ms_step, float *ms_gen)
{
    if (!p || !actions_dev || !obs_dev || !reward_dev || !done_dev || !ms_step || !ms_gen) return fail("bad arguments");
    if (action_bytes != 1 && action_bytes != 8) return fail("action_bytes must be 1 or 8");
    BB_CHECK_RINGS(p);
    CU(cudaSetDevice(p->device));
    if (!p->ev[0]) for (int i = 0; i < 3; i++) CU(cudaEventCreate(&p->ev[i]));
    if (order_after_last(p, p->stream)) return 1;
    if (sched_join(p, p->stream)) return 1;
    p->after_rollout = false;
    launch_gen(p, p->stream);                           // rings full before the timed pair
    CU(cudaEventRecord(p->ev[0], p->stream));
    launch_step(p, actions_dev, action_bytes, obs_dev, reward_dev, done_dev, dir_dev, 0, p->stream);
    CU(cudaEventRecord(p->ev[1], p->stream));
    launch_gen(p, p->stream);                           // one step's worth of refills, timed in isolation
    CU(cudaEventRecord(p->ev[2], p->stream));
    CU(cudaEventSynchronize(p->ev[2]));
    CU(cudaEventElapsedTime(ms_step, p->ev[0], p->ev[1]));
    CU(cudaEventElapsedTime(ms_gen, p->ev[1], p->ev[2]));
    return 0;
}

// T steps per launch.  Small grids with a ring deep enough (D >= 2T): the persistent kernel k_rollout, with
// k_gen refilling on the side stream what the PREVIOUS launch consumed (head snapshot taken before this
// launch starts, so generation never writes a slot this launch may read).  Otherwise: a captured CUDA graph
// of T per-step launches with the k_gen branch forked and joined inside.
static int rollout_graph(bb_pool *p, const int8_t *actions_dev, int32_t T, uint8_t *obs_dev, float *reward_dev,
                         uint8_t *done_dev, int8_t *dir_dev, cudaStream_t user);

int bb_pool_rollout(bb_pool *p, const int8_t *actions_dev, int32_t T, uint8_t *obs_dev, float *reward_dev,
                    uint8_t *done_dev, int8_t *dir_dev, void *stream)
{
    if (!p || !actions_dev || !obs_dev || !reward_dev || !done_dev || T < 1) return fail("bad arguments");
    BB_CHECK_RINGS(p);
    CU(cudaSetDevice(p->device));
    cudaStream_t user = (cudaStream_t)stream;
    if (order_after_last(p, user)) return 1;          // before rollout_graph captures on the internal stream
    // Level supply of the persistent kernels.  In-stream refill passes (single-room levels without the fused generator warp):
    // one pass per `refill_every` launches, needs D >= (refill_every + 1) T.  Concurrent passes (multi-room levels: k_gen on
    // the side stream, beside the rollouts): a pass is forked at every R-th launch from a head snapshot taken before that
    // launch and joined R launches later, so it overlaps R launches; it tops every ring up to D relative to its snapshot,
    // the R launches it overlaps and the R launches until the next pass is joined consume at most 2 R T: R = D / 2T.
    // Chain cap (k_gen levels): a pass gives a ring that is at least half full at most `chain_cap` levels, a ring below half
    // is filled up.  Then every ring holds >= D/2 - RT levels at a fork (induction over the passes), its additions may be
    // published as late as the join, R launches later: D/2 - 2RT >= 0, R = D / 4T.
    const bool conc = p->gen_concurrent && p->mode == BB_MODE_AUTORESET;
    const bool kgen_levels = !(p->lp.small && !p->gen_generic);
    const int cap = kgen_levels && p->chain_cap > 0 && p->D >= 4 * T ? p->chain_cap : 0;
    int R = p->refill_every;
    if (conc) R = p->D / (2 * T);
    if (cap) R = p->D / (4 * T);
    if (conc || cap) { if (R > 8) R = 8; if (p->refill_cap > 0 && R > p->refill_cap) R = p->refill_cap; }
    const bool persistent = p->lp.cells_pad <= p->persist_max_cells && !p->no_persistent &&
                            (p->mode == BB_MODE_FREEZE || (conc || cap ? R >= 1 : p->D >= (p->refill_every + 1) * T));
    if (!persistent) return rollout_graph(p, actions_dev, T, obs_dev, reward_dev, done_dev, dir_dev, user);
    if (T != p->last_T) { p->rollouts = 0; p->last_T = T; }       // a different rollout length restarts the refill schedule
    const bool refill_slot = (p->rollouts % R) == 0;
    // join what is outstanding: always for in-stream refills / ManyEnvs mode; for concurrent passes only where the next one forks
    if (!conc || refill_slot) { if (sched_join(p, user)) return 1; }
    const size_t smem = (size_t)R_WARPS * rl_warp_words(p->lp) * 4;
    const int blocks = (p->n + 32 * R_WARPS - 1) / (32 * R_WARPS);
    // Single-room levels: FUSED -- a generator warp inside every CTA of k_rollout refills the rings of the CTA's envs
    // while the stepping warps run (no refill pass at all).  It guarantees >= 2T levels per ring at the end of a
    // launch (must_complete rule in the kernel), so the next launch cannot run dry; needs D > 2T.
    // One generator warp per 64 envs keeps up while an env needs at most ~1.5 levels per launch: episodes last up to
    // max_steps = room_size^2 steps, so fused when 3 max_steps >= 2 T (on the
    // smaller rooms the GPU-wide refill passes win).  BB_GEN_FUSED=0/1/2:
    // never / by this rule (default) / whenever possible.
    const bool fused = !p->rollout_cta && p->gen_fused != 0 && (p->gen_fused == 2 || 3 * p->lp.nav_time_maze >= 2 * T) &&
                       p->lp.small && !p->gen_generic && !p->gen_concurrent && p->mode == BB_MODE_AUTORESET &&
                       p->D >= 2 * T + 8 && !getenv("BB_DEBUG_NO_REFILL");
    // a fused launch leaves >= T levels in every ring (must-complete rule in the kernel: >= 2T before they are consumed), which
    // covers the next launch only if it is not longer: a longer one tops every ring up first (blocking pass)
    if (fused && T > p->fused_T) launch_gen(p, user);
    p->fused_T = fused ? T : 0;
    // otherwise one refill pass serves `refill_every` launches (more envs per pass = more lanes busy in k_gen_small)
    const bool refill = !fused && p->mode == BB_MODE_AUTORESET && !getenv("BB_DEBUG_NO_REFILL") && refill_slot;
    p->rollouts++;
    const bool dbg_timing = p->time_rollout;
    cudaEvent_t *dbg_ev = p->tev;
    if (dbg_timing && !dbg_ev[0]) for (int i = 0; i < 4; i++) CU(cudaEventCreate(&dbg_ev[i]));
    const size_t nb = (size_t)p->n * sizeof(uint32_t);
    // Small levels: refill in-stream, right before the stepping kernel, with a bounded iteration budget.  Running
    // k_gen_small on the side stream BESIDE k_rollout does not pay: both are issue/latency bound on the same SMs.  Multi-room levels:
    // k_gen (one warp per level, thousands of levels per pass) runs on the side stream beside k_rollout_cta, forked every R-th
    // launch and joined R launches later (see the top of this function).
    // BB_GEN_CONCURRENT=0/1 overrides.
    const bool gen_serial = !p->gen_concurrent;
    if (refill && gen_serial) {
        if (dbg_timing) cudaEventRecord(dbg_ev[2], user);
        const bool fused_snap = p->lp.small && !p->gen_generic;       // k_gen_scan takes the head snapshot itself
        if (!fused_snap) CU(cudaMemcpyAsync(p->P.head_snap, p->P.head, nb, cudaMemcpyDeviceToDevice, user));
        launch_gen_kernel(p, p->D, user, p->gen_budget, p->gen_min_active, fused_snap, p->refill_every * T, false, cap);
        cudaMemcpyAsync(p->P.tail_pub, p->P.tail, nb, cudaMemcpyDeviceToDevice, user);
        if (dbg_timing) { cudaEventRecord(dbg_ev[3], user); p->tev_refill = true; }
        p->launches++;
    } else if (refill) {
        // fork point: the head snapshot k_gen will work from (levels consumed before this launch)
        CU(cudaMemcpyAsync(p->P.head_snap, p->P.head, nb, cudaMemcpyDeviceToDevice, user));
        CU(cudaEventRecord(p->ev_fork, user));
    }
    if (dbg_timing) cudaEventRecord(dbg_ev[0], user);
    if (p->rollout_cta) {                  // multi-room levels: 32 envs per CTA, step phase + 4-lanes-per-env observation phase
        const int blocks_c = (p->n + RC_ENVS - 1) / RC_ENVS;
        const size_t smc = (size_t)rc2_cta_words(p->lp) * 4;
        if (p->lp.kind == KIND_UNLOCK) k_rollout_cta<true><<<blocks_c, RC_THREADS, smc, user>>>(p->lp, p->P, actions_dev, obs_dev, reward_dev, done_dev, dir_dev, p->n, T, p->mode);
        else k_rollout_cta<false><<<blocks_c, RC_THREADS, smc, user>>>(p->lp, p->P, actions_dev, obs_dev, reward_dev, done_dev, dir_dev, p->n, T, p->mode);
    }
    else {
        const int gr = fused ? (p->gen_budget > 0 ? p->gen_budget : 1 << 20) : 0, gm = fused ? p->gen_min_active : 0;
        const int threads = fused ? R_THREADS_FUSED : R_THREADS;
        const size_t sm = fused ? smem + RG_AREA_WORDS * 4 : smem;
#define BB_LAUNCH_ROLLOUT(...) k_rollout<__VA_ARGS__><<<blocks, threads, sm, user>>>(p->lp, p->P, actions_dev, obs_dev, reward_dev, done_dev, dir_dev, p->n, T, p->mode, 0, gr, gm)
        if (p->lp.kind == KIND_UNLOCK) BB_LAUNCH_ROLLOUT(1, true);                         // (never fused: not a small level)
        else if (p->room_kinds == (1 << I_GOTO)) BB_LAUNCH_ROLLOUT(1, false, 1 << I_GOTO);
        else if (p->room_kinds == (1 << I_PICKUP)) BB_LAUNCH_ROLLOUT(1, false, 1 << I_PICKUP);
        else BB_LAUNCH_ROLLOUT(1);
#undef BB_LAUNCH_ROLLOUT
    }
    if (dbg_timing) { cudaEventRecord(dbg_ev[1], user); p->tev_kernel = true; }
    p->launches++;
    if (refill && !gen_serial) {
        CU(cudaStreamWaitEvent(p->gen_stream, p->ev_fork, 0));
        if (dbg_timing) cudaEventRecord(dbg_ev[2], p->gen_stream);
        launch_gen_kernel(p, p->D, p->gen_stream, p->gen_budget, p->gen_min_active, false, (p->refill_every + 1) * T, true, cap);      // bounded: runs beside k_rollout
        cudaMemcpyAsync(p->P.tail_pub, p->P.tail, nb, cudaMemcpyDeviceToDevice, p->gen_stream);
        if (dbg_timing) { cudaEventRecord(dbg_ev[3], p->gen_stream); p->tev_refill = true; }
        p->gen_outstanding = true;
        p->launches++;
    }
    p->rel = 0;
    p->after_rollout = true;                           // a per-step call that follows tops the rings up first
    CU(cudaGetLastError());
    return 0;
}

int bb_pool_rollout_timed(bb_pool *p, const int8_t *actions_dev, int32_t T, uint8_t *obs_dev, float *reward_dev,
                          uint8_t *done_dev, int8_t *dir_dev, float *ms_rollout_kernel, float *ms_refill)
{
    if (!p || !ms_rollout_kernel || !ms_refill) return fail("bad arguments");
    *ms_rollout_kernel = 0; *ms_refill = 0;
    p->time_rollout = true; p->tev_kernel = false; p->tev_refill = false;
    const int rc = bb_pool_rollout(p, actions_dev, T, obs_dev, reward_dev, done_dev, dir_dev, p->stream);
    p->time_rollout = false;
    if (rc) return rc;
    CU(cudaStreamSynchronize(p->stream));
    CU(cudaDeviceSynchronize());
    if (p->tev[0] && p->tev_kernel) {
        CU(cudaEventElapsedTime(ms_rollout_kernel, p->tev[0], p->tev[1]));
        if (p->tev_refill) CU(cudaEventElapsedTime(ms_refill, p->tev[2], p->tev[3]));
    }
    return 0;
}

static int rollout_graph(bb_pool *p, const int8_t *actions_dev, int32_t T, uint8_t *obs_dev, float *reward_dev,
                         uint8_t *done_dev, int8_t *dir_dev, cudaStream_t user)
{
    GraphKey key = { actions_dev, obs_dev, reward_dev, done_dev, dir_dev, T, p->mode };
    if (!p->graph || memcmp(&key, &p->gkey, sizeof key) != 0) {
        if (p->graph) { cudaGraphExecDestroy(p->graph); p->graph = nullptr; }
        cudaGraph_t g;
        const size_t n = (size_t)p->n;
        const long long l0 = p->launches;
        const bool saved_out = p->gen_outstanding;
        // the generation branch forks from and joins back into the origin stream inside the capture
        CU(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
        p->gen_outstanding = false;
        for (int t = 0; t < T; t++) {
            if (sched_before_step(p, t, p->stream)) return 1;
            launch_step(p, actions_dev + t * n, 1, obs_dev + t * n * OBS_BYTES, reward_dev + t * n, done_dev + t * n,
                        dir_dev ? dir_dev + t * n : nullptr, 0, p->stream);
            if (sched_after_step(p, t, p->stream)) return 1;
        }
        if (p->gen_outstanding) {
            CU(cudaEventRecord(p->ev_join, p->gen_stream));
            CU(cudaStreamWaitEvent(p->stream, p->ev_join, 0));
        }
        CU(cudaStreamEndCapture(p->stream, &g));
        p->gen_outstanding = saved_out;
        p->launches = l0;
        CU(cudaGraphInstantiate(&p->graph, g, 0));
        CU(cudaGraphDestroy(g));
        p->gkey = key;
    }
    if (sched_leave_rollout(p, user)) return 1;
    if (sched_join(p, user)) return 1;                  // per-step k_gens still in flight come first
    CU(cudaGraphLaunch(p->graph, user));
    p->rel = 0;                                         // the graph ends with its k_gens joined: a sync point
    p->launches += (long long)T + (p->mode == BB_MODE_AUTORESET ? (T + p->G - 1) / p->G : 0);
    return 0;
}

static bool is_pinned(const void *ptr)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

int bb_pool_step_host(bb_pool *p, const int8_t *actions_host, uint8_t *obs_host, float *reward_host,
                      uint8_t *done_host, int8_t *dir_host)
{
    if (!p || !actions_host || !obs_host || !reward_host || !done_host) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    const size_t n = (size_t)p->n;
    // page-locked caller buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory) are the DMA targets
    // themselves; pageable ones go through the pool's pinned staging buffers + a host memcpy
    // the probe result is cached per (obs, reward, done, dir) pointer set; the observation buffer is re-probed on every call
    // (a buffer freed and reallocated at the same address as pageable memory must not keep its old mapping)
    const bool obs_pinned = is_pinned(obs_host);
    if (obs_host != p->chk_obs || reward_host != p->chk_rew || done_host != p->chk_done || dir_host != p->chk_dir || obs_pinned != p->chk_pinned) {
        p->chk_obs = obs_host; p->chk_rew = reward_host; p->chk_done = done_host; p->chk_dir = dir_host; p->chk_pinned = obs_pinned;
        p->direct = obs_pinned && is_pinned(reward_host) && is_pinned(done_host) && (!dir_host || is_pinned(dir_host));
        // BB_HOST_ZEROCOPY (page-locked caller buffers only): 1 = the step kernel reads the actions from the pool's pinned
        // staging buffer and writes reward / done / direction straight into the caller's buffers over PCIe (mapped host
        // memory: 1 H2D + 3 small D2H copies less per step); 2 = the observations too (no copy at all)
        p->zc_level = 0;
        if (p->direct && p->zerocopy > 0) {
            void *da = nullptr, *dr = nullptr, *dd = nullptr, *dq = nullptr, *dobs = nullptr;
            bool ok = cudaHostGetDevicePointer(&da, p->h_act, 0) == cudaSuccess && cudaHostGetDevicePointer(&dr, reward_host, 0) == cudaSuccess &&
                      cudaHostGetDevicePointer(&dd, done_host, 0) == cudaSuccess && (!dir_host || cudaHostGetDevicePointer(&dq, dir_host, 0) == cudaSuccess);
            if (ok && p->zerocopy > 1) ok = cudaHostGetDevicePointer(&dobs, obs_host, 0) == cudaSuccess;
            if (ok) { p->zc_level = p->zerocopy > 1 ? 2 : 1; p->zc_act = (int8_t *)da; p->zc_rew = (float *)dr; p->zc_done = (uint8_t *)dd; p->zc_dir = (int8_t *)dq; p->zc_obs = (uint8_t *)dobs; }
            else cudaGetLastError();
        }
    }
    const bool direct = p->direct;
    const int zc = p->zc_level;
    if (order_after_last(p, p->stream)) return 1;
    memcpy(p->h_act, actions_host, n);
    if (!zc) CU(cudaMemcpyAsync(p->d_act, p->h_act, n, cudaMemcpyHostToDevice, p->stream));
    if (sched_leave_rollout(p, p->stream)) return 1;
    if (sched_before_step(p, p->rel, p->stream)) return 1;
    if (zc) launch_step(p, p->zc_act, 1, zc > 1 ? p->zc_obs : p->d_obs, p->zc_rew, p->zc_done, dir_host ? p->zc_dir : p->d_dir, 0, p->stream);
    else launch_step(p, p->d_act, 1, p->d_obs, p->d_rew, p->d_done, p->d_dir, 0, p->stream);
    if (sched_after_step(p, p->rel, p->stream)) return 1;
    p->rel++;
    if (zc < 2) CU(cudaMemcpyAsync(direct ? obs_host : p->h_obs, p->d_obs, n * OBS_BYTES, cudaMemcpyDeviceToHost, p->stream));
    if (!zc) {
        CU(cudaMemcpyAsync(direct ? (void *)reward_host : (void *)p->h_rew, p->d_rew, n * sizeof(float), cudaMemcpyDeviceToHost, p->stream));
        CU(cudaMemcpyAsync(direct ? done_host : p->h_done, p->d_done, n, cudaMemcpyDeviceToHost, p->stream));
        if (!direct || dir_host) CU(cudaMemcpyAsync(direct ? dir_host : p->h_dir, p->d_dir, n, cudaMemcpyDeviceToHost, p->stream));
    }
    CU(cudaStreamSynchronize(p->stream));
    BB_CHECK_RINGS(p);
    if (!direct) {
        memcpy(obs_host, p->h_obs, n * OBS_BYTES);
        memcpy(reward_host, p->h_rew, n * sizeof(float));
        memcpy(done_host, p->h_done, n);
        if (dir_host) memcpy(dir_host, p->h_dir, n);
    }
    return 0;
}

// The learner's step (babyai_b200/learner.py): actions arrive from the host (base.py:144 hands numpy), the observation
// stays on the device, reward / done go back to the host (base.py:158-179 reads them there).  The step kernel reads the
// actions from and writes reward / done to the pool's page-locked staging buffers over PCIe (mapped memory), so the
// call is: one host memcpy, one kernel, one stream synchronise, two host memcpys -- no copy-engine transfers at all.
int bb_pool_step_learner(bb_pool *p, const int8_t *actions_host, uint8_t *obs_dev, float *reward_host, uint8_t *done_host,
                         int8_t *dir_dev, void *stream)
{
    if (!p || !actions_host || !obs_dev || !reward_host || !done_host) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)p->n;
    if (p->lz_state == 0) {
        void *da = nullptr, *dr = nullptr, *dd = nullptr;
        const bool ok = p->zerocopy > 0 && cudaHostGetDevicePointer(&da, p->h_act, 0) == cudaSuccess &&
                        cudaHostGetDevicePointer(&dr, p->h_rew, 0) == cudaSuccess && cudaHostGetDevicePointer(&dd, p->h_done, 0) == cudaSuccess;
        if (ok) { p->lz_state = 1; p->lz_act = (int8_t *)da; p->lz_rew = (float *)dr; p->lz_done = (uint8_t *)dd; }
        else { cudaGetLastError(); p->lz_state = 2; }
    }
    const bool zc = p->lz_state == 1;
    if (order_after_last(p, st)) return 1;
    memcpy(p->h_act, actions_host, n);
    if (!zc) CU(cudaMemcpyAsync(p->d_act, p->h_act, n, cudaMemcpyHostToDevice, st));
    if (sched_leave_rollout(p, st)) return 1;
    if (sched_before_step(p, p->rel, st)) return 1;
    launch_step(p, zc ? p->lz_act : p->d_act, 1, obs_dev, zc ? p->lz_rew : p->d_rew, zc ? p->lz_done : p->d_done, dir_dev, 0, st);
    if (sched_after_step(p, p->rel, st)) return 1;
    p->rel++;
    if (!zc) {
        CU(cudaMemcpyAsync(p->h_rew, p->d_rew, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(p->h_done, p->d_done, n, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    BB_CHECK_RINGS(p);
    memcpy(reward_host, p->h_rew, n * sizeof(float));
    memcpy(done_host, p->h_done, n);
    return 0;
}

int bb_pool_reset_host(bb_pool *p, uint8_t *obs_host, int8_t *dir_host)
{
    if (!p || !obs_host) return fail("bad arguments");
    const size_t n = (size_t)p->n;
    if (bb_pool_reset(p, p->d_obs, p->d_dir, p->stream)) return 1;
    CU(cudaMemcpyAsync(p->h_obs, p->d_obs, n * OBS_BYTES, cudaMemcpyDeviceToHost, p->stream));
    CU(cudaMemcpyAsync(p->h_dir, p->d_dir, n, cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    memcpy(obs_host, p->h_obs, n * OBS_BYTES);
    if (dir_host) memcpy(dir_host, p->h_dir, n);
    return 0;
}

int bb_rgb_tiles(uint8_t *tiles_host)
{
    if (!tiles_host) return fail("bad arguments");
    bb_rgb::render_all_tiles(tiles_host);
    return 0;
}

int bb_pool_render_rgb(bb_pool *p, const uint8_t *obs_dev, uint8_t *rgb_dev, int32_t n_obs, void *stream)
{
    if (!p || !obs_dev || !rgb_dev || n_obs < 0) return fail("bad arguments");
    if ((((uintptr_t)rgb_dev) & 15) != 0) return fail("rgb_dev must be 16-byte aligned");
    CU(cudaSetDevice(p->device));
    if (!p->d_rgb_lut) {                                   // rasterise the tile table once (host), keep it on the device
        std::vector<uint8_t> lut((size_t)bb_rgb::N_TILES * bb_rgb::TILE_BYTES);
        bb_rgb::render_all_tiles(lut.data());
        if (upload_table(p, lut, &p->d_rgb_lut)) return 1;
    }
    if (n_obs == 0) return 0;
    int blocks = (n_obs + RGB_THREADS / 32 - 1) / (RGB_THREADS / 32);
    if (blocks > p->sm_count * 8) blocks = p->sm_count * 8;          // grid-stride over the envs: a multiple of the SM count
    k_render_rgb<<<blocks, RGB_THREADS, 0, (cudaStream_t)stream>>>(obs_dev, rgb_dev, p->d_rgb_lut, n_obs);
    p->launches++;
    CU(cudaGetLastError());
    return 0;
}

int bb_grid_tiles(int32_t tile_size, uint8_t *tiles_host)
{
    if (!tiles_host || tile_size < 1 || tile_size > bb_rgb::MAX_TILE_SIZE) return fail("bad arguments (tile_size must be 1..64)");
    bb_rgb::render_grid_tiles(tile_size, tiles_host);
    return 0;
}

int bb_pool_render_grid(bb_pool *p, const int32_t *env_ids_host, int32_t n_sel, int32_t tile_size, int32_t highlight,
                        uint8_t *rgb_dev, void *stream)
{
    if (!p || n_sel < 0 || (n_sel > 0 && !rgb_dev)) return fail("bad arguments");
    if (tile_size < 1 || tile_size > bb_rgb::MAX_TILE_SIZE) return fail("tile_size must be 1..64");
    if (!env_ids_host && n_sel != p->n) return fail("env_ids_host = NULL renders every env: n_sel must equal n_envs");
    if ((((uintptr_t)rgb_dev) & 15) != 0) return fail("rgb_dev must be 16-byte aligned");
    if (env_ids_host)
        for (int32_t k = 0; k < n_sel; k++)
            if (env_ids_host[k] < 0 || env_ids_host[k] >= p->n) return fail("env id out of range [0, n_envs)");
    CU(cudaSetDevice(p->device));
    const uint8_t *lut = nullptr;
    if (grid_table(p, tile_size, &lut)) return 1;
    if (n_sel == 0) return 0;
    // the widest store that divides the tile row (3 ts bytes): the lowest set bit of ts, at most 16
    const int v = tile_size & -tile_size;
    cudaStream_t st = (cudaStream_t)stream;
    if (order_after_last(p, st)) return 1;
    const int hl = highlight ? 1 : 0;
    if (v >= 16) launch_render_grid<16>(p, env_ids_host, n_sel, tile_size, hl, rgb_dev, st, lut);
    else if (v == 8) launch_render_grid<8>(p, env_ids_host, n_sel, tile_size, hl, rgb_dev, st, lut);
    else if (v == 4) launch_render_grid<4>(p, env_ids_host, n_sel, tile_size, hl, rgb_dev, st, lut);
    else if (v == 2) launch_render_grid<2>(p, env_ids_host, n_sel, tile_size, hl, rgb_dev, st, lut);
    else launch_render_grid<1>(p, env_ids_host, n_sel, tile_size, hl, rgb_dev, st, lut);
    CU(cudaGetLastError());
    return 0;
}

int bb_pool_mission_tokens(bb_pool *p, const int16_t **tokens_dev, int32_t *max_len)
{
    if (!p || !tokens_dev || !max_len) return fail("bad arguments");
    *tokens_dev = p->P.tok; *max_len = p->lp.max_tokens;
    return 0;
}

static const char *VOCAB[W_COUNT] = {
    "", "go", "to", "pick", "up", "open", "put", "next", "the", "a", "object",
    "red", "green", "blue", "purple", "yellow", "grey", "box", "ball", "key", "door",
    "in", "front", "of", "you", "behind", "on", "your", "left", "right", "then", "after", "and" };

int32_t bb_vocab_size(void) { return W_COUNT - 1; }
const char *bb_vocab_word(int32_t id) { return (id >= 0 && id < W_COUNT) ? VOCAB[id] : ""; }

int bb_pool_get_state(bb_pool *p, int32_t env, uint8_t *grid_host, int32_t *info)
{
    if (!p || env < 0 || env >= p->n || !grid_host || !info) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    CU(cudaDeviceSynchronize());
    EnvHot h; ObjTab ot; RngRec r; uint32_t att;
    {
        const LevelParams &lp = p->lp;
        std::vector<uint8_t> raw((size_t)lp.cells_pad);
        CU(cudaMemcpy(raw.data(), p->P.grid + (size_t)env * lp.cells_pad, raw.size(), cudaMemcpyDeviceToHost));
        for (int y = 0; y < lp.H; y++)
            for (int x = 0; x < lp.W; x++) {
                grid_host[y * lp.W + x] = raw[(size_t)y * lp.rs_g + x];
                if (raw[(size_t)lp.gt_off + x * lp.rs_t + y] != raw[(size_t)y * lp.rs_g + x]) return fail("internal: row-major / column-major grid copies differ");
            }
    }
    CU(cudaMemcpy(&h, p->P.hot + env, sizeof h, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&ot, p->P.obj + env, sizeof ot, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&r, p->P.rng + env, sizeof r, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&att, p->P.attempts + env, sizeof att, cudaMemcpyDeviceToHost));
    info[0] = h.x; info[1] = h.y; info[2] = h.dirflags & 3;
    info[3] = h.carry == NO_OBJ ? 0 : (p->lp.kind == KIND_UNLOCK && (h.carry & CARRY_UNTRACKED)) ? (h.carry & 0x3F) : ot.tc[h.carry];
    info[4] = h.step_count; info[5] = h.max_steps;
    info[6] = (int32_t)(r.draws & 0x7FFFFFFF); info[7] = (int32_t)att;
    return 0;
}

int32_t bb_pool_width(const bb_pool *p) { return p ? p->lp.W : 0; }
int32_t bb_pool_height(const bb_pool *p) { return p ? p->lp.H : 0; }
int32_t bb_pool_num_envs(const bb_pool *p) { return p ? p->n : 0; }
int64_t bb_pool_launches(const bb_pool *p) { return p ? p->launches : 0; }

int bb_pool_counters(bb_pool *p, int64_t *out4)
{
    if (!p || !out4) return fail("bad arguments");
    CU(cudaSetDevice(p->device));
    CU(cudaDeviceSynchronize());
    std::vector<unsigned long long> c((size_t)p->num_warps * 4);
    CU(cudaMemcpy(c.data(), p->P.warp_counters, c.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 4; k++) out4[k] = 0;
    for (int wi = 0; wi < p->num_warps; wi++) for (int k = 0; k < 4; k++) out4[k] += (int64_t)c[(size_t)wi * 4 + k];
    return 0;
}

}  // extern "C"
