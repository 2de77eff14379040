// rollout_lane.cuh -- the stepping role of k_rollout (pool.cu): ONE LANE PER ENVIRONMENT, persistent over the T steps of
// a bb_pool_rollout call, the state of the warp's 32 envs resident in shared memory (single-room levels: every size;
// multi-room levels use rollout_cta.cuh).
//
// Per step a warp reads 32 action bytes (prefetched one step ahead), runs step_env + the verifier, swaps finished
// episodes for their next pre-generated level, computes the 32 observations, stages them as one 4704-byte tile and
// hands the tile to the copy engine: ONE cp.async.bulk (shared -> global, SASS UBLKCP) issued by lane 0 replaces the
// 294 LDS.128 + STG.128 pairs the warp issued before (the kernel is issue / latency bound, so tile
// movement belongs on the async proxy, not on the issue path).  The tile is single-buffered: the bulk read of step t is
// waited for (cp.async.bulk.wait_group.read) right before step t+1 stages its observations -- a whole step_env +
// observe later, so the wait never stalls.
//
// Episode swap-in (46 % of the warp-steps of GoToLocal contain a finished env): the WARP copies the level -- for every
// finished lane in turn, 17 lanes move one 16-byte chunk each (grid, object table, verifier record) and up to 9 more the
// mission tokens -- instead of the finished lane alone issuing ~20 LDG.128 and ~80 STS while 31 lanes wait.
//
// The warp primitives are macros (simt.cuh) so that tests/hostemu compiles this very function for the host with one OS
// thread per lane (tests/hostemu/simt_rollout.cpp) and steps whole rollouts through it against the per-step path.
#pragma once
#include "simt.cuh"

namespace bb {

constexpr int RL_OBJ_STRIDE = 25, RL_INS_STRIDE = 13;             // odd word strides of the lane records (= pool.cu SM_*_STRIDE)
constexpr int RL_TILE_WORDS = 32 * OBS_BYTES / 4;                 // 1176 words = 4704 B per warp
constexpr int R_STEP_WARPS = 2;                                   // stepping warps per CTA of k_rollout (pool.cu R_WARPS)

BB_HD int rl_warp_words(const LevelParams &lp) { return 32 * (((lp.cells_pad >> 2) | 1) + RL_OBJ_STRIDE + RL_INS_STRIDE) + RL_TILE_WORDS; }

// coalesced copy of `chunks_per_env` 16-byte chunks per env between global memory (contiguous records of the warp's
// envs) and the lane-strided shared-memory records
template <bool TO_SMEM>
BB_DEV void rl_copy_records(uint32_t *sm, int stride_words, uint4 *glob, int chunks_per_env, int nv, int lane)
{
    for (int idx = lane; idx < nv * chunks_per_env; idx += 32) {
        const int e = idx / chunks_per_env, w0 = (idx - e * chunks_per_env) * 4;
        uint32_t *d = sm + e * stride_words + w0;
        if (TO_SMEM) { const uint4 v = glob[idx]; d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }
        else glob[idx] = make_uint4(d[0], d[1], d[2], d[3]);
    }
}

// ragged tail / unaligned destination: plain stores
BB_DEV void rl_store_tile_plain(const uint32_t *tile, uint8_t *dst, int lane, int valid_envs)
{
    const uint8_t *s = reinterpret_cast<const uint8_t *>(tile);
    const int nbytes = valid_envs * OBS_BYTES;
    for (int i = lane; i < nbytes; i += 32) dst[i] = s[i];
}

// MemT: the accessor of the lane's records in shared memory (pool.cu SmemOnlyMem; HostSmemMem in the host build)
template <class PP, class MemT, int ACT_BYTES, bool UNTR>
BB_DEV void rollout_lane_step_warp(const LevelParams &lp, const PP &P, const void *actions_v, uint8_t *obs, float *reward, uint8_t *done,
                                   int8_t *dirs, const int n, const int T, const int mode, const int force_reset, const bool fused,
                                   uint32_t *warp_smem, const int lane, const int warp_global, volatile int *s_done,
                                   const int row_stride = 0)
{
    // rows between the steps of the [T][.] action and output buffers: n for a pool's own buffers (0), the mixed pool's env
    // count for a group of a mixed pool (its rows are a column block of the caller's buffers)
    const size_t rs = row_stride ? (size_t)row_stride : (size_t)n;
    const int8_t *actions = reinterpret_cast<const int8_t *>(actions_v);
    const int gs = (lp.cells_pad >> 2) | 1;
    const int env0 = warp_global * 32, env = env0 + lane;
    int nv = n - env0; nv = nv > 32 ? 32 : (nv < 0 ? 0 : nv);
    const bool valid = lane < nv;
    uint32_t *sg = warp_smem, *so = sg + 32 * gs, *si = so + 32 * RL_OBJ_STRIDE;
    uint32_t *tile = si + 32 * RL_INS_STRIDE;           // 16-byte aligned: every term is a multiple of 4 words
    // ---- load the state of the warp's envs once ---------------------------------------------------
    rl_copy_records<true>(sg, gs, reinterpret_cast<uint4 *>(P.grid + (size_t)env0 * lp.cells_pad), lp.cells_pad >> 4, nv, lane);
    rl_copy_records<true>(so, RL_OBJ_STRIDE, reinterpret_cast<uint4 *>(P.obj + env0), 6, nv, lane);
    rl_copy_records<true>(si, RL_INS_STRIDE, reinterpret_cast<uint4 *>(P.ins + env0), 3, nv, lane);
    EnvHot h;
    { uint4 z = make_uint4(0, 0, 0, 0); h = *reinterpret_cast<EnvHot *>(&z); }
    uint32_t head = 0, avail = 0;
    float last_rew = 0.0f;
    if (valid) {
        h = P.hot[env];
        head = P.head[env];
        // fused launch: the CTA's generator warp is the only producer and has not started yet (barrier below)
        avail = (fused ? P.tail[env] : BB_LDCG(P.tail_pub + env)) - head;
        if (mode == BB_MODE_FREEZE) last_rew = P.last_reward[env];
    }
    if (fused) BB_ROLE_SYNC(32 * (R_STEP_WARPS + 1));       // heads / tails are read: the CTA's generator warp may start
    BB_SYNCWARP();
    MemT mem(lp, reinterpret_cast<uint8_t *>(sg + lane * gs), reinterpret_cast<uint8_t *>(so + lane * RL_OBJ_STRIDE),
             reinterpret_cast<uint8_t *>(si + lane * RL_INS_STRIDE));
    uint32_t n_step = 0, n_end = 0, n_succ = 0, n_err = 0, consumed = 0;
    const int gchunks = lp.cells_pad >> 4, tchunks = lp.max_tokens >> 3;
    const int rec_chunks = gchunks + 6 + 3;              // grid, object table, verifier record
    bool bulk_pending = false;
    // actions are read one step ahead with a sign-extending load (no dependent conversion instruction: the
    // compiler otherwise converts the byte right after the load and the warp waits for DRAM there)
    int a_next = 0;
    if (valid && !force_reset) {
        if (ACT_BYTES == 1) a_next = BB_LD_S8(actions + env);
        else a_next = (int)reinterpret_cast<const long long *>(actions_v)[env];      // int64 actions: single-step calls only
    }
    for (int t = 0; t < T; t++) {
        const int a = a_next;
        if (ACT_BYTES == 1 && valid && t + 1 < T) a_next = BB_LD_S8(actions + (t + 1) * rs + env);
        float rew = 0.0f; bool dn = false, begin = false;
        if (valid) {
            begin = force_reset != 0;
            if (force_reset) {
            } else if (!(h.dirflags & 4)) {
                const StepResult sr = step_env<UNTR>(h, mem, a);
                rew = sr.reward; dn = sr.done;
                n_step++; n_end += dn; n_succ += sr.success;
                if (dn) {
                    if (mode == BB_MODE_AUTORESET) begin = true;
                    else { h.dirflags |= 4; last_rew = rew; }
                }
            } else { rew = last_rew; dn = true; }
            if (begin && !(consumed < avail && avail <= (uint32_t)P.depth)) { begin = false; n_err++; *P.err_flag = 1; }   // ring dry: the host fails the next call
        }
        // ---- episode swap-in by the whole warp: ring slot -> the finished lane's records ----------------
        uint32_t mbeg = BB_BALLOT(begin);
        if (mbeg) {
            const uint32_t my_slot = (head + consumed) % (uint32_t)P.depth;
            BB_SYNCWARP();                                         // step_env's writes to the finished lanes' records come first
            while (mbeg) {
                const int src = ffs32(mbeg);
                mbeg &= mbeg - 1;
                const int slot = (int)BB_SHFL(my_slot, src);
                const int e = env0 + src;
                const LevelOut o = r2_ring_slot(lp, P, e, slot);
                for (int c = lane; c < rec_chunks + tchunks; c += 32) {
                    if (c < rec_chunks) {
                        const uint4 *sp; uint32_t *dp; int k = c;
                        if (k < gchunks) { sp = reinterpret_cast<const uint4 *>(o.grid) + k; dp = sg + src * gs + 4 * k; }
                        else if ((k -= gchunks) < 6) { sp = reinterpret_cast<const uint4 *>(o.obj) + k; dp = so + src * RL_OBJ_STRIDE + 4 * k; }
                        else { k -= 6; sp = reinterpret_cast<const uint4 *>(o.ins) + k; dp = si + src * RL_INS_STRIDE + 4 * k; }
                        const uint4 v = BB_LDCG(sp);
                        dp[0] = v.x; dp[1] = v.y; dp[2] = v.z; dp[3] = v.w;
                    } else {
                        const int k = c - rec_chunks;
                        reinterpret_cast<uint4 *>(P.tok + (size_t)e * lp.max_tokens)[k] = BB_LDCG(reinterpret_cast<const uint4 *>(o.tok) + k);
                    }
                }
                if (lane == src) {                                 // the finished lane fetches its new hot record itself
                    const uint4 hv = BB_LDCG(reinterpret_cast<const uint4 *>(o.hot));
                    h = *reinterpret_cast<const EnvHot *>(&hv);
                    consumed++;
                }
            }
            BB_SYNCWARP();                                         // the new records -> their lanes
        }
        uint32_t w[OBS_WORDS];
#pragma unroll
        for (int k = 0; k < OBS_WORDS; k++) w[k] = 0;
        if (valid) {
            // an episode about to time out (73 % of the episode ends under random actions) will need its next
            // level two steps from now: pull that ring slot into L2 ahead of the swap-in
            if (mode == BB_MODE_AUTORESET && (int)h.step_count + 2 == (int)h.max_steps && consumed < avail) {
                const LevelOut o = r2_ring_slot(lp, P, env, (int)((head + consumed) % (uint32_t)P.depth));
                BB_PREFETCH_L2(o.grid);
                BB_PREFETCH_L2(o.obj);
                BB_PREFETCH_L2(reinterpret_cast<const uint8_t *>(o.obj) + 64);
                BB_PREFETCH_L2(o.ins);
                BB_PREFETCH_L2(reinterpret_cast<const uint8_t *>(o.ins) + 32);
                BB_PREFETCH_L2(o.hot);
                BB_PREFETCH_L2(o.tok);
            }
            observe(lp, mem, h.x, h.y, h.dirflags & 3, carry_cell_of<UNTR>(h, mem), w);
            const size_t oi = t * rs + env;
            if (reward) reward[oi] = rew;
            if (done) done[oi] = dn ? 1 : 0;
            if (dirs) dirs[oi] = (int8_t)(h.dirflags & 3);
        }
        // ---- the warp's 32 observations: stage as one tile, hand it to the copy engine ------------------
        if (lane == 0 && bulk_pending) BB_BULK_WAIT_READ();       // the copy engine has read the previous tile (issued a whole step ago)
        bulk_pending = false;
        BB_SYNCWARP();
        {
            const uint32_t next_w0 = BB_SHFL_DOWN(w[0], 1);
            stage_obs_words(tile, w, lane, next_w0);
        }
        uint8_t *dst = obs + (t * rs + env0) * OBS_BYTES;
        const bool bulk = nv == 32 && (((uintptr_t)dst) & 15) == 0;
        if (bulk) BB_FENCE_ASYNC_SMEM();                           // generic-proxy tile writes -> visible to the async proxy
        BB_SYNCWARP();
        if (bulk) {
            if (lane == 0) { BB_BULK_STORE(dst, tile, 32 * OBS_BYTES); bulk_pending = true; }
        } else if (nv > 0) {
            rl_store_tile_plain(tile, dst, lane, nv);
            BB_SYNCWARP();                                         // the tile is rewritten in the next iteration
        }
    }
    if (lane == 0 && bulk_pending) BB_BULK_WAIT_READ();            // shared memory must outlive the copy engine's reads
    // ---- store the state back ---------------------------------------------------------------------
    BB_SYNCWARP();
    rl_copy_records<false>(sg, gs, reinterpret_cast<uint4 *>(P.grid + (size_t)env0 * lp.cells_pad), lp.cells_pad >> 4, nv, lane);
    rl_copy_records<false>(so, RL_OBJ_STRIDE, reinterpret_cast<uint4 *>(P.obj + env0), 6, nv, lane);
    rl_copy_records<false>(si, RL_INS_STRIDE, reinterpret_cast<uint4 *>(P.ins + env0), 3, nv, lane);
    if (valid) {
        P.hot[env] = h;
        P.head[env] = head + consumed;
        if (mode == BB_MODE_FREEZE) P.last_reward[env] = last_rew;
    }
    // counters: warp sums, one RED per counter per warp
    for (int off = 16; off; off >>= 1) {
        n_step += BB_SHFL_DOWN(n_step, off); n_end += BB_SHFL_DOWN(n_end, off);
        n_succ += BB_SHFL_DOWN(n_succ, off); n_err += BB_SHFL_DOWN(n_err, off);
    }
    if (fused && lane == 0) BB_ATOMIC_ADD(const_cast<int *>(s_done), 1);     // tells the generator warp not to start another round
    if (lane == 0) {
        unsigned long long *c = P.warp_counters + 4ull * warp_global;
        if (n_step) BB_ATOMIC_ADD(c + 0, (unsigned long long)n_step);
        if (n_end) BB_ATOMIC_ADD(c + 1, (unsigned long long)n_end);
        if (n_succ) BB_ATOMIC_ADD(c + 2, (unsigned long long)n_succ);
        if (n_err) BB_ATOMIC_ADD(c + 3, (unsigned long long)n_err);
    }
}

}  // namespace bb
