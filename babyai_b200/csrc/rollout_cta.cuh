// rollout_cta.cuh -- the role function of k_rollout_cta (pool.cu): the persistent rollout kernel for MULTI-ROOM levels
// (grids up to 25 x 25: GoTo, BossLevel, ...; BASELINE configs 4 and 5).
//
// Why a second kernel.  The lane-per-env kernel (rollout_lane.cuh) keeps both orientations of the grid of 32 envs per warp
// in shared memory: 2 x 43 KB per CTA on 22 x 22 levels, 4 resident warps per SM, one dependent ~1 000-instruction program
// per warp and step -- 32 768 envs are only 1 024 such warps, a few per scheduler.  The parallelism that is left is INSIDE an env, and it
// is all in the observation (7 view columns), not in the step (one action, one verifier).  So a CTA of 160 threads serves 32
// envs with two ROLES that run concurrently (the protocol is described above rollout_cta_role below):
//   the stepper   warp 4, one lane per env: action, step_env, verifier, reward / done -- the efficient SIMT shape for that
//                 code; publishes each env's pose word in shared memory.  A finished env only raises a flag;
//   the observers warps 0..3, FOUR LANES PER ENV: lane q gathers view columns 2q, 2q+1 (7 cells each) from the row-major grid,
//                 computes their see-through bits, two xor-shuffles give every lane of the env all 7 column masks,
//                 process_vis (vis_rows) runs on them, the lane encodes its two columns (42 output bytes) and stages them as
//                 21-byte records into one of the CTA's two 4 704-byte tiles;
//   (swap)        rare on multi-room levels (episodes last hundreds of steps): the observers copy the finished env's next
//                 level from its ring, 128 threads x one 16-byte chunk, while the stepper waits;
//   store         one elected thread hands the tile to the copy engine (cp.async.bulk shared -> global, SASS UBLKCP).
// Shared memory per env: the ROW-MAJOR grid only (528 B for 22 x 22; the observers gather the columns of vertical views byte
// by byte, so the transposed copy is not needed), object table, verifier record: 684 B instead of 1 204 B; with the two tiles
// 31.3 KB per CTA -> 7 CTAs = 224 envs = 35 warps per SM, the whole 32 768-env pool in one wave.  The transposed grid copy
// that the per-step kernels use is regenerated from the row-major one when the state is written back at the end of the launch.
//
// Results are identical to rollout_lane.cuh / the per-step kernels (tests: the GPU-less suite runs this very function with
// one OS thread per lane, tests/hostemu/simt_rollout.cpp; test_rollout_equals_stepwise on the GPU).
#pragma once
#include "simt.cuh"

namespace bb {

constexpr int RC_ENVS = 32;                    // envs per CTA
constexpr int RC_THREADS = 160;                // warps 0..3: observers, 4 lanes per env; warp 4: the stepper, one lane per env
constexpr int RC_OBJ_STRIDE = 25, RC_INS_STRIDE = 13;             // odd word strides: lane-per-env accesses are conflict free
constexpr int RC_TILE_WORDS = RC_ENVS * OBS_BYTES / 4;            // 1176 words = 4704 B

BB_HD int rc_grid_stride(const LevelParams &lp) { return (lp.gt_off >> 2) | 1; }          // words per env: the row-major part only
// shared-memory words of one CTA: records, pose words, swap flags, hot records of swapped-in envs, the tile (16-byte aligned)
BB_HD int rc_cta_words(const LevelParams &lp)
{
    int w = RC_ENVS * (rc_grid_stride(lp) + RC_OBJ_STRIDE + RC_INS_STRIDE) + 2 * RC_ENVS + 4 * RC_ENVS;
    w = (w + 3) & ~3;
    return w + RC_TILE_WORDS;
}

// an env's records in shared memory, row-major grid only
struct SmemGMem {
    const LevelParams &lp; uint8_t *g, *o, *i;
    BB_HD SmemGMem(const LevelParams &lp_, uint8_t *g_, uint8_t *o_, uint8_t *i_) : lp(lp_), g(g_), o(o_), i(i_) {}
    BB_HD int cell(int x, int y) const { return g[y * lp.rs_g + x]; }
    BB_HD void set_cell(int x, int y, int v) { g[y * lp.rs_g + x] = (uint8_t)v; }
    BB_HD int ox(int k) const { return o[k]; }
    BB_HD int oy(int k) const { return o[MAXOBJ + k]; }
    BB_HD int otc(int k) const { return o[2 * MAXOBJ + k]; }
    BB_HD uint32_t oxw(int i) const { return load_u32_any(o + 4 * i); }
    BB_HD uint32_t oyw(int i) const { return load_u32_any(o + MAXOBJ + 4 * i); }
    BB_HD void set_oxy(int k, int x, int y) { o[k] = (uint8_t)x; o[MAXOBJ + k] = (uint8_t)y; }
    BB_HD uint32_t desc_mask(int d) const { return reinterpret_cast<const uint32_t *>(i)[d]; }
    BB_HD int leaf_kind(int l) const { return i[32 + l]; }
    BB_HD int leaf_pre(int l) const { return i[36 + l]; }
    BB_HD void set_leaf_pre(int l, int v) { i[36 + l] = (uint8_t)v; }
    BB_HD int root_kind() const { return i[40]; }
    BB_HD int side_and() const { return i[41]; }
    BB_HD void set_side_and(int v) { i[41] = (uint8_t)v; }
    BB_HD int flags() const { return i[42]; }
    BB_HD void set_flags(int v) { i[42] = (uint8_t)v; }
    BB_HD int start_carry() const { return i[43]; }
};

// The agent's 7 x 7 view on the row-major grid: view cell (vi, vj) is world cell  a + f (6 - vj) + r (vi - 3),
// f = DIR_TO_VEC[dir], r = (-f.y, f.x); outside the grid: wall.  Per pose: the byte offset of view cell (0, 0), the offset
// steps per column / per depth, the depths that lie inside the grid (the same for every column) and the lateral range.
struct RcView { int a00, di, dj, lat0, lstep, nlat; uint32_t dm; };
BB_HD RcView rc_view(const LevelParams &lp, int ax, int ay, int dir)
{
    const int fx = dir_dx(dir), fy = dir_dy(dir), rx = -fy, ry = fx;
    RcView v;
    v.a00 = (ay + 6 * fy - 3 * ry) * lp.rs_g + ax + 6 * fx - 3 * rx;
    v.di = ry * lp.rs_g + rx;
    v.dj = -(fy * lp.rs_g + fx);
    // cells from the agent to the edge of the grid it faces: depths vj >= 6 - dist are inside
    const int dist = dir == 0 ? lp.W - 1 - ax : dir == 1 ? lp.H - 1 - ay : dir == 2 ? ax : ay;
    v.dm = dist >= 6 ? 0x7Fu : (0x7Fu << (6 - dist)) & 0x7Fu;
    const bool horiz = fy == 0;                // facing left / right: columns are spread along y
    v.lat0 = (horiz ? ay - 3 * ry : ax - 3 * rx);
    v.lstep = horiz ? ry : rx;
    v.nlat = horiz ? lp.H : lp.W;
    return v;
}
// view column vi: lo = depths vj 0..3, hi = vj 4..6 (+ a zero byte) -- what col_load() yields from the two stored orientations
BB_HD void rc_col_gather(const uint8_t *g, const RcView &v, int vi, uint32_t &lo, uint32_t &hi)
{
    const uint32_t cm = (unsigned)(v.lat0 + vi * v.lstep) < (unsigned)v.nlat ? v.dm : 0u;     // depths of this column inside the grid
    const int a0 = v.a00 + vi * v.di;
    uint32_t c[7];
#pragma unroll
    for (int vj = 0; vj < 7; vj++) c[vj] = ((cm >> vj) & 1u) ? (uint32_t)g[a0 + vj * v.dj] : 0u;
    const uint32_t WALLW = 0x2A2A2A2Au;
    lo = (c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24)) | (WALLW & ~expand4(cm));
    hi = (c[4] | (c[5] << 8) | (c[6] << 16)) | (WALLW & ~expand4(cm >> 4) & 0x00FFFFFFu);
}

// =====================================================================================================================
// The stepper runs AHEAD of the observers.
//
// Version 1 of this kernel (git history) ran the two roles in lock-step with two CTA barriers per step.  Profiled
// (BossLevel, 32 768 envs), half of its stall samples sat at the first barrier -- the four observer warps wait
// for the stepper (A takes ~0.78 of a step, B2 ~0.18), and then the stepper waits at barrier Y while the observers gather
// (B1, ~0.22): a step lasts A + B1.  The only thing of the stepper's that the observers read is the row-major grid and the
// pose word, and step_env writes at most two grid cells per step.  So the stepper computes step t + 1 WHILE the observers
// gather step t, with its cell writes deferred (DeferGMem), and only the commit -- two byte stores and the pose word --
// waits for them: a step lasts max(A + commit, B1 + B2).  The rendezvous are producer / consumer named barriers
// (barrier.arrive on one side, barrier.sync on the other): X "step t is committed" (stepper -> observers), Y "gather of
// step t is done" (observers -> stepper).  The tile is double-buffered, so the observers need one barrier of their own per
// step (tile complete -> one thread issues the bulk store).  An episode swap-in (rare) is done by the 128 observer threads
// while the stepper waits at barrier Z.
// =====================================================================================================================
constexpr int RC_BAR_X = 2, RC_BAR_Y = 3, RC_BAR_Z = 4, RC_BAR_OBS = 5;      // barrier 0: __syncthreads, 1: BB_ROLE_SYNC
constexpr int RC_OBS_THREADS = RC_THREADS - 32;

BB_HD int rc2_cta_words(const LevelParams &lp) { return rc_cta_words(lp) + RC_TILE_WORDS + 4; }     // second tile + flag word

// SmemGMem whose cell writes wait for commit(): what the stepper uses while the observers still read the grid
struct DeferGMem : SmemGMem {
    int off0, off1, val0, val1;
    BB_HD DeferGMem(const LevelParams &lp_, uint8_t *g_, uint8_t *o_, uint8_t *i_) : SmemGMem(lp_, g_, o_, i_), off0(-1), off1(-1), val0(0), val1(0) {}
    BB_HD int cell(int x, int y) const
    {
        const int off = y * lp.rs_g + x;
        if (off == off1) return val1;
        if (off == off0) return val0;
        return g[off];
    }
    BB_HD void set_cell(int x, int y, int v)
    {
        const int off = y * lp.rs_g + x;
        if (off0 < 0 || off0 == off) { off0 = off; val0 = v; }
        else { off1 = off; val1 = v; }
    }
    BB_HD void commit()
    {
        if (off0 >= 0) { g[off0] = (uint8_t)val0; off0 = -1; }
        if (off1 >= 0) { g[off1] = (uint8_t)val1; off1 = -1; }
    }
};

template <class PP, bool UNTR>
BB_DEV void rollout_cta_role(const LevelParams &lp, const PP &P, const int8_t *actions, uint8_t *obs, float *reward, uint8_t *done,
                             int8_t *dirs, const int n, const int T, const int mode, uint32_t *smem, const int tid, const int cta,
                             const int row_stride = 0)
{
    const size_t rs = row_stride ? (size_t)row_stride : (size_t)n;     // rows between steps of the [T][.] buffers (rollout_lane.cuh)
    const int lane = tid & 31, warp = tid >> 5;
    const int gs = rc_grid_stride(lp);
    const int env0 = cta * RC_ENVS;
    int nv = n - env0; nv = nv > RC_ENVS ? RC_ENVS : (nv < 0 ? 0 : nv);
    uint32_t *sg = smem, *so = sg + RC_ENVS * gs, *si = so + RC_ENVS * RC_OBJ_STRIDE;
    uint32_t *s_pose = si + RC_ENVS * RC_INS_STRIDE;               // x | y << 8 | dir << 16 | carried cell byte << 24
    uint32_t *s_swap = s_pose + RC_ENVS;                           // ring slot + 1 of an env whose episode begins, else 0
    uint32_t *s_hot = s_swap + RC_ENVS;                            // hot record of a swapped-in level (4 words per env)
    uint32_t *tiles = smem + (rc_cta_words(lp) - RC_TILE_WORDS);   // two tiles, 16-byte aligned
    volatile uint32_t *s_any = tiles + 2 * RC_TILE_WORDS;          // "an episode begins at this step" (written at commit)
    const int gchunks = lp.gt_off >> 4, tchunks = lp.max_tokens >> 3;
    // ---- load the state of the CTA's envs once: row-major grid part, object table, verifier record -------------
    for (int idx = tid; idx < nv * gchunks; idx += RC_THREADS) {
        const int e = idx / gchunks, k = idx - e * gchunks;
        const uint4 v = reinterpret_cast<const uint4 *>(P.grid + (size_t)(env0 + e) * lp.cells_pad)[k];
        uint32_t *d = sg + e * gs + 4 * k;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
    for (int idx = tid; idx < nv * 6; idx += RC_THREADS) {
        const int e = idx / 6, k = idx - e * 6;
        const uint4 v = reinterpret_cast<const uint4 *>(P.obj + env0)[idx];
        uint32_t *d = so + e * RC_OBJ_STRIDE + 4 * k;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
    for (int idx = tid; idx < nv * 3; idx += RC_THREADS) {
        const int e = idx / 3, k = idx - e * 3;
        const uint4 v = reinterpret_cast<const uint4 *>(P.ins + env0)[idx];
        uint32_t *d = si + e * RC_INS_STRIDE + 4 * k;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
    if (tid < RC_ENVS) s_swap[tid] = 0;
    if (tid == 0) *s_any = 0;
    const bool stepper = warp == RC_THREADS / 32 - 1;
    BB_SYNCTHREADS();
    if (stepper) {
        // ================= the stepper: warp 4, lane = env within the CTA =================
        const int env_a = env0 + lane;
        const bool valid_a = lane < nv;
        EnvHot h;
        { uint4 z = make_uint4(0, 0, 0, 0); h = *reinterpret_cast<EnvHot *>(&z); }
        uint32_t head = 0, avail = 0, consumed = 0;
        float last_rew = 0.0f;
        uint32_t n_step = 0, n_end = 0, n_succ = 0, n_err = 0;
        int a_next = 0;
        if (valid_a) {
            h = P.hot[env_a];
            head = P.head[env_a];
            avail = BB_LDCG(P.tail_pub + env_a) - head;
            if (mode == BB_MODE_FREEZE) last_rew = P.last_reward[env_a];
            a_next = BB_LD_S8(actions + env_a);
        }
        DeferGMem mem_a(lp, reinterpret_cast<uint8_t *>(sg + lane * gs), reinterpret_cast<uint8_t *>(so + lane * RC_OBJ_STRIDE),
                        reinterpret_cast<uint8_t *>(si + lane * RC_INS_STRIDE));
        for (int t = 0; t < T; t++) {
            // ---- A(t): step the env; grid writes are deferred, nothing the observers read is touched ----
            bool begin = false;
            uint32_t pose = 0;
            const int a = a_next;
            if (valid_a && t + 1 < T) a_next = BB_LD_S8(actions + (t + 1) * rs + env_a);
            if (valid_a) {
                float rew = 0.0f; bool dn = false;
                if (!(h.dirflags & 4)) {
                    const StepResult sr = step_env<UNTR>(h, mem_a, a);
                    rew = sr.reward; dn = sr.done;
                    n_step++; n_end += dn; n_succ += sr.success;
                    if (dn) {
                        if (mode == BB_MODE_AUTORESET) begin = true;
                        else { h.dirflags |= 4; last_rew = rew; }
                    }
                } else { rew = last_rew; dn = true; }
                if (begin && !(consumed < avail && avail <= (uint32_t)P.depth)) { begin = false; n_err++; *P.err_flag = 1; }   // ring dry
                pose = (uint32_t)h.x | ((uint32_t)h.y << 8) | ((uint32_t)(h.dirflags & 3) << 16) | ((uint32_t)carry_cell_of<UNTR>(h, mem_a) << 24);
                const size_t oi = t * rs + env_a;
                if (reward) reward[oi] = rew;
                if (done) done[oi] = dn ? 1 : 0;
            }
            const bool any_begin = BB_ANY(begin);
            // ---- commit(t): after the observers have gathered step t - 1 ----
            if (t > 0) BB_BAR_SYNC(RC_BAR_Y, RC_THREADS);
            if (valid_a) {
                mem_a.commit();
                if (begin) s_swap[lane] = (head + consumed) % (uint32_t)P.depth + 1u;
                else s_pose[lane] = pose;
            }
            if (lane == 0) *s_any = any_begin ? 1u : 0u;
            BB_BAR_ARRIVE(RC_BAR_X, RC_THREADS);
            if (any_begin) {
                BB_BAR_SYNC(RC_BAR_Z, RC_THREADS);                 // the observers have copied the new levels in
                if (begin) {
                    const uint4 hv = make_uint4(s_hot[4 * lane], s_hot[4 * lane + 1], s_hot[4 * lane + 2], s_hot[4 * lane + 3]);
                    h = *reinterpret_cast<const EnvHot *>(&hv);
                    consumed++;
                    s_swap[lane] = 0;
                }
            }
        }
        if (valid_a) {
            P.hot[env_a] = h;
            P.head[env_a] = head + consumed;
            if (mode == BB_MODE_FREEZE) P.last_reward[env_a] = last_rew;
        }
        for (int off = 16; off; off >>= 1) {
            n_step += BB_SHFL_DOWN(n_step, off); n_end += BB_SHFL_DOWN(n_end, off);
            n_succ += BB_SHFL_DOWN(n_succ, off); n_err += BB_SHFL_DOWN(n_err, off);
        }
        if (lane == 0) {
            unsigned long long *c = P.warp_counters + 4ull * cta;
            if (n_step) BB_ATOMIC_ADD(c + 0, (unsigned long long)n_step);
            if (n_end) BB_ATOMIC_ADD(c + 1, (unsigned long long)n_end);
            if (n_succ) BB_ATOMIC_ADD(c + 2, (unsigned long long)n_succ);
            if (n_err) BB_ATOMIC_ADD(c + 3, (unsigned long long)n_err);
        }
    } else {
        // ================= the observers: warps 0..3, 4 lanes per env =================
        const int el = (tid >> 2) & (RC_ENVS - 1), q = tid & 3;
        const bool valid_b = el < nv;
        const uint8_t *g_b = reinterpret_cast<const uint8_t *>(sg + el * gs);
        const bool bulk_ok = nv == RC_ENVS && (((uintptr_t)(obs + (size_t)env0 * OBS_BYTES)) & 15) == 0 && ((rs * OBS_BYTES) & 15) == 0;
        for (int t = 0; t < T; t++) {
            BB_BAR_SYNC(RC_BAR_X, RC_THREADS);                     // step t is committed
            if (*s_any) {
                // ---- episode swap-in by the 128 observer threads (rare) ----
                for (int e = 0; e < RC_ENVS; e++) {
                    const uint32_t sw = s_swap[e];
                    if (!sw) continue;                             // uniform: every thread reads the same flag
                    const LevelOut o = r2_ring_slot(lp, P, env0 + e, (int)sw - 1);
                    for (int c = tid; c < gchunks + 9 + tchunks + 1; c += RC_OBS_THREADS) {
                        int k = c;
                        if (k < gchunks + 9) {
                            const uint4 *sp; uint32_t *dp;
                            if (k < gchunks) { sp = reinterpret_cast<const uint4 *>(o.grid) + k; dp = sg + e * gs + 4 * k; }
                            else if ((k -= gchunks) < 6) { sp = reinterpret_cast<const uint4 *>(o.obj) + k; dp = so + e * RC_OBJ_STRIDE + 4 * k; }
                            else { k -= 6; sp = reinterpret_cast<const uint4 *>(o.ins) + k; dp = si + e * RC_INS_STRIDE + 4 * k; }
                            const uint4 v = BB_LDCG(sp);
                            dp[0] = v.x; dp[1] = v.y; dp[2] = v.z; dp[3] = v.w;
                        } else if ((k -= gchunks + 9) < tchunks) {
                            reinterpret_cast<uint4 *>(P.tok + (size_t)(env0 + e) * lp.max_tokens)[k] = BB_LDCG(reinterpret_cast<const uint4 *>(o.tok) + k);
                        } else {                                   // the hot record: to the stepping lane, and the pose word of the new episode
                            const uint4 hv = BB_LDCG(reinterpret_cast<const uint4 *>(o.hot));
                            s_hot[4 * e] = hv.x; s_hot[4 * e + 1] = hv.y; s_hot[4 * e + 2] = hv.z; s_hot[4 * e + 3] = hv.w;
                            const EnvHot nh = *reinterpret_cast<const EnvHot *>(&hv);
                            s_pose[e] = (uint32_t)nh.x | ((uint32_t)nh.y << 8) | ((uint32_t)(nh.dirflags & 3) << 16) | ((uint32_t)CELL_EMPTY << 24);
                        }
                    }
                }
                BB_BAR_ARRIVE(RC_BAR_Z, RC_THREADS);               // the stepper may take the new episodes over
                BB_BAR_SYNC(RC_BAR_OBS, RC_OBS_THREADS);           // ... and the observers see each other's copies
            }
            // ---- B1(t): pose, the lane's two view columns, the env's see-through masks -> registers ----
            const uint32_t pose = valid_b ? s_pose[el] : 0u;
            const int ax = (int)(pose & 0xFF), ay = (int)((pose >> 8) & 0xFF), dir = (int)((pose >> 16) & 3);
            const uint32_t carry_b = pose >> 24;
            uint32_t cmA = 0, cmB = 0, loA = 0, hiA = 0, loB = 0, hiB = 0;
            if (valid_b) {
                const RcView view = rc_view(lp, ax, ay, dir);
                rc_col_gather(g_b, view, 2 * q, loA, hiA);
                cmA = col_see(loA, hiA);
                if (q < 3) { rc_col_gather(g_b, view, 2 * q + 1, loB, hiB); cmB = col_see(loB, hiB); }
            }
            if (t + 1 < T) BB_BAR_ARRIVE(RC_BAR_Y, RC_THREADS);    // the grid and the pose words may change now
            // the 7 column masks (see-through bits, bit vj) of the env to all of its 4 lanes: byte vi of (blo : bhi)
            const uint32_t v16 = cmA | (cmB << 8);
            const uint32_t p1 = BB_SHFL_XOR(v16, 1);
            const uint32_t mine = (q & 1) ? (p1 | (v16 << 16)) : (v16 | (p1 << 16));
            const uint32_t other = BB_SHFL_XOR(mine, 2);
            const uint32_t blo = (q & 2) ? other : mine, bhi = (q & 2) ? mine : other;
            if (valid_b && q == 0 && dirs) dirs[t * rs + env0 + el] = (int8_t)dir;
            // ---- B2(t): process_vis, encode, stage into tile t & 1 ----
            uint32_t *tile = tiles + (t & 1) * RC_TILE_WORDS;
            uint32_t tlo = blo, thi = bhi;
            transpose8(tlo, thi);                                  // column masks -> per view row (bit vi)
            uint32_t see[7], vis[7];
#pragma unroll
            for (int vj = 0; vj < 7; vj++) see[vj] = ((vj < 4 ? tlo >> (8 * vj) : thi >> (8 * (vj - 4)))) & 0x7Fu;
            vis_rows(see, vis);
            uint32_t vlo = 0, vhi = 0;
#pragma unroll
            for (int vj = 0; vj < 7; vj++) { if (vj < 4) vlo |= vis[vj] << (8 * vj); else vhi |= vis[vj] << (8 * (vj - 4)); }
            transpose8(vlo, vhi);                                  // byte vi = visibility of column vi, bit vj
            const uint32_t vmine = (q & 2) ? vhi : vlo;            // columns 4..7 / 0..3
            const uint32_t cvA = (vmine >> (16 * (q & 1))) & 0x7Fu, cvB = (vmine >> (16 * (q & 1) + 8)) & 0x7Fu;
            uint32_t hB = hiB;
            if (q == 1) hB = (hB & 0xFF00FFFFu) | (carry_b << 16);     // view cell (3, 6): the agent's own cell shows what it carries
            uint32_t oA[6], oB[6];
            col_encode(loA, hiA, valid_b ? cvA : 0u, oA);
            col_encode(loB, hB, (valid_b && q < 3) ? cvB : 0u, oB);
            const uint32_t nextA = BB_SHFL_DOWN(oA[0], 1);
            if (q < 3) {
                stage_record_words<21, 6>(tile, oA, 7 * el + 2 * q, oB[0]);
                stage_record_words<21, 6>(tile, oB, 7 * el + 2 * q + 1, nextA);
            } else stage_record_words<21, 6>(tile, oA, 7 * el + 6, nextA);
            BB_FENCE_ASYNC_SMEM();                                 // tile writes -> visible to the copy engine
            BB_BAR_SYNC(RC_BAR_OBS, RC_OBS_THREADS);               // the tile is complete
            uint8_t *dst = obs + (t * rs + env0) * OBS_BYTES;
            if (bulk_ok) {
                // the other tile is rewritten at step t + 1: its bulk copy (step t - 1) must have read it by then; every
                // observer passes barrier X of step t + 1 only after this thread has
                if (tid == 0) { BB_BULK_STORE(dst, tile, RC_ENVS * OBS_BYTES); BB_BULK_WAIT_READ_N(1); }
            } else {
                const uint8_t *sb = reinterpret_cast<const uint8_t *>(tile);
                for (int i = tid; i < nv * OBS_BYTES; i += RC_OBS_THREADS) dst[i] = sb[i];
            }
        }
        if (tid == 0) BB_BULK_WAIT_READ();                         // shared memory must outlive the copy engine's reads
    }
    BB_SYNCTHREADS();                                              // both roles are done with step T - 1
    // ---- store the state back: row-major part as is, the transposed part regenerated from it ---------------------------
    for (int idx = tid; idx < nv * gchunks; idx += RC_THREADS) {
        const int e = idx / gchunks, k = idx - e * gchunks;
        const uint32_t *d = sg + e * gs + 4 * k;
        reinterpret_cast<uint4 *>(P.grid + (size_t)(env0 + e) * lp.cells_pad)[k] = make_uint4(d[0], d[1], d[2], d[3]);
    }
    {
        const int twords = lp.rs_t >> 2, per_env = lp.W * twords;
        for (int idx = tid; idx < nv * per_env; idx += RC_THREADS) {
            const int e = idx / per_env, r = idx - e * per_env;
            const int x = r / twords, y0 = (r - x * twords) * 4;
            const uint8_t *ge = reinterpret_cast<const uint8_t *>(sg + e * gs);
            uint32_t wv = 0;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int y = y0 + b;
                const uint32_t c = y < lp.H ? (uint32_t)ge[y * lp.rs_g + x] : (uint32_t)CELL_WALL;      // row padding is wall
                wv |= c << (8 * b);
            }
            reinterpret_cast<uint32_t *>(P.grid + (size_t)(env0 + e) * lp.cells_pad + lp.gt_off)[r] = wv;
        }
    }
    for (int idx = tid; idx < nv * 6; idx += RC_THREADS) {
        const int e = idx / 6, k = idx - e * 6;
        const uint32_t *d = so + e * RC_OBJ_STRIDE + 4 * k;
        reinterpret_cast<uint4 *>(P.obj + env0)[idx] = make_uint4(d[0], d[1], d[2], d[3]);
    }
    for (int idx = tid; idx < nv * 3; idx += RC_THREADS) {
        const int e = idx / 3, k = idx - e * 3;
        const uint32_t *d = si + e * RC_INS_STRIDE + 4 * k;
        reinterpret_cast<uint4 *>(P.ins + env0)[idx] = make_uint4(d[0], d[1], d[2], d[3]);
    }
}

}  // namespace bb
