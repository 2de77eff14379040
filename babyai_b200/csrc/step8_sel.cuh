// step8_sel.cuh -- the role function of k_step8_sel (pool.cu, bb_pool_step_envs): one step of the envs of an id list, EIGHT
// LANES PER ENVIRONMENT.  The lanes of group g serve list entry k = 4 w + g of warp w, env ids[k], with action actions[k]:
// they stage the env's record with cp.async (observe8_role's staging), the group's leader steps it (step8_role's step_env,
// frozen-env replay, swap_in8 of the next ring level on an episode end in auto-reset mode, ring-dry error) and the warp writes
// the observations to rows `env` of the output (observe8_rows).  Reward, done and direction go to rows `env` as well; unlisted
// envs and rows are not read or written.  Its warp primitives are the macros of simt.cuh, so tests/hostemu compiles this very
// function for the host with one OS thread per lane (tests/hostemu/step_envs_host.cpp).
#pragma once
#include "simt.cuh"
#include "step8.cuh"
#include "reset8.cuh"

namespace bb {

template <class PP, int ACT_BYTES, bool UNTR>
BB_DEV void step8_sel_role(const LevelParams &lp, const PP &P, const int32_t *__restrict__ ids, const int n_sel,
                           const void *__restrict__ actions, uint8_t *__restrict__ obs, float *__restrict__ reward,
                           uint8_t *__restrict__ done, int8_t *__restrict__ dirs, const int mode, uint8_t *smem8,
                           const int lane, const int warp, const unsigned cta)
{
    // smem8: [16 envs][cells_pad + 144] then the tiles (k_step8's layout)
    const int r = lane & 7, g = lane >> 3;
    const int wg = cta * S8_WARPS + warp;
    const int k = wg * 4 + g;
    const bool valid = k < n_sel;
    const int env = valid ? ids[k] : 0;
    const int leader = lane & ~7;
    const unsigned gmask = 0xFFu << (8 * g);
    const int rec_bytes = lp.cells_pad + S8_REC_FIXED;
    uint8_t *srec = smem8 + (size_t)(warp * 4 + g) * rec_bytes;    // this env's staged record
    uint32_t *tile = reinterpret_cast<uint32_t *>(smem8 + (size_t)S8_WARPS * 4 * rec_bytes) + warp * (S8_TILE_WORDS + 1);
    const int gch = lp.cells_pad / 16;
    const size_t e = (size_t)env;

    // ---- the listed env's state in flight: asynchronous copies to shared memory + the hot record and the action
    if (valid) {
        const uint4 *gsrc = reinterpret_cast<const uint4 *>(P.grid + e * lp.cells_pad);
        for (int i = r; i < gch; i += 8) BB_CP_ASYNC16(srec + 16 * i, gsrc + i);
        if (r < 6) BB_CP_ASYNC16(srec + 16 * (gch + r), reinterpret_cast<const uint4 *>(P.obj + e) + r);
        if (r >= 5) BB_CP_ASYNC16(srec + 16 * (gch + 6 + r - 5), reinterpret_cast<const uint4 *>(P.ins + e) + (r - 5));
    }
    EnvHot h;
    { uint4 z = make_uint4(0, 0, 0, 0); h = *reinterpret_cast<EnvHot *>(&z); }
    int a = 0;
    if (valid) {
        h = P.hot[env];
        if (r == 0) {                                             // actions are indexed by list position
            if (ACT_BYTES == 1) a = reinterpret_cast<const int8_t *>(actions)[k];
            else a = (int)reinterpret_cast<const long long *>(actions)[k];
        }
    }
    BB_CP_ASYNC_WAIT_ALL();
    BB_SYNCWARP();
    StagedMem mem(lp, srec, reinterpret_cast<ObjTab *>(srec + lp.cells_pad), reinterpret_cast<InstrRec *>(srec + lp.cells_pad + sizeof(ObjTab)),
                  P.grid + e * lp.cells_pad, P.obj + e, P.ins + e);
    bool stepped = false, ended = false, succeeded = false, error = false, begin = false;
    float rew = 0.0f; bool dn = false;
    if (valid && r == 0) {                                        // the group's leader steps the env
        if (!(h.dirflags & 4)) {
            const StepResult sr = step_env<UNTR>(h, mem, a);
            rew = sr.reward; dn = sr.done;
            stepped = true; ended = dn; succeeded = sr.success;
            if (dn) {
                if (mode == BB_MODE_AUTORESET) begin = true;
                else { h.dirflags |= 4; P.last_reward[env] = rew; }
            }
        } else { rew = P.last_reward[env]; dn = true; }           // ManyEnvs: replay the last result
    }
    BB_SYNCWARP();
    {   // leader's pose and "episode begins" flag to the whole group
        uint4 hv = *reinterpret_cast<uint4 *>(&h);
        hv.x = BB_SHFL(hv.x, leader); hv.y = BB_SHFL(hv.y, leader);
        hv.z = BB_SHFL(hv.z, leader); hv.w = BB_SHFL(hv.w, leader);
        h = *reinterpret_cast<EnvHot *>(&hv);
        begin = BB_SHFL(begin ? 1 : 0, leader) != 0;
    }
    if (begin && valid) {                                         // uniform within the group
        const uint32_t hd = P.head[env];
        const uint32_t tl = BB_LDCG(P.tail_pub + env);
        if (tl - hd >= 1u && tl - hd <= (uint32_t)P.depth) {
            const int slot = (int)(hd % (uint32_t)P.depth);
            swap_in8(lp, P, env, slot, r, srec);                  // the 8 lanes copy the level together
            const uint4 hv = BB_LDCG(reinterpret_cast<const uint4 *>(r2_ring_slot(lp, P, env, slot).hot));
            h = *reinterpret_cast<const EnvHot *>(&hv);
            BB_SYNCWARP_MASK(gmask);
            if (r == 0) P.head[env] = hd + 1u;
        } else if (r == 0) { error = true; *P.err_flag = 1; }     // ring dry (the host orders the generation first): the next call fails
    }
    if (valid && r == 0) {
        P.hot[env] = h;
        reward[env] = rew;
        done[env] = dn ? 1 : 0;
        if (dirs) dirs[env] = (int8_t)(h.dirflags & 3);
    }
    BB_SYNCWARP();                                                 // staged-copy writes above are visible to the column loads
    observe8_rows<UNTR>(lp, mem, h, valid, env, obs, tile, lane);
    // ---- counters: one slot per warp, as k_step8 ---------------------------------------------------------------
    const uint32_t m_step = BB_BALLOT(stepped), m_end = BB_BALLOT(ended);
    const uint32_t m_succ = BB_BALLOT(succeeded), m_err = BB_BALLOT(error);
    if (lane == 0) {
        unsigned long long *c = P.warp_counters + 4ull * wg;
        if (m_step) BB_ATOMIC_ADD(c + 0, (unsigned long long)BB_POPC(m_step));
        if (m_end) BB_ATOMIC_ADD(c + 1, (unsigned long long)BB_POPC(m_end));
        if (m_succ) BB_ATOMIC_ADD(c + 2, (unsigned long long)BB_POPC(m_succ));
        if (m_err) BB_ATOMIC_ADD(c + 3, (unsigned long long)BB_POPC(m_err));
    }
}

}  // namespace bb
