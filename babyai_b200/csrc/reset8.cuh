// reset8.cuh -- the role function of k_reset8 (pool.cu, bb_pool_reset_envs): a new episode for the envs of an id list, EIGHT
// LANES PER ENVIRONMENT as in k_step8's reset path (step8.cuh).  The lanes of group g serve env ids[4 w + g] of warp w: they
// copy the level at the head of its ring into the live state (swap_in8), advance the head, and write the first observation to
// row `env` of the output -- only the listed rows.  Its warp primitives are the macros of simt.cuh, so tests/hostemu compiles
// this very function for the host with one OS thread per lane (tests/hostemu/simt_reset.cpp).
#pragma once
#include "simt.cuh"
#include "step8.cuh"

namespace bb {

template <class PP, bool UNTR>
BB_DEV void reset8_role(const LevelParams &lp, const PP &P, const int32_t *__restrict__ ids, const int n_sel,
                        uint8_t *__restrict__ obs, int8_t *__restrict__ dirs, uint8_t *smem8, const int lane, const int warp,
                        const unsigned cta)
{
    // smem8: [16 envs][cells_pad + 144] then the tiles (k_step8's layout)
    const int r = lane & 7, g = lane >> 3;
    const int wg = cta * S8_WARPS + warp;
    const int k = wg * 4 + g;
    const bool valid = k < n_sel;
    const int env = valid ? ids[k] : 0;
    const int rec_bytes = lp.cells_pad + S8_REC_FIXED;
    uint8_t *srec = smem8 + (size_t)(warp * 4 + g) * rec_bytes;    // this env's staged record
    uint32_t *tile = reinterpret_cast<uint32_t *>(smem8 + (size_t)S8_WARPS * 4 * rec_bytes) + warp * (S8_TILE_WORDS + 1);
    const size_t e = (size_t)env;

    EnvHot h;
    { uint4 z = make_uint4(0, 0, 0, 0); h = *reinterpret_cast<EnvHot *>(&z); }
    uint32_t hd = 0;
    bool ok = false;                                              // uniform within the group
    if (valid) {
        hd = P.head[env];
        const uint32_t tl = BB_LDCG(P.tail_pub + env);
        ok = tl - hd >= 1u && tl - hd <= (uint32_t)P.depth;
    }
    if (ok) {
        const int slot = (int)(hd % (uint32_t)P.depth);
        swap_in8(lp, P, env, slot, r, srec);                      // the 8 lanes copy the level together
        const uint4 hv = BB_LDCG(reinterpret_cast<const uint4 *>(r2_ring_slot(lp, P, env, slot).hot));
        h = *reinterpret_cast<const EnvHot *>(&hv);
    }
    BB_SYNCWARP();                                                 // every lane has read the head, the staged copy is complete
    const bool error = valid && !ok && r == 0;                    // ring dry (the host runs a selected pass first): the next call fails
    if (error) *P.err_flag = 1;
    if (ok && r == 0) {
        P.head[env] = hd + 1u;
        P.hot[env] = h;                                           // a fresh level: the frozen flag is clear
        if (dirs) dirs[env] = (int8_t)(h.dirflags & 3);
    }
    StagedMem mem(lp, srec, reinterpret_cast<ObjTab *>(srec + lp.cells_pad), reinterpret_cast<InstrRec *>(srec + lp.cells_pad + sizeof(ObjTab)),
                  P.grid + e * lp.cells_pad, P.obj + e, P.ins + e);
    // ---- observation: lane r < 7 holds view column vi = r (step8_role's code) ----------------------
    const ViewGeom v = view_geom(lp, h.x, h.y, h.dirflags & 3);
    uint32_t lo = 0, hi = 0, cm = 0;
    if (ok && r < 7) { col_load(mem, v, r, lo, hi); cm = col_see(lo, hi); }
    uint32_t see[7], vis[7];
#pragma unroll
    for (int j = 0; j < 7; j++) see[j] = (BB_BALLOT((cm >> j) & 1u) >> (8 * g)) & 0x7Fu;
    vis_rows(see, vis);
    uint32_t cv = 0;
#pragma unroll
    for (int j = 0; j < 7; j++) cv |= ((vis[j] >> r) & 1u) << j;
    if (r == 3 && ok) hi = (hi & 0xFF00FFFFu) | ((uint32_t)carry_cell_of<UNTR>(h, mem) << 16);   // own cell: what it carries
    uint32_t o[6];
    col_encode(lo, hi, (ok && r < 7) ? cv : 0u, o);
    const uint32_t next_w0 = BB_SHFL(o[0], r < 6 ? lane + 1 : lane + 2);
    if (r < 7) stage_record_words<21, 6>(tile, o, 7 * g + r, next_w0);
    BB_SYNCWARP();
    // ---- the four rows go to rows ids[4 w + q] of the output: byte stores by the whole warp -------------
    const uint32_t m_ok = BB_BALLOT(ok);
    const int row0 = BB_SHFL(env, 0), row1 = BB_SHFL(env, 8), row2 = BB_SHFL(env, 16), row3 = BB_SHFL(env, 24);
    const uint8_t *sb = reinterpret_cast<const uint8_t *>(tile);
    for (int i = lane; i < 4 * OBS_BYTES; i += 32) {
        const int q = i / OBS_BYTES;
        const int rq = q == 0 ? row0 : q == 1 ? row1 : q == 2 ? row2 : row3;
        if ((m_ok >> (8 * q)) & 1u) obs[(size_t)rq * OBS_BYTES + (i - q * OBS_BYTES)] = sb[i];
    }
    // ---- a reset ends no counted episode: only the error counter ---------------------------------------
    const uint32_t m_err = BB_BALLOT(error);
    if (lane == 0 && m_err) BB_ATOMIC_ADD(P.warp_counters + 4ull * wg + 3, (unsigned long long)BB_POPC(m_err));
}

}  // namespace bb
