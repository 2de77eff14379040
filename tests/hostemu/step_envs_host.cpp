// step_envs_host.cpp -- TEST-ONLY: k_step8_sel's role (babyai_b200/csrc/step8_sel.cuh) on the host with ONE OS THREAD PER LANE,
// over the ring-layout pool of simt_rollout.cpp, beside the reset / save / load entry points of save_load_host.cpp (included as
// is).  Never loaded by babyai_b200/.
#include "save_load_host.cpp"
#include "../../babyai_b200/csrc/step8_sel.cuh"

extern "C" {

// bb_pool_step_envs: k_step8_sel over the id list (every CTA of the grid, 128 threads each; the device splits longer lists into
// launches of 4 096 ids, which changes nothing a role computes), then what the generation schedule has done by the next step in
// auto-reset mode: the listed rings topped up to D (an unlisted env has consumed nothing)
void r2_step_envs(RPool *p, const int32_t *ids, int k, const void *actions, int action_bytes, uint8_t *obs, float *reward,
                  uint8_t *done, int8_t *dirs, int64_t *counters4)
{
    const LevelParams &lp = p->lp;
    const size_t sm8 = (size_t)S8_WARPS * 4 * (lp.cells_pad + S8_REC_FIXED) + (size_t)S8_WARPS * (S8_TILE_WORDS + 1) * 4;
    const int nctas = (k + 4 * S8_WARPS - 1) / (4 * S8_WARPS);
    const bool untr = lp.kind == KIND_UNLOCK;
    for (int cta = 0; cta < nctas; cta++) {
        std::vector<WarpCtx> ctx(S8_WARPS);
        std::vector<uint8_t> smem(sm8 + 32, 0xEE);
        uint8_t *base = smem.data();
        while (((uintptr_t)base) & 15) base++;
        std::vector<std::thread> th;
        for (int tid = 0; tid < S8_THREADS; tid++)
            th.emplace_back([&, tid]() {
                tl_warp = &ctx[tid >> 5]; tl_lane = tid & 31;
                const int lane = tid & 31, warp = tid >> 5;
                if (action_bytes == 8) {
                    if (untr) step8_sel_role<HostPoolPtrs, 8, true>(lp, p->P, ids, k, actions, obs, reward, done, dirs, p->mode, base, lane, warp, (unsigned)cta);
                    else step8_sel_role<HostPoolPtrs, 8, false>(lp, p->P, ids, k, actions, obs, reward, done, dirs, p->mode, base, lane, warp, (unsigned)cta);
                } else {
                    if (untr) step8_sel_role<HostPoolPtrs, 1, true>(lp, p->P, ids, k, actions, obs, reward, done, dirs, p->mode, base, lane, warp, (unsigned)cta);
                    else step8_sel_role<HostPoolPtrs, 1, false>(lp, p->P, ids, k, actions, obs, reward, done, dirs, p->mode, base, lane, warp, (unsigned)cta);
                }
            });
        for (auto &t : th) t.join();
    }
    if (p->mode == BB_MODE_AUTORESET) refill_sel(p, ids, k, p->D);
    for (int q = 0; q < 4; q++) counters4[q] = 0;
    for (size_t w = 0; w < p->counters.size() / 4; w++) for (int q = 0; q < 4; q++) counters4[q] += (int64_t)p->counters[4 * w + q];
}

}  // extern "C"
