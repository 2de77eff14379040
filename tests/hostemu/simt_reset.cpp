// simt_reset.cpp -- TEST-ONLY: k_reset8's role (babyai_b200/csrc/reset8.cuh) on the host with ONE OS THREAD PER LANE, over
// the pool of simt_rollout.cpp (included as is), together with what bb_pool_reset_envs runs around it: k_seed_sel and the
// selected generation passes.  Never loaded by babyai_b200/.
#include "simt_rollout.cpp"
#include "../../babyai_b200/csrc/reset8.cuh"

// a selected generation pass: the rings of the listed envs up to `target` levels, then their tail_pub
static void refill_sel(RPool *p, const int32_t *ids, int k, int target)
{
    for (int i = 0; i < k; i++) {
        const int e = ids[i];
        while ((int)(p->tail[e] - p->head[e]) < target) {
            GenMemX mem;
            p->attempts[e] += (uint32_t)generate_level(p->lp, slot_of(p, e, (int)(p->tail[e] % (uint32_t)p->D)), &p->rng[e], &p->locked_room[e], &mem);
            p->tail[e]++;
        }
        p->tail_pub[e] = p->tail[e];
    }
}

extern "C" {

void r2_seed_envs(RPool *p, const int32_t *ids, const uint64_t *seeds, int k)
{
    for (int i = 0; i < k; i++) {
        const int e = ids[i];
        p->rng[e].seed = seeds[i]; p->rng[e].draws = 0; p->locked_room[e] = 0xFF;
        p->tail[e] = p->head[e]; p->tail_pub[e] = p->head[e]; p->attempts[e] = 0;
    }
}

// bb_pool_reset_envs after the seeds: selected pass (freeze: 1 level, auto-reset: D), k_reset8 over the id list (every CTA
// of the grid, 128 threads each), and in auto-reset mode the second selected pass
void r2_reset_envs(RPool *p, const int32_t *ids, int k, uint8_t *obs, int8_t *dirs, int64_t *counters4)
{
    const LevelParams &lp = p->lp;
    refill_sel(p, ids, k, p->mode == BB_MODE_AUTORESET ? p->D : 1);
    const size_t sm8 = (size_t)S8_WARPS * 4 * (lp.cells_pad + S8_REC_FIXED) + (size_t)S8_WARPS * (S8_TILE_WORDS + 1) * 4;
    const int nctas = (k + 4 * S8_WARPS - 1) / (4 * S8_WARPS);
    for (int cta = 0; cta < nctas; cta++) {
        std::vector<WarpCtx> ctx(S8_WARPS);
        std::vector<uint8_t> smem(sm8 + 32, 0xEE);
        uint8_t *base = smem.data();
        while (((uintptr_t)base) & 15) base++;
        std::vector<std::thread> th;
        for (int tid = 0; tid < S8_THREADS; tid++)
            th.emplace_back([&, tid]() {
                tl_warp = &ctx[tid >> 5]; tl_lane = tid & 31;
                if (lp.kind == KIND_UNLOCK) reset8_role<HostPoolPtrs, true>(lp, p->P, ids, k, obs, dirs, base, tid & 31, tid >> 5, (unsigned)cta);
                else reset8_role<HostPoolPtrs, false>(lp, p->P, ids, k, obs, dirs, base, tid & 31, tid >> 5, (unsigned)cta);
            });
        for (auto &t : th) t.join();
    }
    if (p->mode == BB_MODE_AUTORESET) refill_sel(p, ids, k, p->D);
    for (int q = 0; q < 4; q++) counters4[q] = 0;
    for (size_t w = 0; w < p->counters.size() / 4; w++) for (int q = 0; q < 4; q++) counters4[q] += (int64_t)p->counters[4 * w + q];
}

}  // extern "C"
