// reset_envs_host.cpp -- TEST-ONLY host build of bb_pool_reset_envs' semantics: the host build of the kernel logic
// (hostemu.cpp, included as is) plus a per-env seed and reset.  Never loaded by babyai_b200/.
#include "hostemu.cpp"

extern "C" {

// env.seed(seeds[k]) for envs ids[k] only: what k_seed_sel does (a fresh random stream, locked_room cleared, no level kept)
void he_seed_envs(HPool *p, const int32_t *ids, const uint64_t *seeds, int k)
{
    for (int i = 0; i < k; i++) {
        const int e = ids[i];
        p->rng[e].seed = seeds[i]; p->rng[e].draws = 0; p->locked_room[e] = 0xFF; p->sready[e] = 0; p->attempts[e] = 0;
    }
}

// env.reset() for envs ids[k] only (he_reset per env): the next level of the env's stream, its first observation to row
// ids[k] of obs; other rows are not written
void he_reset_envs(HPool *p, const int32_t *ids, int k, uint8_t *obs, int8_t *dir)
{
    for (int i = 0; i < k; i++) {
        const int e = ids[i];
        if (!p->sready[e]) gen_spare(p, e);
        p->live[e] = p->spare[e]; p->sready[e] = 0;
        if (p->mode == BB_MODE_AUTORESET) gen_spare(p, e);
        obs_of(p, e, obs + (size_t)e * OBS_BYTES);
        if (dir) dir[e] = (int8_t)(p->live[e].hot.dirflags & 3);
    }
}

}  // extern "C"
