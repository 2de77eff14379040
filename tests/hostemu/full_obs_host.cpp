// full_obs_host.cpp -- TEST-ONLY host build of the fully observable observations: the host build of the full-grid frames
// (render_grid_host.cpp: hostemu.cpp + grid_render.cuh, included as is; RGBImgObsWrapper) plus k_full_obs's per-env source
// (babyai_b200/csrc/full_obs.cuh; FullyObsWrapper), its 32 lanes run one after another.  Never loaded by babyai_b200/.
#include "render_grid_host.cpp"
#include "../../babyai_b200/csrc/full_obs.cuh"

extern "C" {

// FullyObsWrapper.observation(obs)['image'] of env e's current state -> uint8[W][H][3] at out (any alignment: the kernel's
// frames start at every offset modulo 4)
void fo_full_obs(HPool *p, int e, uint8_t *out)
{
    const Slot &s = p->live[e];
    uint8_t cells[FO_CELLS];
    full_obs_frame(p->lp, s.grid.data(), s.hot, s.obj, s.ins, cells, out, 32);
}

}  // extern "C"
