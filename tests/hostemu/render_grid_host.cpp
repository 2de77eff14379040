// render_grid_host.cpp -- TEST-ONLY host build of the full-grid frame path: the host build of the kernel logic (hostemu.cpp,
// included as is) plus k_render_grid's per-env source (babyai_b200/csrc/grid_render.cuh) over the host-rasterised table
// (rgb_tiles.h).  Never loaded by babyai_b200/.
#include "hostemu.cpp"
#include "../../babyai_b200/csrc/grid_render.cuh"

extern "C" {

// MiniGridEnv.render('rgb_array') of env e's current state, assembled cell by cell -> uint8[H * ts][W * ts][3]
void rg_render_grid(HPool *p, int e, int ts, int highlight, uint8_t *out)
{
    const LevelParams &lp = p->lp;
    const size_t tb = (size_t)ts * ts * 3, row = (size_t)lp.W * ts * 3;
    std::vector<uint8_t> lut(bb_rgb::GRID_TILES * tb);
    bb_rgb::render_grid_tiles(ts, lut.data());
    std::vector<uint16_t> ids((size_t)lp.H * lp.W);
    const Slot &s = p->live[e];
    grid_tile_ids(lp, s.grid.data(), s.hot, s.obj, s.ins, highlight != 0, ids.data());
    for (int y = 0; y < lp.H; y++)
        for (int x = 0; x < lp.W; x++)
            for (int ty = 0; ty < ts; ty++)
                memcpy(out + ((size_t)y * ts + ty) * row + (size_t)x * ts * 3, lut.data() + ids[y * lp.W + x] * tb + (size_t)ty * ts * 3,
                       (size_t)ts * 3);
}
void rg_grid_tiles(int ts, uint8_t *out) { bb_rgb::render_grid_tiles(ts, out); }
int rg_grid_cell_index(int b) { return bb_rgb::grid_cell_index(b); }

}  // extern "C"
