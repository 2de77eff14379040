// grid_render.cuh -- the per-environment part of full-grid frames (MiniGridEnv.render('rgb_array', highlight, tile_size),
// gym_minigrid 1.0.x): which table tile (rgb_tiles.h, render_grid_tiles) every grid cell shows.  k_render_grid (pool.cu)
// runs it per selected env and streams the tiles out; tests/hostemu compiles the same source for the host.
//
// The reference draws cell (x, y) as Grid.render_tile(cell, agent_dir if the agent is at (x, y), highlight_mask[x, y]).
// The highlight mask is gen_obs_grid()'s vis_mask (process_vis of the agent's 7 x 7 view, before the carried object is
// written into the agent's view cell) mapped to the world: view cell (vi, vj) is agent_pos + f (6 - vj) + r (vi - 3), and
// only cells inside the grid are marked.  The visibility is the observation kernels' own code (col_load / col_see /
// vis_rows, env_logic.cuh), so a cell is highlighted exactly when its view cell in the env's observation has type != 0.
#pragma once
#include "env_logic.cuh"
#include "rgb_tiles.h"

namespace bb {

// read-only word access to one env's grid bytes (both stored orientations), what col_load needs
struct GridWords {
    const uint8_t *g;
    BB_HD uint32_t word_at(int off) const { return load_u32(g + off); }
};

// vis_mask of the pose as a 64-bit set: bit 8 vj + vi = view cell (vi, vj) is visible
template <class M>
BB_HD uint64_t grid_view_vis(const LevelParams &lp, const M &mem, int ax, int ay, int dir)
{
    const ViewGeom v = view_geom(lp, ax, ay, dir);
    uint32_t see[7] = { 0, 0, 0, 0, 0, 0, 0 }, vis[7];
    for (int vi = 0; vi < 7; vi++) {
        uint32_t lo, hi;
        col_load(mem, v, vi, lo, hi);
        const uint32_t cm = col_see(lo, hi);                   // bit vj
        for (int vj = 0; vj < 7; vj++) see[vj] |= ((cm >> vj) & 1u) << vi;
    }
    vis_rows(see, vis);
    uint64_t m = 0;
    for (int vj = 0; vj < 7; vj++) m |= (uint64_t)vis[vj] << (8 * vj);
    return m;
}

// Level_PutNext*Carrying (bonus_levels.py:821-829) takes obj_a off the grid into the agent's hands right after reset; the pool
// does it at the start of the first step (step_env), so while step_count is 0 the pool's grid still holds it.  Returns the
// index y * W + x of the cell to draw as empty, or -1.
BB_HD int grid_hidden_cell(const LevelParams &lp, const EnvHot &h, const ObjTab &ot, const InstrRec &ins)
{
    if (lp.bonus != BN_PUTNEXT || h.step_count != 0 || ins.pad0 == 0) return -1;
    return ot.y[ins.pad0 - 1] * lp.W + ot.x[ins.pad0 - 1];
}

// table tile of cell (x, y) holding `cell` (a cell byte), for the agent at (ax, ay) facing `dir` with view visibility `vis`
BB_HD int grid_tile_id(int cell, int x, int y, int ax, int ay, int dir, uint64_t vis, bool highlight)
{
    const int fx = dir_dx(dir), fy = dir_dy(dir), rx = -fy, ry = fx;
    const int dx = x - ax, dy = y - ay;
    const int vj = 6 - (dx * fx + dy * fy), vi = 3 + (dx * rx + dy * ry);        // the inverse of the view -> world map
    const bool hl = highlight && vi >= 0 && vi < 7 && vj >= 0 && vj < 7 && ((vis >> (8 * vj + vi)) & 1u);
    const int agent = (x == ax && y == ay) ? 1 + dir : 0;
    return ((hl ? bb_rgb::GRID_AGENTS : 0) + agent) * bb_rgb::GRID_CELLS + bb_rgb::grid_cell_index(cell);
}

// every cell of one env, row-major (H x W tile ids); the kernel splits this loop over its threads
BB_HD void grid_tile_ids(const LevelParams &lp, const uint8_t *grid, const EnvHot &h, const ObjTab &ot, const InstrRec &ins,
                         bool highlight, uint16_t *ids)
{
    const GridWords mem{ grid };
    const int dir = h.dirflags & 3;
    const uint64_t vis = grid_view_vis(lp, mem, h.x, h.y, dir);
    const int hidden = grid_hidden_cell(lp, h, ot, ins);
    for (int y = 0; y < lp.H; y++)
        for (int x = 0; x < lp.W; x++) {
            const int cell = y * lp.W + x == hidden ? CELL_EMPTY : get_cell(lp, grid, x, y);
            ids[y * lp.W + x] = (uint16_t)grid_tile_id(cell, x, y, h.x, h.y, dir, vis, highlight);
        }
}

}  // namespace bb
