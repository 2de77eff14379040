// full_obs.cuh -- the per-environment part of fully observable observations (gym_minigrid 1.0.x FullyObsWrapper):
// obs['image'] = grid.encode() of the whole grid, uint8[W][H][3] in x-major order, with the agent's cell overwritten by
// (OBJECT_TO_IDX['agent'] = 10, COLOR_TO_IDX['red'] = 0, agent_dir).  k_full_obs (pool.cu) runs it per selected env, one warp
// per env; tests/hostemu/full_obs_host.cpp compiles the same source for the host.
//
// The column-major copy of the grid (GT: W rows of rs_t bytes at gt_off, level_params.h) is already x-major, one cell byte
// type | color << 3 | state << 6 per cell, and the empty cell byte 0x01 decodes to (1, 0, 0) as Grid.encode() writes an
// empty cell.  So the frame is the GT rows without their padding, each byte split into its three fields.
#pragma once
#include "env_logic.cuh"
#include "grid_render.cuh"

namespace bb {

constexpr int FO_AGENT = 10;                               // OBJECT_TO_IDX['agent']
constexpr int FO_CELLS = MAXH * MAXH;                      // cells of the largest grid: bytes of one env's staged cells

// what one env's frame needs besides its cells: x-major indices x H + y of the agent's cell and of the cell to read as
// empty (-1: none), and the agent's heading
struct FullObsPose { int agent, hidden, dir; };

// grid_hidden_cell (grid_render.cuh): while a PutNext*Carrying episode is at step 0 the pool's grid still holds the object
// the reference has already put into the agent's hands
BB_HD FullObsPose full_obs_pose(const LevelParams &lp, const EnvHot &h, const ObjTab &ot, const InstrRec &ins)
{
    FullObsPose e;
    e.agent = h.x * lp.H + h.y;
    e.dir = h.dirflags & 3;
    const int c = grid_hidden_cell(lp, h, ot, ins);         // y W + x
    e.hidden = c < 0 ? -1 : (c % lp.W) * lp.H + c / lp.W;
    return e;
}

// byte r of the frame (cell r / 3, field r % 3), from the x-major cell bytes `cells` (the hidden cell already emptied)
BB_HD uint32_t full_obs_byte(const FullObsPose &e, const uint8_t *cells, int r)
{
    const int c = r / 3, f = r - 3 * c;
    if (c == e.agent) return f == 0 ? FO_AGENT : f == 1 ? C_RED : e.dir;
    const uint32_t b = cells[c];
    return f == 0 ? (b & 7u) : f == 1 ? ((b >> 3) & 7u) : (b >> 6);
}

// bytes r .. r + 3 of the frame as one little-endian word
BB_HD uint32_t full_obs_word(const FullObsPose &e, const uint8_t *cells, int r)
{
    return full_obs_byte(e, cells, r) | full_obs_byte(e, cells, r + 1) << 8 | full_obs_byte(e, cells, r + 2) << 16 |
           full_obs_byte(e, cells, r + 3) << 24;
}

// lane `lane` of `lanes`: its share of copying the env's x-major cell bytes (GT row x, byte y) into `cells`, the hidden cell as
// empty
BB_HD void full_obs_stage(const LevelParams &lp, const uint8_t *grid, const FullObsPose &e, uint8_t *cells, int lane, int lanes)
{
    for (int c = lane; c < lp.W * lp.H; c += lanes) {
        const int x = c / lp.H, y = c - x * lp.H;
        cells[c] = c == e.hidden ? (uint8_t)CELL_EMPTY : grid[lp.gt_off + x * lp.rs_t + y];
    }
}

// lane `lane` of `lanes` (>= 7): its share of storing the frame (F = 3 W H bytes) at dst, any alignment.  Consecutive lanes store
// consecutive aligned 32-bit words; the up to three bytes before the first word boundary (lanes 0-2) and after the last one
// (lanes 4-6) are stored singly.
BB_HD void full_obs_store(const FullObsPose &e, const uint8_t *cells, int F, uint8_t *dst, int lane, int lanes)
{
    const int head = (int)(-(uintptr_t)dst & 3u), nw = (F - head) >> 2, tail = head + 4 * nw;
    uint32_t *words = reinterpret_cast<uint32_t *>(dst + head);
    for (int i = lane; i < nw; i += lanes) words[i] = full_obs_word(e, cells, head + 4 * i);
    if (lane < head) dst[lane] = (uint8_t)full_obs_byte(e, cells, lane);
    else if (lane >= 4 && tail + lane - 4 < F) dst[tail + lane - 4] = (uint8_t)full_obs_byte(e, cells, tail + lane - 4);
}

// the whole frame of one env by `lanes` lanes run one after another (the host build; k_full_obs runs them as a warp)
BB_HD void full_obs_frame(const LevelParams &lp, const uint8_t *grid, const EnvHot &h, const ObjTab &ot, const InstrRec &ins,
                          uint8_t *cells, uint8_t *out, int lanes)
{
    const FullObsPose e = full_obs_pose(lp, h, ot, ins);
    for (int l = 0; l < lanes; l++) full_obs_stage(lp, grid, e, cells, l, lanes);
    for (int l = 0; l < lanes; l++) full_obs_store(e, cells, 3 * lp.W * lp.H, out, l, lanes);
}

}  // namespace bb
