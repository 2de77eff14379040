// rgb_tiles.h -- the 8 x 8 pixel tiles of RGBImgPartialObsWrapper (gym_minigrid 1.0.x `wrappers.py` / `minigrid.py`
// Grid.render_tile / `rendering.py`; used by the reference when 'pixel' is in the architecture name:
// scripts/train_rl.py:54-58, babyai/evaluate.py:91-92), rasterised ONCE on the host when a pool first renders.
//
// The wrapper's image is a pure function of the 7 x 7 x 3 observation: every view cell becomes one tile that depends only
// on (type, color, state), on whether the cell is visible (highlight) and on whether it is the agent's cell (3, 6) --
// 513 distinct tiles of 192 bytes:
//   id 0..255     visible cell with cell byte  type | color << 3 | state << 6   (object drawn, highlighted)
//   id 256        unseen cell (type 0): grid lines only, no highlight
//   id 257..512   the agent's own cell: 257 + cell byte (what it carries, or empty), the agent triangle on top, highlighted
// Each tile is drawn exactly as the reference package draws it: shapes are predicates on the unit square sampled at the
// pixel centres of a 24 x 24 supersampled tile (float64, same operation order as the Python code so that the comparisons
// and the box filter round identically), highlight = img + 0.3 (255 - img), 3 x 3 box filter as two successive means,
// truncation to uint8.  tests/test_rgb.py compares every tile with the oracle shim's literal restatement of that code.
//
// The same rasteriser, at any tile size from 1 to 64 and with the agent facing any direction, builds the tables of
// full-grid frames (MiniGridEnv.render('rgb_array'), k_render_grid): render_grid_tiles() at the end of this file,
// rasterised on the host the first time a pool renders at a tile size (tests/test_render_grid.py checks every tile).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

namespace bb_rgb {

constexpr int TILE = 8, SUB = 3;                                // the partial-view tiles: 8 px, drawn at 24 x 24 samples
constexpr int N_TILES = 513, TILE_BYTES = TILE * TILE * 3;      // 192
constexpr int ID_UNSEEN = 256, ID_AGENT0 = 257;
constexpr int MAX_TILE_SIZE = 64;                               // largest tile size the full-grid table is built for

// a square RGB canvas of res x res samples (tile_size * SUB)
struct Canvas {
    int res; std::vector<uint8_t> px;
    explicit Canvas(int r) : res(r), px((size_t)r * r * 3, 0) {}
    uint8_t *at(int y, int x) { return &px[((size_t)y * res + x) * 3]; }
    const uint8_t *at(int y, int x) const { return &px[((size_t)y * res + x) * 3]; }
};

struct Rect { double x0, x1, y0, y1; bool in(double x, double y) const { return x >= x0 && x <= x1 && y >= y0 && y <= y1; } };
struct Circle { double cx, cy, r; bool in(double x, double y) const { return (x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r; } };

template <class F>
static void fill(Canvas &c, const F &f, const double col[3])
{
    for (int y = 0; y < c.res; y++)
        for (int x = 0; x < c.res; x++) {
            const double yf = (y + 0.5) / c.res, xf = (x + 0.5) / c.res;
            if (f.in(xf, yf)) for (int k = 0; k < 3; k++) c.at(y, x)[k] = (uint8_t)col[k];     // float -> uint8: truncation
        }
}

// point_in_triangle(a, b, c) behind rotate_fn(.., cx = cy = 0.5, theta)
struct RotTriangle {
    double ax, ay, bx, by, cx_, cy_, cs, sn;
    bool in(double x, double y) const
    {
        x = x - 0.5; y = y - 0.5;
        const double x2 = 0.5 + x * cs - y * sn;
        const double y2 = 0.5 + y * cs + x * sn;
        const double v0x = cx_ - ax, v0y = cy_ - ay, v1x = bx - ax, v1y = by - ay, v2x = x2 - ax, v2y = y2 - ay;
        const double dot00 = v0x * v0x + v0y * v0y, dot01 = v0x * v1x + v0y * v1y, dot02 = v0x * v2x + v0y * v2y;
        const double dot11 = v1x * v1x + v1y * v1y, dot12 = v1x * v2x + v1y * v2y;
        const double inv = 1 / (dot00 * dot11 - dot01 * dot01);
        const double u = (dot11 * dot02 - dot01 * dot12) * inv, v = (dot00 * dot12 - dot01 * dot02) * inv;
        return u >= 0 && v >= 0 && (u + v) < 1;
    }
};

static const double COLORS[6][3] = { { 255, 0, 0 }, { 0, 255, 0 }, { 0, 0, 255 }, { 112, 39, 195 }, { 255, 255, 0 }, { 100, 100, 100 } };

// WorldObj.render of the object a cell byte decodes to (WorldObj.decode: empty / unseen -> nothing)
static void draw_object(Canvas &cv, int type, int color, int state)
{
    if (color > 5) return;
    const double *c = COLORS[color];
    const double black[3] = { 0, 0, 0 };
    if (type == 2) fill(cv, Rect{ 0, 1, 0, 1 }, c);                                   // wall
    else if (type == 4) {                                                             // door
        if (state == 0) {
            fill(cv, Rect{ 0.88, 1.00, 0.00, 1.00 }, c);
            fill(cv, Rect{ 0.92, 0.96, 0.04, 0.96 }, black);
        } else if (state == 2) {
            const double dim[3] = { 0.45 * c[0], 0.45 * c[1], 0.45 * c[2] };
            fill(cv, Rect{ 0.00, 1.00, 0.00, 1.00 }, c);
            fill(cv, Rect{ 0.06, 0.94, 0.06, 0.94 }, dim);
            fill(cv, Rect{ 0.52, 0.75, 0.50, 0.56 }, c);
        } else {
            fill(cv, Rect{ 0.00, 1.00, 0.00, 1.00 }, c);
            fill(cv, Rect{ 0.04, 0.96, 0.04, 0.96 }, black);
            fill(cv, Rect{ 0.08, 0.92, 0.08, 0.92 }, c);
            fill(cv, Rect{ 0.12, 0.88, 0.12, 0.88 }, black);
            fill(cv, Circle{ 0.75, 0.50, 0.08 }, c);
        }
    } else if (type == 5) {                                                           // key
        fill(cv, Rect{ 0.50, 0.63, 0.31, 0.88 }, c);
        fill(cv, Rect{ 0.38, 0.50, 0.59, 0.66 }, c);
        fill(cv, Rect{ 0.38, 0.50, 0.81, 0.88 }, c);
        fill(cv, Circle{ 0.56, 0.28, 0.190 }, c);
        fill(cv, Circle{ 0.56, 0.28, 0.064 }, black);
    } else if (type == 6) fill(cv, Circle{ 0.5, 0.5, 0.31 }, c);                      // ball
    else if (type == 7) {                                                             // box
        fill(cv, Rect{ 0.12, 0.88, 0.12, 0.88 }, c);
        fill(cv, Rect{ 0.18, 0.82, 0.18, 0.82 }, black);
        fill(cv, Rect{ 0.16, 0.84, 0.47, 0.53 }, c);
    }
    // (floor / goal / lava never occur in BabyAI levels: drawn as empty)
}

// Grid.render_tile(obj, agent_dir, highlight, tile_size, subdivs = 3) for BOTH highlight values at once (the highlight is applied
// after everything is drawn, so the two tiles share one canvas): out_plain / out_hl receive tile_size x tile_size x 3 bytes
// each (either may be null).  agent_dir: -1 = no agent, else 0..3 (theta = 0.5 * pi * agent_dir, evaluated as Python does).
static void render_tile_pair(int cell_byte, bool has_obj, int agent_dir, int tile_size, uint8_t *out_plain, uint8_t *out_hl)
{
    const int res = tile_size * SUB;
    Canvas cv(res);
    const double grey[3] = { 100, 100, 100 }, red[3] = { 255, 0, 0 };
    fill(cv, Rect{ 0, 0.031, 0, 1 }, grey);
    fill(cv, Rect{ 0, 1, 0, 0.031 }, grey);
    if (has_obj) draw_object(cv, cell_byte & 7, (cell_byte >> 3) & 7, cell_byte >> 6);
    if (agent_dir >= 0) {
        const double theta = 0.5 * M_PI * agent_dir;
        fill(cv, RotTriangle{ 0.12, 0.19, 0.87, 0.50, 0.12, 0.81, cos(-theta), sin(-theta) }, red);
    }
    for (int hl = 0; hl < 2; hl++) {
        uint8_t *out = hl ? out_hl : out_plain;
        if (!out) continue;
        // highlight = img + 0.3 (255 - img), clipped and truncated; then the downsample: mean over the 3 sub-columns, then
        // mean over the 3 sub-rows (numpy float64, in that order), truncated
        auto px = [&](int y, int x, int k) -> double {
            const uint8_t p = cv.at(y, x)[k];
            if (!hl) return (double)p;
            double b = (double)p + 0.30 * (double)(uint8_t)(255 - p);
            b = b < 0 ? 0 : b > 255 ? 255 : b;
            return (double)(uint8_t)b;
        };
        for (int ty = 0; ty < tile_size; ty++)
            for (int tx = 0; tx < tile_size; tx++)
                for (int k = 0; k < 3; k++) {
                    double m[SUB];
                    for (int sy = 0; sy < SUB; sy++) {
                        const int y = ty * SUB + sy, x = tx * SUB;
                        m[sy] = ((px(y, x, k) + px(y, x + 1, k)) + px(y, x + 2, k)) / 3.0;
                    }
                    const double v = ((m[0] + m[1]) + m[2]) / 3.0;
                    out[((size_t)ty * tile_size + tx) * 3 + k] = (uint8_t)v;
                }
    }
}

// the partial-view table: N_TILES x 8 x 8 x 3 bytes (the agent of the view always faces up: agent_dir 3)
inline void render_all_tiles(uint8_t *lut)
{
    for (int b = 0; b < 256; b++) {
        const bool obj = (b & 7) >= 2;                   // types 0 (unseen) and 1 (empty) decode to no object
        render_tile_pair(b, obj, -1, TILE, nullptr, lut + (size_t)b * TILE_BYTES);
        render_tile_pair(b, obj, 3, TILE, nullptr, lut + (size_t)(ID_AGENT0 + b) * TILE_BYTES);
    }
    render_tile_pair(0, false, -1, TILE, lut + (size_t)ID_UNSEEN * TILE_BYTES, nullptr);
}

// ---- full-grid frames (MiniGridEnv.render('rgb_array'), k_render_grid) -------------------------------------------------
// A BabyAI grid cell holds one of 43 cell bytes: empty; wall, key, ball, box in six colours; doors in six colours and three
// states.  The full-grid table is COMPACT over those 43 (not over all 256 bytes: 430 tiles instead of 2 560, a sixth of the
// host rasterisation time on first use and of the table the kernel keeps in L2 -- 5.3 MB at tile size 64):
//   tile id = (highlight * GRID_AGENTS + agent) * GRID_CELLS + cell index
//   highlight 0 / 1; agent 0 = no agent on the cell, 1 + d = the agent facing direction d; cell index: grid_cell_index()
// Each tile is tile_size x tile_size x 3 bytes.
constexpr int GRID_CELLS = 43, GRID_AGENTS = 5, GRID_TILES = 2 * GRID_AGENTS * GRID_CELLS;

// cell index 0 = empty, 1 + 6 k + color for k = 0 wall, 1 key, 2 ball, 3 box, 25 + 6 state + color for doors.  Bytes no
// BabyAI grid holds (unseen, bad colours or states) map to 0.
#if defined(__CUDACC__)
__host__ __device__
#endif
inline int grid_cell_index(int b)
{
    const int t = b & 7, c = (b >> 3) & 7, s = b >> 6;
    if (c > 5) return 0;
    if (t == 4) return s <= 2 ? 25 + 6 * s + c : 0;
    if (s != 0) return 0;
    if (t == 2) return 1 + c;
    if (t >= 5) return 1 + 6 * (t - 4) + c;
    return 0;
}
// the cell byte of cell index k (the inverse of grid_cell_index on the 43 bytes)
inline int grid_cell_byte(int k)
{
    if (k == 0) return 1;
    if (k <= 24) { const int t = k <= 6 ? 2 : 4 + (k - 1) / 6; return t | (((k - 1) % 6) << 3); }
    return 4 | (((k - 25) % 6) << 3) | (((k - 25) / 6) << 6);
}

// the whole full-grid table for one tile size: GRID_TILES x tile_size x tile_size x 3 bytes
static void render_grid_tiles(int tile_size, uint8_t *lut)
{
    const size_t tb = (size_t)tile_size * tile_size * 3;
    for (int agent = 0; agent < GRID_AGENTS; agent++)
        for (int k = 0; k < GRID_CELLS; k++) {
            const int b = grid_cell_byte(k);
            render_tile_pair(b, (b & 7) >= 2, agent - 1, tile_size, lut + (size_t)(agent * GRID_CELLS + k) * tb,
                             lut + (size_t)((GRID_AGENTS + agent) * GRID_CELLS + k) * tb);
        }
}

}  // namespace bb_rgb
