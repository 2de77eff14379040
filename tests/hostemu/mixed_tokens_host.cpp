// mixed_tokens_host.cpp -- TEST-ONLY host build of the level generators (env_logic.cuh) for the mission-token width of mixed
// pools.  A group of a mixed pool generates its levels with lp.max_tokens raised to the widest group's; this file generates the
// same stream of levels at the level's natural width and at a wider one and compares every output byte.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../babyai_b200/csrc/env_logic.cuh"
#include "../../babyai_b200/csrc/level_params.h"
#include "../../include/babyai_b200.h"

using namespace bb;

struct Out {
    std::vector<uint8_t> grid; EnvHot hot; ObjTab obj; InstrRec ins; int16_t tok[MAXTOK];
    Out(const LevelParams &lp, int16_t fill) : grid(lp.cells_pad, 0) { memset(&hot, 0, sizeof hot); memset(&obj, 0, sizeof obj);
                                                                      memset(&ins, 0, sizeof ins); for (int k = 0; k < MAXTOK; k++) tok[k] = fill; }
    LevelOut out() { LevelOut o; o.grid = grid.data(); o.hot = &hot; o.obj = &obj; o.ins = &ins; o.tok = tok; return o; }
};

// one level from the stream (rng, locked_room): the small-level generator (generate_small + emit_small_level) where the level
// has one, else generate_level -- what k_gen_small / k_gen run
static int gen(const LevelParams &lp, Out &o, RngRec *r, uint8_t *lr)
{
    if (lp.small) {
        RngScalar rng; rng.init(r->seed, r->draws);
        SmallLevel L;
        const int att = generate_small(lp, rng, L);
        emit_small_level(lp, L, o.out());
        r->draws = rng.draws;
        return att;
    }
    GenMemX mem;
    return generate_level(lp, o.out(), r, lr, &mem);
}

extern "C" {

// natural width of the level's missions
int mt_max_tokens(const bb_level_spec *spec)
{
    LevelParams lp;
    return make_level_params(spec, &lp) ? -1 : lp.max_tokens;
}

// `levels` consecutive levels of stream `seed` at the natural width and at `wide` tokens.  Returns 0 when every level agrees:
// grid, hot record, object table, instruction record, draws, attempts and locked room equal; tokens equal up to the natural
// width, the natural run writes nothing after it and the wide run writes zeros there.  Else 1 + the first level that differs.
// tok_out: int16 [levels][MAXTOK] tokens of the wide run (for the caller's own look).
int mt_compare(const bb_level_spec *spec, uint64_t seed, int levels, int wide, int16_t *tok_out)
{
    LevelParams lp, lw;
    if (make_level_params(spec, &lp) || make_level_params(spec, &lw)) return -1;
    lw.max_tokens = wide;
    RngRec ra, rb; ra.seed = rb.seed = seed; ra.draws = rb.draws = 0;
    uint8_t la = 0xFF, lb = 0xFF;
    for (int k = 0; k < levels; k++) {
        Out a(lp, 0x7777), b(lw, 0x5555);
        const int aa = gen(lp, a, &ra, &la), ab = gen(lw, b, &rb, &lb);
        bool ok = aa == ab && ra.draws == rb.draws && la == lb && a.grid == b.grid && !memcmp(&a.hot, &b.hot, sizeof(EnvHot)) &&
                  !memcmp(&a.obj, &b.obj, sizeof(ObjTab)) && !memcmp(&a.ins, &b.ins, sizeof(InstrRec));
        for (int t = 0; t < MAXTOK && ok; t++) {
            if (t < lp.max_tokens) ok = a.tok[t] == b.tok[t];
            else ok = a.tok[t] == 0x7777 && (t < wide ? b.tok[t] == 0 : b.tok[t] == 0x5555);
        }
        if (tok_out) memcpy(tok_out + (size_t)k * MAXTOK, b.tok, sizeof b.tok);
        if (!ok) return 1 + k;
    }
    return 0;
}

}  // extern "C"
