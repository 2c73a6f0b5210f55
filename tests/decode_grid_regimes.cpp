// decode_grid_regimes.cpp -- which code paths of decode_step_kernel a plan reaches at a given grid, from the schedule alone.
//
// Compiled by tests/test_decode_grid_regimes.py with g++ against exllama_b200/csrc/decode_step_sched.h, the header decode_step.cu
// includes.  The GEMV, ATT and HEAD phases cut their units with range_lo(U, cta, G), so the grid decides whether a CTA's range
// crosses a matrix boundary, whether it runs past one tile's K stages, and whether the grid or the per-head cap limits ATT.  The
// proofs themselves are the other checkers' (decode_sched_check*.cpp); this only names the regimes a case reaches.
#include "../exllama_b200/csrc/decode_step_sched.h"

using namespace ds_sched;

namespace {

// a CTA's unit range of a GEMV phase spans tiles of two matrices (the producer's matrix switch inside one range)
bool crosses_matrix(const Phase& p)
{
    for (int c = 0; c < p.G; c++) {
        const int lo = range_lo(p.U, c, p.G), hi = range_lo(p.U, c + 1, p.G);
        if (hi > lo && mat_of_tile(p, lo / p.spt) != mat_of_tile(p, (hi - 1) / p.spt)) return true;
    }
    return false;
}

// the longest unit range of a phase
int longest_share(const Phase& p)
{
    int m = 0;
    for (int c = 0; c < p.G; c++) {
        const int n = range_lo(p.U, c + 1, p.G) - range_lo(p.U, c, p.G);
        m = n > m ? n : m;
    }
    return m;
}

} // namespace

enum {
    RG_QKV_CROSS,          // a QKV range crosses q|k or k|v
    RG_GU_CROSS,           // a GU range crosses gate|up
    RG_QKV_LONG,           // a QKV range is longer than one tile's K stages (spt)
    RG_GU_LONG,
    RG_DOWN_LONG,
    RG_ATT_GRID_LIMITED,   // ATT: every CTA of the grid takes part, fewer than cap x KV heads
    RG_ATT_CAP_LIMITED,    // ATT: cap x KV heads < grid, the rest of the grid sits the phase out
    RG_RESET,              // the host resets the attention partial table before this launch
    RG_XST_COMPACT,        // batched / multi-token plan: compact x staging (batch_xstages < spt_max)
    RG_XST_FULL,           // ... batch_xstages == spt_max
    RG_COUNT
};

// kind: 0 one sequence, 1 a batch of nb sequences (the longest at past_len), 2 nb tokens of one sequence at past_len.
// out[RG_COUNT]: 1 where the launch reaches the regime.  Returns RG_COUNT.
extern "C" int dg_regimes(int H, int HQ, int I, int heads, int kv_heads, int grid, int kind, int nb, int past_len, int* out)
{
    AttDims a = {};
    a.H = H; a.HQ = HQ; a.HKV = kv_heads * TILE; a.I = I; a.heads = heads; a.kv_heads = kv_heads; a.past_len = past_len;
    for (int i = 0; i < RG_COUNT; i++) out[i] = 0;
    const Phase qkv = phase_of(a, PH_QKV, grid), gu = phase_of(a, PH_GU, grid), down = phase_of(a, PH_DOWN, grid);
    out[RG_QKV_CROSS] = crosses_matrix(qkv);
    out[RG_GU_CROSS] = crosses_matrix(gu);
    out[RG_QKV_LONG] = longest_share(qkv) > qkv.spt;
    out[RG_GU_LONG] = longest_share(gu) > gu.spt;
    out[RG_DOWN_LONG] = longest_share(down) > down.spt;
    const int kvh = (kind == 1 ? nb : 1) * kv_heads;
    const int cap = kind == 2 ? ATT_CTAS_PER_KV_HEAD : att_cap((kind == 1 ? nb : 1) * heads, kvh);
    const Phase att = kind == 2 ? phase_of_multi(a, PH_ATT, grid) : phase_of(a, PH_ATT, grid, kind == 1 ? nb : 1);
    out[RG_ATT_GRID_LIMITED] = att.G == grid && grid < cap * kvh;
    out[RG_ATT_CAP_LIMITED] = att.G == cap * kvh && att.G < grid;
    out[RG_RESET] = kind == 2 ? att_needs_reset_multi(heads, kv_heads, past_len, grid) : att_needs_reset(heads, kv_heads, past_len, grid, kind == 1 ? nb : 1);
    if (kind != 0) {
        const int xst = batch_xstages(H, HQ, kv_heads * TILE, I, grid);
        out[RG_XST_COMPACT] = xst < spt_max_for(H, HQ, I);
        out[RG_XST_FULL] = xst == spt_max_for(H, HQ, I);
    }
    return RG_COUNT;
}
