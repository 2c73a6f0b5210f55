// prefill_attn_sched.h -- the work list of prefill_attn_kernel (prefill_attn.cu): which (sequence, KV group, 64-row query tile) a
// CTA computes, and how many CTAs a launch has.
//
// Plain C++ with no CUDA types: the kernel includes it as device code, and tests/test_prefill_ragged_schedule.py compiles the same
// header with g++ (tests/prefill_ragged_check.cpp) to check on the CPU that every tile is computed exactly once and no CTA is empty.
//
// One description covers both entry points:
//   uniform  (n_seq == 0, exl_prefill_attn)  bsz sequences of q_len tokens at one past_len, sequence b in cache sequence b and in
//            token rows [b * q_len, (b + 1) * q_len).  Grid (kv_heads * bsz, row_tiles): x = b * kv_heads + g, y = the row tile
//            counted from the last, so the longest rows start first.  A stride rule, not a table: any bsz.
//   ragged   (n_seq >= 1, exl_prefill_attn_ragged)  up to PA_MAX_SEQ sequences, each with its own q_len, past_len, cache
//            sequence and first token row.  Grid (cta0[n_seq], 1): the sequences in descending past_len + q_len order, each owning
//            kv_heads * its own row tiles CTAs (none for padding), within a sequence the row tiles from the last, as uniform.
#pragma once

#if defined(__CUDACC__)
#define PA_HD __host__ __device__ __forceinline__
#else
#define PA_HD static inline
#endif

namespace pa_sched {

constexpr int BM = 64;                   // query rows per CTA (row r of a (sequence, KV group) = token r / n_rep, head r % n_rep)
constexpr int MAX_SEQ = 64;              // sequences of one ragged description (EXL_RAGGED_MAX_SEQ)

struct Work {
    int n_seq;                           // 0: uniform; else the ragged sequences below, in launch order
    int kv_heads, n_rep;
    int bsz, q_len, past_len, row_tiles; // uniform
    int cta0[MAX_SEQ + 1];               // ragged: launch-order sequence s owns CTAs [cta0[s], cta0[s + 1])
    int q_len_s[MAX_SEQ], past_s[MAX_SEQ], cache_s[MAX_SEQ], tok0_s[MAX_SEQ];
};

// one CTA's tile: query rows [m0, min(m0 + BM, q_len * n_rep)) of KV group g of the sequence whose tokens start at token row tok0 and
// whose keys are rows [0, past_len + t] of cache sequence cache_seq
struct Tile { int cache_seq, tok0, q_len, past_len, g, m0; };

PA_HD int row_tiles_of(int q_len, int n_rep) { return (int)(((long long)q_len * n_rep + BM - 1) / BM); }

// uniform description: bsz sequences of q_len tokens at past_len
PA_HD void make_uniform(Work& w, int bsz, int q_len, int past_len, int kv_heads, int n_rep)
{
    w.n_seq = 0; w.kv_heads = kv_heads; w.n_rep = n_rep;
    w.bsz = bsz; w.q_len = q_len; w.past_len = past_len; w.row_tiles = row_tiles_of(q_len, n_rep);
}

// ragged description of n (1..MAX_SEQ, arguments already validated) sequences given in packed token order: sequence i owns token
// rows [sum_{j<i} q_len[j], + q_len[i]).  Returns the CTA count, sum_i kv_heads * row_tiles_of(q_len[i], n_rep).
PA_HD long long make_ragged(Work& w, int n, const int* q_len, const int* past_len, const int* cache_seq, int kv_heads, int n_rep)
{
    w.n_seq = n; w.kv_heads = kv_heads; w.n_rep = n_rep;
    w.bsz = n; w.q_len = 0; w.past_len = 0; w.row_tiles = 0;
    int order[MAX_SEQ], tok0[MAX_SEQ];
    int t = 0;
    for (int i = 0; i < n; i++) { tok0[i] = t; t += q_len[i]; }
    for (int i = 0; i < n; i++) {        // stable insertion sort, descending past_len + q_len (the longest rows first)
        const long long c = (long long)past_len[i] + q_len[i];
        int j = i;
        for (; j > 0 && (long long)past_len[order[j - 1]] + q_len[order[j - 1]] < c; j--) order[j] = order[j - 1];
        order[j] = i;
    }
    long long ctas = 0;
    for (int s = 0; s < n; s++) {
        const int i = order[s];
        w.cta0[s] = (int)ctas;
        w.q_len_s[s] = q_len[i]; w.past_s[s] = past_len[i]; w.cache_s[s] = cache_seq[i]; w.tok0_s[s] = tok0[i];
        ctas += (long long)kv_heads * row_tiles_of(q_len[i], n_rep);
    }
    w.cta0[n] = (int)ctas;
    return ctas;
}

// grid of a description: (x, y)
PA_HD long long grid_x(const Work& w) { return w.n_seq ? w.cta0[w.n_seq] : (long long)w.kv_heads * w.bsz; }
PA_HD int grid_y(const Work& w) { return w.n_seq ? 1 : w.row_tiles; }

// the tile of CTA (bx, by)
PA_HD Tile tile_of(const Work& w, int bx, int by)
{
    Tile t;
    if (w.n_seq == 0) {
        const int b = bx / w.kv_heads;
        t.cache_seq = b; t.tok0 = b * w.q_len; t.q_len = w.q_len; t.past_len = w.past_len;
        t.g = bx - b * w.kv_heads;
        t.m0 = (w.row_tiles - 1 - by) * BM;
        return t;
    }
    int s = 0;
    while (s + 1 < w.n_seq && bx >= w.cta0[s + 1]) s++;
    const int local = bx - w.cta0[s], rt = local / w.kv_heads;
    t.cache_seq = w.cache_s[s]; t.tok0 = w.tok0_s[s]; t.q_len = w.q_len_s[s]; t.past_len = w.past_s[s];
    t.g = local - rt * w.kv_heads;
    t.m0 = (row_tiles_of(t.q_len, w.n_rep) - 1 - rt) * BM;
    return t;
}

} // namespace pa_sched
