// logprob_sched.h -- the work list of token_logprob_kernel (logprob.cu): which (row tile, vocab chunk) a CTA computes, which vocab
// tiles a chunk holds, where its per-row partial goes, and how large the caller's work buffer must be.
//
// Plain C++ with no CUDA types: the kernel includes it as device code, and tests/test_logprob_oracle.py compiles the same header with
// g++ (tests/logprob_sched_check.cpp) to check on the CPU that every (row tile, vocab tile) is computed exactly once, that every
// partial slot is written once and read by the combine, and that the work size covers every slot.
//
// The logits [T, V] are cut into row tiles of BM rows and vocab tiles of BN ids.  The vocab tiles are split into `chunks` contiguous
// chunks of near-equal length; a CTA owns one (row tile, chunk) and walks the chunk's vocab tiles in order, carrying each row's
// running (max, sum of exp, argmax, target logit).  CTA c = chunk * row_tiles + row tile: the CTAs of one chunk are consecutive, so
// every row tile of a vocab tile runs at the same time and each lm_head tile is read from HBM once and from L2 by the other row tiles.
// chunks = num_sms / row_tiles (at least 1, at most the vocab tiles): one CTA per SM, one wave, whenever row_tiles <= num_sms.
#pragma once

#if defined(__CUDACC__)
#define LP_HD __host__ __device__ __forceinline__
#else
#define LP_HD static inline
#endif

namespace lp_sched {

constexpr int BM = 128;                  // rows (tokens) per tile: two warpgroups of 64
constexpr int BN = 256;                  // vocab ids per tile: one wgmma m64n256 per warpgroup and k-step
constexpr int BK = 64;                   // hidden features per k-block (128 bytes of fp16: one SWIZZLE_128B row)
constexpr int PART_BYTES = 16;           // one partial: {max, sum of exp relative to max, argmax, target logit}

struct Plan { int T, V, row_tiles, vocab_tiles, chunks; };

LP_HD Plan make_plan(int T, int V, int num_sms)
{
    Plan p;
    p.T = T; p.V = V;
    p.row_tiles = (int)(((long long)T + BM - 1) / BM);
    p.vocab_tiles = (int)(((long long)V + BN - 1) / BN);
    int c = num_sms / p.row_tiles;
    if (c < 1) c = 1;
    if (c > p.vocab_tiles) c = p.vocab_tiles;
    p.chunks = c;
    return p;
}

LP_HD long long ctas(const Plan& p) { return (long long)p.row_tiles * p.chunks; }

// CTA cta's row tile and chunk
LP_HD int row_tile_of(const Plan& p, long long cta) { return (int)(cta % p.row_tiles); }
LP_HD int chunk_of(const Plan& p, long long cta) { return (int)(cta / p.row_tiles); }

// chunk c holds vocab tiles [chunk_begin(c), chunk_begin(c + 1)); chunk_begin(chunks) == vocab_tiles
LP_HD int chunk_begin(const Plan& p, int c) { return (int)((long long)c * p.vocab_tiles / p.chunks); }

// partial of row t (0 <= t < T) from chunk c: slot t * chunks + c of the work buffer (the combine reads a row's slots in chunk order)
LP_HD long long slot(const Plan& p, int t, int c) { return (long long)t * p.chunks + c; }

// bytes of the caller's work buffer: one partial per (row, chunk)
LP_HD long long work_bytes(const Plan& p) { return (long long)p.T * p.chunks * PART_BYTES; }

} // namespace lp_sched
