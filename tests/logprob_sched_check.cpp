// CPU proof of the token_logprob_kernel work list (exllama_b200/csrc/logprob_sched.h), compiled with g++ by
// tests/test_logprob_oracle.py.  For one (T, V, num_sms): every (row tile, vocab tile) is computed by exactly one CTA; a CTA's chunk
// is a non-empty run of vocab tiles; every partial slot of a row below T is written exactly once, inside the work size; and the
// combine, which reads slot(t, c) for c = 0 .. chunks - 1, reads exactly the slots written.
#include "../exllama_b200/csrc/logprob_sched.h"

#include <cstdio>
#include <vector>

extern "C" int lp_check(int T, int V, int num_sms, long long* work_bytes_out, char* msg, int msg_len)
{
    using namespace lp_sched;
    const Plan p = make_plan(T, V, num_sms);
    *work_bytes_out = work_bytes(p);
    if (p.row_tiles != (T + BM - 1) / BM || p.vocab_tiles != (V + BN - 1) / BN)
        return snprintf(msg, msg_len, "tile counts %d x %d", p.row_tiles, p.vocab_tiles), 1;
    if (p.chunks < 1 || p.chunks > p.vocab_tiles) return snprintf(msg, msg_len, "chunks %d of %d tiles", p.chunks, p.vocab_tiles), 1;
    if (chunk_begin(p, 0) != 0 || chunk_begin(p, p.chunks) != p.vocab_tiles) return snprintf(msg, msg_len, "chunk ends"), 1;
    if (p.row_tiles <= num_sms && ctas(p) > num_sms) return snprintf(msg, msg_len, "%lld CTAs for %d SMs", ctas(p), num_sms), 1;
    std::vector<int> tile_hits((size_t)p.row_tiles * p.vocab_tiles, 0);
    std::vector<int> slot_writes((size_t)T * p.chunks, 0);
    for (long long cta = 0; cta < ctas(p); cta++) {
        const int rt = row_tile_of(p, cta), ch = chunk_of(p, cta);
        if (rt < 0 || rt >= p.row_tiles || ch < 0 || ch >= p.chunks) return snprintf(msg, msg_len, "CTA %lld -> (%d, %d)", cta, rt, ch), 1;
        if (cta > 0 && chunk_of(p, cta - 1) > ch) return snprintf(msg, msg_len, "CTA %lld: chunks out of order", cta), 1;
        const int v0 = chunk_begin(p, ch), v1 = chunk_begin(p, ch + 1);
        if (v1 <= v0) return snprintf(msg, msg_len, "chunk %d empty", ch), 1;
        for (int vt = v0; vt < v1; vt++) tile_hits[(size_t)rt * p.vocab_tiles + vt]++;
        for (int r = rt * BM; r < rt * BM + BM && r < T; r++) {
            const long long s = slot(p, r, ch);
            if (s < 0 || (s + 1) * PART_BYTES > work_bytes(p)) return snprintf(msg, msg_len, "slot %lld outside the work", s), 1;
            slot_writes[(size_t)s]++;
        }
    }
    for (size_t i = 0; i < tile_hits.size(); i++)
        if (tile_hits[i] != 1) return snprintf(msg, msg_len, "tile (%zu, %zu) computed %d times", i / p.vocab_tiles, i % p.vocab_tiles, tile_hits[i]), 1;
    std::vector<int> slot_reads((size_t)T * p.chunks, 0);
    for (int t = 0; t < T; t++)
        for (int c = 0; c < p.chunks; c++) slot_reads[(size_t)slot(p, t, c)]++;
    for (size_t i = 0; i < slot_writes.size(); i++) {
        if (slot_writes[i] != 1) return snprintf(msg, msg_len, "slot %zu written %d times", i, slot_writes[i]), 1;
        if (slot_reads[i] != 1) return snprintf(msg, msg_len, "slot %zu read %d times", i, slot_reads[i]), 1;
    }
    if (work_bytes(p) != (long long)slot_writes.size() * PART_BYTES) return snprintf(msg, msg_len, "work %lld bytes", work_bytes(p)), 1;
    return 0;
}
