// decode_sched_check_batch.cpp -- the proof obligations of tests/decode_sched_check_gqa.cpp for batched decode: bsz sequences of one
// launch, each at its own context, on a plan made for max_batch of them.
//
// Compiled by tests/test_batch_schedule.py with g++.  It includes decode_sched_check_gqa.cpp (and through it the multi-head checker), so
// one library exports ds_check_gqa / ds_plan_gqa next to the batch entry points and the test can compare them at bsz 1.  What changes:
//   P1   the GEMV phases are those of one sequence; ATT units are (virtual KV head b * kv_heads + kvh, 16-position chunk), with the
//        chunk count of the LONGEST context: bsz * kv_heads * max(1, ceil(longest / 16)) per layer.  Shorter sequences own empty units
//        past their end, so the schedule depends on the longest context alone and proving it for every longest context covers every
//        mix of contexts
//   P3   a CTA touches at most 2 virtual KV heads
//   P4   the slot table of every virtual query head: unique slots, the combine reads only written ones unless att_needs_reset(longest)
//   P5   (batch) every CTA's K stages of every GEMV phase fit the compacted per-sequence staging (batch_xstages)
//   P7   >= 2 ring stages fit with max_batch residual streams and compacted staging; the head's normalised x fits a sequence's area;
//        max_batch * heads (kv_heads under GQA) <= grid and <= DS_MAX_HEADS
#include "decode_sched_check_gqa.cpp"

namespace {

struct BDims
{
    int H, HQ, HKV, I, heads, kv_heads, past_len, vocab;
    const void* lm_head;
    float *acc_qkv, *acc_o, *acc_gu, *acc_d;
};

} // namespace

// returns 0 when every property holds for every longest context in [past_lo, past_hi]; else 1 with a message
extern "C" int ds_check_batch(int H, int HQ, int I, int heads, int kv_heads, int vocab, int grid, int bsz, int max_batch, int past_lo,
                              int past_hi, long long dev_smem, char* msg, int msg_len, long long* n_gaps, int* n_resets)
{
    long long gaps = 0; int resets = 0;
    g_msg = msg; g_len = msg_len;
    if (msg && msg_len > 0) msg[0] = 0;
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads) return fail("shape: kv_heads (%lld) must divide heads (%lld)", kv_heads, heads);
    if (max_batch < 1 || max_batch > MAX_BATCH || bsz < 1 || bsz > max_batch) return fail("batch: bsz %lld, max_batch %lld", bsz, max_batch);
    const int n_rep = heads / kv_heads;
    BDims a; memset(&a, 0, sizeof a);
    a.H = H; a.HQ = HQ; a.HKV = kv_heads * TILE; a.I = I; a.heads = heads; a.kv_heads = kv_heads; a.vocab = vocab;
    a.lm_head = vocab ? (const void*)&a : nullptr;

    // ---- P7 ----
    const int xst = max_batch > 1 ? batch_xstages(H, HQ, a.HKV, I, grid) : 0;
    const size_t fixed = smem_fixed_bytes(H, HQ, I, false, n_rep, max_batch, xst);
    const int depth = ring_depth_for((size_t)dev_smem, fixed);
    if (depth < 2) return fail("P7: only %lld ring stages per pipeline fit (fixed part %lld B of %lld B)", depth, (long long)fixed, dev_smem);
    if (smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE > (size_t)dev_smem) return fail("P7: plan of %lld B exceeds %lld B", (long long)(smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE), dev_smem);
    const int head_stages = max_batch > 1 ? xst : spt_max_for(H, HQ, I);
    if ((size_t)H * 2 > (size_t)head_stages * 256) return fail("P7: normalised x of the head (%lld B) does not fit a sequence's staging area", (long long)H * 2);
    if (H % 512 || HQ % TILE || I % TILE || HQ != heads * TILE) return fail("shape: widths must be multiples of 128 (hidden of 512), HQ == heads * 128");
    if (heads > grid) return fail("shape: more heads (%lld) than CTAs (%lld)", heads, grid);
    if (max_batch * (n_rep > 1 ? kv_heads : heads) > grid) return fail("P3: %lld sequences x %lld (KV) heads exceed %lld CTAs", max_batch, n_rep > 1 ? kv_heads : heads, grid);
    if (max_batch * heads > DS_MAX_HEADS) return fail("P4: %lld virtual heads exceed the CTA-range table (%lld)", max_batch * heads, DS_MAX_HEADS);

    // ---- P1, P2, P5 for the GEMV phases (independent of the batch and of the context) ----
    const int kinds[4] = {PH_QKV, PH_O, PH_GU, PH_DOWN};
    const char* names[4] = {"QKV", "O", "GU", "DOWN"};
    for (int k = 0; k < 4; k++) {
        const Phase p = phase_of(a, kinds[k], grid, bsz), p1 = phase_of(a, kinds[k], grid);
        if (p.U != p1.U || p.G != p1.G || p.spt != p1.spt) return fail("phase %lld depends on the batch", kinds[k]);
        const long long cols = kinds[k] == PH_QKV ? (long long)HQ + 2LL * a.HKV : (long long)p.nmat * p.N;
        if (p.U != (p.tq + (p.nmat - 1) * p.tpm) * p.spt || p.U <= 0 || (long long)(p.tq + (p.nmat - 1) * p.tpm) * TILE != cols)
            return fail("phase %lld: unit count %lld", kinds[k], p.U);
        if (check_partition(p, grid, names[k])) return 1;
        for (int c = 0; c < grid; c++) {
            const int lo = range_lo(p.U, c, p.G), hi = range_lo(p.U, c + 1, p.G);
            const int n = hi - lo < p.spt ? hi - lo : p.spt;            // s_rng[.][3]: the K stages the CTA quantises per sequence
            const int room = max_batch > 1 ? xst : spt_max_for(H, HQ, I);
            if (n > room) return fail("P5: phase %lld CTA %lld quantises %lld K stages, the staging holds %lld per sequence", kinds[k], c, n, room);
            // compacted index of stage s = (s - s0) mod spt: distinct for the units of the range
            if (max_batch > 1 && hi > lo) {
                const int s0 = lo % p.spt;
                for (int u = lo; u < hi; u++) {
                    int sx = u % p.spt - s0; if (sx < 0) sx += p.spt;
                    if (sx >= n) return fail("P5: phase %lld CTA %lld unit %lld maps to staged stage %lld of %lld", kinds[k], c, u, sx, n);
                }
            }
        }
    }
    // ---- P6 ----
    {
        const Phase p = phase_of(a, PH_HEAD, grid, bsz);
        if (vocab) {
            if (check_partition(p, grid, "HEAD")) return 1;
            const long long bytes = (long long)vocab * H * 2;
            if ((long long)p.U * W_BYTES < bytes || (long long)(p.U - 1) * W_BYTES >= bytes) return fail("P6: %lld stages for %lld bytes of lm_head", p.U, bytes);
            if (bytes % 1024) return fail("P6: lm_head is not a whole number of 1 KB chunks");
        } else if (p.U != 0) return fail("P6: no head but %lld units", p.U);
    }
    // ---- P1..P4 for ATT over virtual heads at every longest context ----
    const int slots = att_slots_for(grid, heads, kv_heads);
    const int vheads = bsz * heads, vkv = bsz * kv_heads;
    std::vector<int> written((size_t)vheads * slots);
    for (int past = past_lo; past <= past_hi; past++) {
        a.past_len = past;
        const Phase p = phase_of(a, PH_ATT, grid, bsz);
        const int nph = p.tpm;
        if (nph != ((past + 15) / 16 > 0 ? (past + 15) / 16 : 1) || p.U != vkv * nph) return fail("ATT longest %lld: units %lld", past, p.U);
        if (check_partition(p, grid, "ATT")) { if (msg) { size_t n = strlen(msg); snprintf(msg + n, (size_t)msg_len - n, " (longest %d)", past); } return 1; }
        std::fill(written.begin(), written.end(), -1);
        for (int c = 0; c < grid; c++) {
            const int u0 = range_lo(p.U, c, p.G), u1 = range_lo(p.U, c + 1, p.G);
            if (u1 <= u0) continue;
            const int h0 = u0 / nph, h1 = (u1 - 1) / nph;                  // virtual KV heads
            if (h1 - h0 + 1 > 2) return fail("P3: longest %lld CTA %lld touches %lld virtual heads", past, c, h1 - h0 + 1);
            for (int kvh = h0; kvh <= h1; kvh++)
                for (int h = kvh * n_rep; h < (kvh + 1) * n_rep; h++) {     // virtual query heads b * heads + h' of the group
                    const int slot = c - cta_of((long long)kvh * nph, p.U, p.G);
                    if (slot < 0 || slot >= slots) return fail("P4: longest %lld CTA %lld head %lld: slot %lld outside the table", past, c, h, slot);
                    if (written[(size_t)h * slots + slot] >= 0) return fail("P4: longest %lld head %lld slot %lld written twice (second writer CTA %lld)", past, h, slot, c);
                    written[(size_t)h * slots + slot] = c;
                }
        }
        const bool reset = att_needs_reset(heads, kv_heads, past, grid, bsz);
        for (int h = 0; h < vheads; h++) {
            const int kvh = h / n_rep;                                      // == b * kv_heads + (h - b * heads) / n_rep
            const int c_lo = cta_of((long long)kvh * nph, p.U, p.G), c_hi = cta_of((long long)(kvh + 1) * nph - 1, p.U, p.G);
            const int ns = c_hi - c_lo + 1;
            if (ns < 1 || ns > slots) return fail("P4: longest %lld head %lld: %lld partials, table has %lld slots", past, h, ns, slots);
            for (int s = 0; s < slots; s++) {
                const bool w = written[(size_t)h * slots + s] >= 0;
                if (w && s >= ns) return fail("P4: longest %lld head %lld slot %lld is written but the combine reads only the first %lld", past, h, s, ns);
                if (!w && s < ns) {
                    gaps++;
                    if (!reset) return fail("P4: longest %lld head %lld slot %lld is read but not written, and the host does not reset the table", past, h, s);
                }
            }
        }
        if (reset) resets++;
        if (reset && p.U >= p.G) return fail("P4: longest %lld: reset requested although every CTA has work", past);
    }
    if (n_gaps) *n_gaps = gaps;
    if (n_resets) *n_resets = resets;
    return 0;
}

extern "C" int ds_plan_batch(int H, int HQ, int I, int heads, int kv_heads, int grid, int max_batch, long long dev_smem, int* depth,
                             long long* smem, int* att_slots, int* xstages)
{
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads || max_batch < 1 || max_batch > MAX_BATCH) return 1;
    const int xst = max_batch > 1 ? batch_xstages(H, HQ, kv_heads * TILE, I, grid) : 0;
    const size_t fixed = smem_fixed_bytes(H, HQ, I, false, heads / kv_heads, max_batch, xst);
    *depth = ring_depth_for((size_t)dev_smem, fixed);
    *smem = (long long)smem_dynamic_bytes(fixed, *depth);
    *att_slots = att_slots_for(grid, heads, kv_heads);
    *xstages = xst;
    return 0;
}

extern "C" int ds_max_batch(int H, int HQ, int I, int heads, int kv_heads, int act, long long dev_smem, int grid)
{
    return max_batch_for(H, HQ, I, heads, kv_heads, act != 0, (size_t)dev_smem, grid);
}
