// decode_sched_check_gqa.cpp -- the proof obligations of tests/decode_sched_check.cpp for grouped-query attention (kv_heads < heads).
//
// Compiled by tests/test_gqa_schedule.py with g++.  It includes decode_sched_check.cpp -- the multi-head checker, ds_check / ds_plan,
// and its partition helpers -- so one library exports both and the test can compare them for kv_heads == heads.  What changes:
//   QKV  q's tiles, then k's and v's (kv_heads * 128 wide), accumulator columns [HQ | HKV | HKV]; every tile maps back to its matrix
//   P1   ATT units are (KV head, 16-position chunk): kv_heads * max(1, ceil(ctx / 16)) per layer
//   P3   a CTA touches at most 2 KV heads
//   P4   for every QUERY head: its CTA range is that of its KV head, each CTA of that range writes one slot, the combine reads only
//        written slots unless att_needs_reset() makes the host reset the table
//   P5   act-order: at most 2 matrices per CTA range, with the matrix boundaries of unequal widths
//   P7   the shared-memory plan includes the GQA attention scratch on the x staging area
#include "decode_sched_check.cpp"

namespace {

struct GDims
{
    int H, HQ, HKV, I, heads, kv_heads, past_len, vocab;
    const void* lm_head;
    float *acc_qkv, *acc_o, *acc_gu, *acc_d;
};

} // namespace

// returns 0 when every property holds for every past_len in [past_lo, past_hi]; else 1 with a message
extern "C" int ds_check_gqa(int H, int HQ, int I, int heads, int kv_heads, int vocab, int grid, int past_lo, int past_hi, int act,
                            long long dev_smem, char* msg, int msg_len, long long* n_gaps, int* n_resets)
{
    long long gaps = 0; int resets = 0;
    g_msg = msg; g_len = msg_len;
    if (msg && msg_len > 0) msg[0] = 0;
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads) return fail("shape: kv_heads (%lld) must divide heads (%lld)", kv_heads, heads);
    const int n_rep = heads / kv_heads;
    GDims a; memset(&a, 0, sizeof a);
    a.H = H; a.HQ = HQ; a.HKV = kv_heads * TILE; a.I = I; a.heads = heads; a.kv_heads = kv_heads; a.vocab = vocab;
    a.lm_head = vocab ? (const void*)&a : nullptr;

    // ---- P7 ----
    const size_t fixed = smem_fixed_bytes(H, HQ, I, act != 0, n_rep);
    const int depth = ring_depth_for((size_t)dev_smem, fixed);
    if (depth < 2) return fail("P7: only %lld ring stages per pipeline fit (fixed part %lld B of %lld B)", depth, (long long)fixed, dev_smem);
    if (smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE > (size_t)dev_smem) return fail("P7: plan of %lld B exceeds %lld B", (long long)(smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE), dev_smem);
    if ((size_t)H * 2 > (size_t)spt_max_for(H, HQ, I) * 256) return fail("P7: normalised x of the head (%lld B) does not fit the staging area", (long long)H * 2);
    if (H % 512 || HQ % TILE || I % TILE || HQ != heads * TILE) return fail("shape: widths must be multiples of 128 (hidden of 512), HQ == heads * 128");
    if (heads > grid) return fail("shape: more heads (%lld) than CTAs (%lld)", heads, grid);

    // ---- P1, P2, P5 for the phases that do not depend on the context length ----
    const int kinds[4] = {PH_QKV, PH_O, PH_GU, PH_DOWN};
    const char* names[4] = {"QKV", "O", "GU", "DOWN"};
    for (int k = 0; k < 4; k++) {
        const Phase p = phase_of(a, kinds[k], grid);
        // accumulator columns: QKV [HQ | HKV | HKV], every other phase nmat x N
        const long long cols = kinds[k] == PH_QKV ? (long long)HQ + 2LL * a.HKV : (long long)p.nmat * p.N;
        if (p.U != (p.tq + (p.nmat - 1) * p.tpm) * p.spt || p.U <= 0 || (long long)(p.tq + (p.nmat - 1) * p.tpm) * TILE != cols)
            return fail("phase %lld: unit count %lld", kinds[k], p.U);
        if (check_partition(p, grid, names[k])) return 1;
        if (p.spt > spt_max_for(H, HQ, I)) return fail("phase %lld: %lld K stages exceed the staging area", kinds[k], p.spt);
        for (int t = 0; t * p.spt < p.U; t++) {
            const int mi = mat_of_tile(p, t);
            if (mi < 0 || mi >= p.nmat || t < mat_tile0(p, mi) || t >= mat_tile0(p, mi) + mat_tiles(p, mi))
                return fail("phase %lld: tile %lld maps to matrix %lld", kinds[k], t, mi);
        }
        if (act) {
            for (int c = 0; c < grid; c++) {
                const int lo = range_lo(p.U, c, p.G), hi = range_lo(p.U, c + 1, p.G);
                if (hi <= lo) continue;
                const int m0 = mat_of_tile(p, lo / p.spt), m1 = mat_of_tile(p, (hi - 1) / p.spt);
                if (m1 - m0 > 1) return fail("P5: phase %lld CTA %lld touches %lld matrices", kinds[k], c, m1 - m0 + 1);
                // the second staging slot holds H / 128 stages: only phases whose K is H may need it
                if (m1 != m0 && p.spt != H / TILE) return fail("P5: phase %lld needs a second slot but K != hidden", kinds[k]);
            }
        }
    }
    // ---- P6 ----
    {
        const Phase p = phase_of(a, PH_HEAD, grid);
        if (vocab) {
            if (check_partition(p, grid, "HEAD")) return 1;
            const long long bytes = (long long)vocab * H * 2;
            if ((long long)p.U * W_BYTES < bytes || (long long)(p.U - 1) * W_BYTES >= bytes) return fail("P6: %lld stages for %lld bytes of lm_head", p.U, bytes);
            if (bytes % 1024) return fail("P6: lm_head is not a whole number of 1 KB chunks");
        } else if (p.U != 0) return fail("P6: no head but %lld units", p.U);
    }
    // ---- P1..P4 for ATT at every context length ----
    const int slots = att_slots_for(grid, heads, kv_heads);
    std::vector<int> written((size_t)heads * slots);
    for (int past = past_lo; past <= past_hi; past++) {
        a.past_len = past;
        const Phase p = phase_of(a, PH_ATT, grid);
        const int nph = p.tpm;
        if (nph != ((past + 15) / 16 > 0 ? (past + 15) / 16 : 1) || p.U != kv_heads * nph) return fail("ATT past %lld: units %lld", past, p.U);
        if (check_partition(p, grid, "ATT")) { if (msg) { size_t n = strlen(msg); snprintf(msg + n, (size_t)msg_len - n, " (past %d)", past); } return 1; }
        std::fill(written.begin(), written.end(), -1);
        for (int c = 0; c < grid; c++) {
            const int u0 = range_lo(p.U, c, p.G), u1 = range_lo(p.U, c + 1, p.G);
            if (u1 <= u0) continue;
            const int h0 = u0 / nph, h1 = (u1 - 1) / nph;                  // KV heads
            if (h1 - h0 + 1 > 2) return fail("P3: past %lld CTA %lld touches %lld heads", past, c, h1 - h0 + 1);
            for (int kvh = h0; kvh <= h1; kvh++)
                for (int h = kvh * n_rep; h < (kvh + 1) * n_rep; h++) {     // the kernel writes a partial for every query head of the group
                    const int slot = c - cta_of((long long)kvh * nph, p.U, p.G);
                    if (slot < 0 || slot >= slots) return fail("P4: past %lld CTA %lld head %lld: slot %lld outside the table", past, c, h, slot);
                    if (written[(size_t)h * slots + slot] >= 0) return fail("P4: past %lld head %lld slot %lld written twice (second writer CTA %lld)", past, h, slot, c);
                    written[(size_t)h * slots + slot] = c;
                }
        }
        for (int h = 0; h < heads; h++) {
            // what combine8 (O prologue) reads: the CTA range of the query head's KV head (s_clo / s_chi)
            const int kvh = h / n_rep;
            const int c_lo = cta_of((long long)kvh * nph, p.U, p.G), c_hi = cta_of((long long)(kvh + 1) * nph - 1, p.U, p.G);
            const int ns = c_hi - c_lo + 1;
            if (ns < 1 || ns > slots) return fail("P4: past %lld head %lld: %lld partials, table has %lld slots", past, h, ns, slots);
            for (int s = 0; s < slots; s++) {
                const bool w = written[(size_t)h * slots + s] >= 0;
                if (w && s >= ns) return fail("P4: past %lld head %lld slot %lld is written but the combine reads only the first %lld", past, h, s, ns);
                if (!w && s < ns) {
                    // a CTA between the head's first and last CTA owns no unit: the combine reads a slot nobody wrote in THIS launch.
                    // Allowed only where the host resets the table before the launch (att_needs_reset).
                    gaps++;
                    if (!att_needs_reset(heads, kv_heads, past, grid)) return fail("P4: past %lld head %lld slot %lld is read but not written, and the host does not reset the table", past, h, s);
                }
            }
        }
        if (att_needs_reset(heads, kv_heads, past, grid)) resets++;
        if (att_needs_reset(heads, kv_heads, past, grid) && p.U >= p.G) return fail("P4: past %lld: reset requested although every CTA has work", past);
    }
    if (n_gaps) *n_gaps = gaps;
    if (n_resets) *n_resets = resets;
    return 0;
}

extern "C" int ds_plan_gqa(int H, int HQ, int I, int heads, int kv_heads, int grid, int act, long long dev_smem, int* depth, long long* smem, int* att_slots)
{
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads) return 1;
    const size_t fixed = smem_fixed_bytes(H, HQ, I, act != 0, heads / kv_heads);
    *depth = ring_depth_for((size_t)dev_smem, fixed);
    *smem = (long long)smem_dynamic_bytes(fixed, *depth);
    *att_slots = att_slots_for(grid, heads, kv_heads);
    return 0;
}
