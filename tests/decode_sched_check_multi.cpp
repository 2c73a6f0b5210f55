// decode_sched_check_multi.cpp -- the proof obligations of tests/decode_sched_check_batch.cpp for multi-token steps: k consecutive
// tokens of ONE sequence per launch, on a plan made for max_tokens of them (exl_decode_plan_create_multi).
//
// Compiled by tests/test_multi_schedule.py with g++.  It includes decode_sched_check_batch.cpp (and through it the GQA and multi-head
// checkers), so the test can hold the multi-token GEMV and head schedules against the batch's at nb = k.  What changes:
//   P1   ATT units are (real KV head, 16-position chunk) at the shared context past_len: kv_heads * max(1, ceil(past_len / 16)),
//        taken by at most ATT_CTAS_PER_KV_HEAD CTAs per KV head (phase_of_multi)
//   P3   a CTA touches at most 2 KV heads
//   P4   exactly one CTA owns each KV head's last chunk (it writes the k new rows and the causal tail); the slot table over the k * heads
//        virtual query heads (token t, head h at t * heads + h, each with the CTA range of its real KV head): unique slots, read by
//        the combine only where written unless att_needs_reset_multi(past_len) holds, and the predicate is exact (a gap exists
//        exactly where it holds)
//   P5   the GEMV and HEAD phases are the batch's at nb = k; every CTA's K stages fit the compacted per-token staging
//   P7   >= 2 ring stages fit with max_tokens residual streams, compacted staging and the n_rep * max_tokens query vectors of the
//        attention scratch; k * heads <= DS_MAX_HEADS
#include "decode_sched_check_batch.cpp"

// returns 0 when every property holds for every past_len in [past_lo, past_hi] with past_len + k <= max_seq; else 1 with a message
extern "C" int ds_check_multi(int H, int HQ, int I, int heads, int kv_heads, int vocab, int grid, int k, int max_tokens, int past_lo,
                              int past_hi, int max_seq, long long dev_smem, char* msg, int msg_len, long long* n_gaps, int* n_resets)
{
    long long gaps = 0; int resets = 0;
    g_msg = msg; g_len = msg_len;
    if (msg && msg_len > 0) msg[0] = 0;
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads) return fail("shape: kv_heads (%lld) must divide heads (%lld)", kv_heads, heads);
    if (max_tokens < 1 || max_tokens > MAX_BATCH || k < 1 || k > max_tokens) return fail("tokens: k %lld, max_tokens %lld", k, max_tokens);
    const int n_rep = heads / kv_heads;
    BDims a; memset(&a, 0, sizeof a);
    a.H = H; a.HQ = HQ; a.HKV = kv_heads * TILE; a.I = I; a.heads = heads; a.kv_heads = kv_heads; a.vocab = vocab;
    a.lm_head = vocab ? (const void*)&a : nullptr;

    // ---- P7 ----
    const int xst = batch_xstages(H, HQ, a.HKV, I, grid);
    const size_t fixed = smem_fixed_bytes_multi(H, n_rep, max_tokens, xst);
    const int depth = ring_depth_for((size_t)dev_smem, fixed);
    if (depth < 2) return fail("P7: only %lld ring stages per pipeline fit (fixed part %lld B of %lld B)", depth, (long long)fixed, dev_smem);
    if (smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE > (size_t)dev_smem) return fail("P7: plan of %lld B exceeds %lld B", (long long)(smem_dynamic_bytes(fixed, depth) + SMEM_STATIC_ALLOWANCE), dev_smem);
    // the kernel lays out the staging area for the k tokens of the launch: it must hold the scratch and sit inside the plan's area
    if (stage_area_bytes_multi(k * xst, n_rep, k) > stage_area_bytes_multi(max_tokens * xst, n_rep, max_tokens)) return fail("P7: staging area of %lld tokens exceeds the plan's", k);
    if (gqa_scratch_bytes_multi(n_rep, k) > stage_area_bytes_multi(k * xst, n_rep, k)) return fail("P7: attention scratch exceeds the staging area");
    if ((size_t)H * 2 > (size_t)xst * 256) return fail("P7: normalised x of the head (%lld B) does not fit a token's staging area", (long long)H * 2);
    if (H % 512 || HQ % TILE || I % TILE || HQ != heads * TILE) return fail("shape: widths must be multiples of 128 (hidden of 512), HQ == heads * 128");
    if (heads > grid || kv_heads > grid) return fail("shape: more heads (%lld) than CTAs (%lld)", heads, grid);
    if (max_tokens * heads > DS_MAX_HEADS) return fail("P4: %lld virtual query heads exceed the CTA-range table (%lld)", max_tokens * heads, DS_MAX_HEADS);

    // ---- P5: GEMV and HEAD phases are the batch's at nb = k ----
    const int kinds[5] = {PH_QKV, PH_O, PH_GU, PH_DOWN, PH_HEAD};
    for (int i = 0; i < 5; i++) {
        const Phase p = phase_of_multi(a, kinds[i], grid), q = phase_of(a, kinds[i], grid, k);
        if (p.U != q.U || p.G != q.G || p.spt != q.spt || p.tpm != q.tpm || p.tq != q.tq || p.nmat != q.nmat || p.mat0 != q.mat0 || p.N != q.N)
            return fail("P5: phase %lld differs from the batch's at nb = %lld", kinds[i], k);
        if (p.U > 0 && check_partition(p, grid, "GEMV/HEAD")) return 1;
        if (kinds[i] == PH_HEAD) continue;
        for (int c = 0; c < grid; c++) {
            const int lo = range_lo(p.U, c, p.G), hi = range_lo(p.U, c + 1, p.G);
            if ((hi - lo < p.spt ? hi - lo : p.spt) > xst) return fail("P5: phase %lld CTA %lld quantises more K stages than a token's staging holds", kinds[i], c);
        }
    }

    // ---- P1..P4 for ATT over the real KV heads at every context ----
    const int slots = att_slots_multi(grid, kv_heads);
    const int vheads = k * heads;
    std::vector<int> written((size_t)vheads * slots), owners((size_t)kv_heads);
    for (int past = past_lo; past <= past_hi && past + k <= max_seq; past++) {
        a.past_len = past;
        const Phase p = phase_of_multi(a, PH_ATT, grid);
        const int nph = p.tpm;
        if (nph != ((past + 15) / 16 > 0 ? (past + 15) / 16 : 1) || p.U != kv_heads * nph) return fail("ATT ctx %lld: units %lld", past, p.U);
        if (p.G > kv_heads * ATT_CTAS_PER_KV_HEAD) return fail("ATT ctx %lld: %lld CTAs over %lld KV heads exceed the cap", past, p.G, kv_heads);
        if (check_partition(p, grid, "ATT")) { if (msg) { size_t n = strlen(msg); snprintf(msg + n, (size_t)msg_len - n, " (ctx %d)", past); } return 1; }
        std::fill(written.begin(), written.end(), -1);
        std::fill(owners.begin(), owners.end(), 0);
        for (int c = 0; c < grid; c++) {
            const int u0 = range_lo(p.U, c, p.G), u1 = range_lo(p.U, c + 1, p.G);
            if (u1 <= u0) continue;
            const int h0 = u0 / nph, h1 = (u1 - 1) / nph;
            if (h1 - h0 + 1 > 2) return fail("P3: ctx %lld CTA %lld touches %lld KV heads", past, c, h1 - h0 + 1);
            for (int kvh = h0; kvh <= h1; kvh++) {
                const int end = (kvh + 1) * nph;
                if ((u1 < end ? u1 : end) == end) owners[(size_t)kvh]++;      // the kernel's owner(kvh)
                for (int t = 0; t < k; t++)
                    for (int r = 0; r < n_rep; r++) {
                        const int h = t * heads + kvh * n_rep + r;           // the kernel's hv
                        const int slot = c - cta_of((long long)kvh * nph, p.U, p.G);
                        if (slot < 0 || slot >= slots) return fail("P4: ctx %lld CTA %lld head %lld: slot %lld outside the table", past, c, h, slot);
                        if (written[(size_t)h * slots + slot] >= 0) return fail("P4: ctx %lld head %lld slot %lld written twice (second writer CTA %lld)", past, h, slot, c);
                        written[(size_t)h * slots + slot] = c;
                    }
            }
        }
        for (int kvh = 0; kvh < kv_heads; kvh++)
            if (owners[(size_t)kvh] != 1) return fail("P4: ctx %lld KV head %lld has %lld tail owners", past, kvh, owners[(size_t)kvh]);
        const bool reset = att_needs_reset_multi(heads, kv_heads, past, grid);
        bool gap = false;
        for (int h = 0; h < vheads; h++) {
            const int kvh = (h % heads) / n_rep;                            // the kernel's table builder
            const int c_lo = cta_of((long long)kvh * nph, p.U, p.G), c_hi = cta_of((long long)(kvh + 1) * nph - 1, p.U, p.G);
            const int ns = c_hi - c_lo + 1;
            if (ns < 1 || ns > slots) return fail("P4: ctx %lld head %lld: %lld partials, table has %lld slots", past, h, ns, slots);
            for (int s = 0; s < slots; s++) {
                const bool w = written[(size_t)h * slots + s] >= 0;
                if (w && s >= ns) return fail("P4: ctx %lld head %lld slot %lld is written but the combine reads only the first %lld", past, h, s, ns);
                if (!w && s < ns) {
                    gaps++; gap = true;
                    if (!reset) return fail("P4: ctx %lld head %lld slot %lld is read but not written, and the host does not reset the table", past, h, s);
                }
            }
        }
        if (reset != gap) return fail("P4: ctx %lld: reset predicate %lld but gap %lld", past, reset, gap);
        if (reset) resets++;
    }
    if (n_gaps) *n_gaps = gaps;
    if (n_resets) *n_resets = resets;
    return 0;
}

extern "C" int ds_plan_multi(int H, int HQ, int I, int heads, int kv_heads, int grid, int max_tokens, long long dev_smem, int* depth,
                             long long* smem, int* att_slots)
{
    if (kv_heads < 1 || kv_heads > heads || heads % kv_heads || max_tokens < 1 || max_tokens > MAX_BATCH) return 1;
    const size_t fixed = smem_fixed_bytes_multi(H, heads / kv_heads, max_tokens, batch_xstages(H, HQ, kv_heads * TILE, I, grid));
    *depth = ring_depth_for((size_t)dev_smem, fixed);
    *smem = (long long)smem_dynamic_bytes(fixed, *depth);
    *att_slots = att_slots_multi(grid, kv_heads);
    return 0;
}

extern "C" int ds_max_tokens(int H, int HQ, int I, int heads, int kv_heads, long long dev_smem, int grid)
{
    return max_tokens_for(H, HQ, I, heads, kv_heads, (size_t)dev_smem, grid);
}

extern "C" int ds_att_needs_reset_multi(int heads, int kv_heads, int past_len, int grid)
{
    return att_needs_reset_multi(heads, kv_heads, past_len, grid) ? 1 : 0;
}
