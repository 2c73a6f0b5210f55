// CPU check of prefill_attn_kernel's work list (exllama_b200/csrc/prefill_attn_sched.h), loaded by test_prefill_ragged_schedule.py.
// Each function returns 0, or 1 with the first violated property written to msg.
#include <cstdio>
#include <map>
#include <set>
#include <tuple>
#include <vector>

#include "../exllama_b200/csrc/prefill_attn_sched.h"

using namespace pa_sched;

namespace {

int fail(char* msg, int len, const char* what, long long a = 0, long long b = 0, long long c = 0)
{
    snprintf(msg, (size_t)len, "%s (%lld, %lld, %lld)", what, a, b, c);
    return 1;
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

using Key = std::tuple<int, int, int, int, int, int>;   // cache_seq, tok0, q_len, past_len, g, m0
Key key_of(const Tile& t) { return Key(t.cache_seq, t.tok0, t.q_len, t.past_len, t.g, t.m0); }

} // namespace

extern "C" {

// ragged description of n sequences (packed in the given order, distinct cache sequences): every (sequence, KV group, row tile)
// exactly once, no empty CTA, the CTA count sum_i kv_heads * ceil(q_len[i] * n_rep / 64), the sequences in non-increasing
// past_len + q_len order and, within a sequence, the row tiles from the last
int pr_check_ragged(int n, const int* q_len, const int* past, const int* cache, int kv_heads, int n_rep, char* msg, int len)
{
    Work w;
    const long long ctas = make_ragged(w, n, q_len, past, cache, kv_heads, n_rep);
    long long want = 0;
    std::map<int, int> seq_of_cache;
    std::vector<int> off(n);
    for (int i = 0, t = 0; i < n; t += q_len[i], i++) {
        want += kv_heads * ceil_div((long long)q_len[i] * n_rep, BM);
        seq_of_cache[cache[i]] = i;
        off[i] = t;
    }
    if (ctas != want || grid_x(w) != want || grid_y(w) != 1) return fail(msg, len, "CTA count", ctas, grid_x(w), want);
    std::set<std::tuple<int, int, int>> seen;
    long long prev_cost = -1;
    int prev_seq = -1, prev_m0 = -1;
    for (long long bx = 0; bx < ctas; bx++) {
        const Tile t = tile_of(w, (int)bx, 0);
        const auto it = seq_of_cache.find(t.cache_seq);
        if (it == seq_of_cache.end()) return fail(msg, len, "CTA names a cache sequence of no sequence", bx, t.cache_seq);
        const int i = it->second;
        if (t.tok0 != off[i] || t.q_len != q_len[i] || t.past_len != past[i])
            return fail(msg, len, "CTA's sequence fields differ from sequence", bx, i, t.tok0);
        if (t.g < 0 || t.g >= kv_heads) return fail(msg, len, "KV group out of range", bx, t.g);
        if (t.m0 < 0 || t.m0 % BM != 0) return fail(msg, len, "row tile start", bx, t.m0);
        if ((long long)t.m0 >= (long long)q_len[i] * n_rep) return fail(msg, len, "empty CTA", bx, i, t.m0);
        if (!seen.insert({i, t.g, t.m0 / BM}).second) return fail(msg, len, "tile computed twice", i, t.g, t.m0);
        const long long cost = (long long)past[i] + q_len[i];
        if (prev_cost >= 0 && cost > prev_cost) return fail(msg, len, "cost order increases at CTA", bx, cost, prev_cost);
        if (i == prev_seq && t.m0 > prev_m0) return fail(msg, len, "row tiles not from the last within a sequence", bx, t.m0, prev_m0);
        prev_cost = cost; prev_seq = i; prev_m0 = t.m0;
    }
    if ((long long)seen.size() != want) return fail(msg, len, "tiles covered", (long long)seen.size(), want);
    return 0;
}

// uniform description of bsz sequences: the grid and every CTA's tile are today's (kv_heads * bsz, row tiles) grid -- x = b * kv_heads
// + g, y counts row tiles from the last -- and, for bsz <= MAX_SEQ, a ragged description of the same batch (cache sequence b, token
// rows b * q_len) yields the same set of tiles
int pr_check_uniform(int bsz, int q_len, int past_len, int kv_heads, int n_rep, char* msg, int len)
{
    Work w;
    make_uniform(w, bsz, q_len, past_len, kv_heads, n_rep);
    const int rt = (int)ceil_div((long long)q_len * n_rep, BM);
    if (grid_x(w) != (long long)kv_heads * bsz || grid_y(w) != rt) return fail(msg, len, "uniform grid", grid_x(w), grid_y(w), rt);
    std::multiset<Key> uni;
    for (int by = 0; by < rt; by++)
        for (int bx = 0; bx < kv_heads * bsz; bx++) {
            const Tile t = tile_of(w, bx, by);
            const int b = bx / kv_heads;
            const Key today(b, b * q_len, q_len, past_len, bx % kv_heads, (rt - 1 - by) * BM);
            if (key_of(t) != today) return fail(msg, len, "uniform tile differs from today's grid", bx, by);
            uni.insert(today);
        }
    if (bsz > MAX_SEQ) return 0;
    std::vector<int> ql(bsz, q_len), pl(bsz, past_len), cs(bsz);
    for (int b = 0; b < bsz; b++) cs[b] = b;
    Work r;
    const long long ctas = make_ragged(r, bsz, ql.data(), pl.data(), cs.data(), kv_heads, n_rep);
    std::multiset<Key> rag;
    for (long long bx = 0; bx < ctas; bx++) rag.insert(key_of(tile_of(r, (int)bx, 0)));
    if (rag != uni) return fail(msg, len, "ragged description of a uniform batch differs", (long long)rag.size(), (long long)uni.size());
    return 0;
}

}
