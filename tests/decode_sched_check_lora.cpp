// decode_sched_check_lora.cpp -- the proof obligations of LoRA adapters in the persistent decode step (exl_decode_plan_create_lora).
//
// Compiled by tests/test_lora_schedule.py with g++.  It includes decode_sched_check_batch.cpp (and through it the GQA and multi-head
// checkers), so one library exports ds_plan_batch / ds_plan_gqa next to the LoRA entry points.  For one shape, grid, max_batch and
// adapter (a rank and the set of adapted projections, the same in every layer or on some layers only) it checks:
//   L1   LA step of every adapted phase: the units (adapted matrix, 128-row K stage) are partitioned over the grid -- every unit owned
//        by exactly one CTA, shares balanced to +-1 -- and cta_of inverts the shares
//   L2   every tile of every adapted matrix gets its B term from exactly one CTA: the one whose GEMV unit range holds the tile's K stage
//        0 (lora_b_cta); tiles of matrices without an adapter get none
//   L3   the LA scratch (x of a K stage and the partial t, per sequence) fits the attention partial area, and >= 2 ring stages fit: an
//        adapter adds no shared memory, so the plan is the one without it
//   L4   the barrier count: lora_barriers (what exl_decode_plan_info adds) is one per adapted phase of every layer, counted here
//        independently from the projections
//   L5   the adapter's rank is one the kernel takes
#include "decode_sched_check_batch.cpp"
#include "../include/exl_b200.h"
#include <cstddef>

extern "C" int ds_check_lora(int H, int HQ, int I, int heads, int kv_heads, int grid, int max_batch, int n_layers, const int* rank,
                             long long dev_smem, char* msg, int msg_len, long long* barriers)
{
    g_msg = msg; g_len = msg_len;
    if (msg && msg_len > 0) msg[0] = 0;
    BDims a; memset(&a, 0, sizeof a);
    a.H = H; a.HQ = HQ; a.HKV = kv_heads * TILE; a.I = I; a.heads = heads; a.kv_heads = kv_heads;
    const int kinds[4] = {PH_QKV, PH_O, PH_GU, PH_DOWN};
    const char* names[4] = {"LA QKV", "LA O", "LA GU", "LA DOWN"};
    long long expect_bar = 0;
    for (int l = 0; l < n_layers; l++) {
        for (int k = 0; k < 4; k++) {
            const Phase p = phase_of(a, kinds[k], grid, max_batch);
            const int* rk = rank + l * 7 + p.mat0;
            int na = 0;
            for (int m = 0; m < p.nmat; m++) {
                if (!lora_rank_ok(rk[m])) return fail("L5: layer %lld matrix %lld rank %lld", l, p.mat0 + m, rk[m]);
                if (rk[m] > 0) na++;
                if (lora_phase_of_mat(p.mat0 + m) != kinds[k]) return fail("L4: matrix %lld is not in phase %lld", p.mat0 + m, kinds[k]);
            }
            if (na == 0) continue;
            expect_bar++;
            // ---- L1 ----
            Phase la = p; la.U = lora_units(na, p.spt); la.G = grid;
            if (la.U != na * p.spt) return fail("L1: %lld units for %lld adapted matrices of %lld K stages", la.U, na, p.spt);
            if (check_partition(la, grid, names[k])) return 1;
            std::vector<int> owners((size_t)la.U, 0);
            for (int c = 0; c < grid; c++)
                for (int v = share_lo(la.U, c, grid); v < share_lo(la.U, c + 1, grid); v++) owners[(size_t)v]++;
            for (int v = 0; v < la.U; v++) if (owners[(size_t)v] != 1) return fail("L1: phase %lld unit %lld has %lld owners", kinds[k], v, owners[(size_t)v]);
            // ---- L2 ----
            const int tiles = p.tq + (p.nmat - 1) * p.tpm;
            std::vector<int> adds((size_t)tiles, 0);
            for (int c = 0; c < grid; c++) {
                const int u0 = range_lo(p.U, c, p.G), u1 = range_lo(p.U, c + 1, p.G);
                if (u1 <= u0) continue;
                for (int t = lora_b_first(p, u0); t * p.spt < u1; t++) {
                    if (t * p.spt < u0) return fail("L2: phase %lld CTA %lld: tile %lld starts before its range", kinds[k], c, t);
                    if (rk[mat_of_tile(p, t)] == 0) continue;
                    if (lora_b_cta(p, t) != c) return fail("L2: phase %lld tile %lld: B term by CTA %lld, lora_b_cta says %lld", kinds[k], t, c, lora_b_cta(p, t));
                    adds[(size_t)t]++;
                }
            }
            for (int t = 0; t < tiles; t++) {
                const int want = rk[mat_of_tile(p, t)] > 0 ? 1 : 0;
                if (adds[(size_t)t] != want) return fail("L2: phase %lld tile %lld gets its B term %lld times (want %lld)", kinds[k], t, adds[(size_t)t], want);
            }
            // ---- L3 (scratch) ----
            for (int m = 0; m < p.nmat; m++)
                if (lora_scratch_floats(max_batch, rk[m]) > LORA_SCRATCH_ROOM) return fail("L3: LA scratch of %lld floats exceeds %lld", lora_scratch_floats(max_batch, rk[m]), LORA_SCRATCH_ROOM);
        }
    }
    // ---- L3 (ring) ----
    const int xst = max_batch > 1 ? batch_xstages(H, HQ, a.HKV, I, grid) : 0;
    const int depth = ring_depth_for((size_t)dev_smem, smem_fixed_bytes(H, HQ, I, false, heads / kv_heads, max_batch, xst));
    if (depth < 2) return fail("L3: only %lld ring stages per pipeline fit", depth);
    // ---- L4 ----
    const long long nb = lora_barriers(rank, n_layers);
    if (nb != expect_bar) return fail("L4: lora_barriers says %lld extra barriers, the phases need %lld", nb, expect_bar);
    if (barriers) *barriers = nb;
    return 0;
}

// The plan of exl_decode_plan_create_lora: the batch plan (ds_plan_batch) and the extra barriers per step
extern "C" int ds_plan_lora(int H, int HQ, int I, int heads, int kv_heads, int grid, int max_batch, int n_layers, const int* rank,
                            long long dev_smem, int* depth, long long* smem, int* att_slots, int* xstages, long long* barriers)
{
    if (ds_plan_batch(H, HQ, I, heads, kv_heads, grid, max_batch, dev_smem, depth, smem, att_slots, xstages)) return 1;
    *barriers = lora_barriers(rank, n_layers);
    return 0;
}

// C layout of struct exl_decode_lora, for the ctypes mirror in exllama_b200/capi.py
extern "C" void ds_lora_layout(long long* out)
{
    out[0] = (long long)sizeof(exl_decode_lora);
    out[1] = (long long)offsetof(exl_decode_lora, n_layers); out[2] = (long long)offsetof(exl_decode_lora, a);
    out[3] = (long long)offsetof(exl_decode_lora, b); out[4] = (long long)offsetof(exl_decode_lora, rank);
}
