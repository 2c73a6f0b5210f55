"""CPU pin of the causal offset convention of prefill over an existing KV cache.

The oracle of a prefill chunk is oracle.decode_attn_f64 composed over its rows (token t at context past_len + t + 1).  Here it is
compared in float64 with the program the reference runs for a chunk at past_len > 0, restated with torch on the CPU: repeat_kv of
the cache rows [0, past_len + q_len), the additive mask [bsz, 1, q_len, past_len + q_len] that is 0 on and below the diagonal and
-65504 above it (row t masks columns past_len + t + 1 ..), and softmax(q k^T / sqrt(d) + mask) v."""
import numpy as np
import pytest

from prefill_oracle import prefill_attn_f64

HD = 128


def _masked_program(q, kc, vc, heads, kv_heads, past_len):
    """q [bsz, q_len, heads, hd], caches [bsz, kv_heads, max_seq, hd] (float64 torch) -> [bsz, q_len, heads, hd]."""
    import torch
    bsz, q_len = q.shape[:2]
    n = past_len + q_len
    rep = heads // kv_heads
    keys = kc[:, :, :n].repeat_interleave(rep, dim=1)                 # repeat_kv: query head h reads KV head h // rep
    values = vc[:, :, :n].repeat_interleave(rep, dim=1)
    mask = torch.zeros((bsz, 1, q_len, n), dtype=torch.float64)
    if q_len > 1:
        mask[:, :, :q_len - 1, past_len + 1:] = torch.triu(torch.full((q_len - 1, q_len - 1), -65504.0, dtype=torch.float64))
    qh = q.transpose(1, 2)
    w = qh @ keys.transpose(2, 3) / np.sqrt(HD) + mask
    w = torch.softmax(w, dim=-1)
    return (w @ values).transpose(1, 2)


@pytest.mark.parametrize("past_len,q_len,heads,kv_heads,bsz", [
    (0, 1, 8, 8, 1), (0, 9, 8, 2, 2), (1, 1, 4, 1, 1), (5, 1, 8, 2, 1), (37, 19, 8, 8, 1), (37, 6, 8, 4, 3), (200, 33, 4, 1, 1),
    (0, 40, 4, 4, 1), (63, 65, 2, 2, 2),
])
def test_composed_decode_oracle_matches_masked_program(oracle, past_len, q_len, heads, kv_heads, bsz):
    import torch
    max_seq = past_len + q_len + 7
    rng = np.random.default_rng(past_len * 131 + q_len * 7 + heads)
    q = (rng.standard_normal((bsz, q_len, heads, HD)) * 1.5).astype(np.float16)
    kc = (rng.standard_normal((bsz, kv_heads, max_seq, HD)) * 1.5).astype(np.float16)
    vc = rng.standard_normal((bsz, kv_heads, max_seq, HD)).astype(np.float16)
    kc[:, :, past_len + q_len:] = np.nan                               # rows past the chunk are never read
    vc[:, :, past_len + q_len:] = np.nan
    want = _masked_program(*(torch.from_numpy(a.astype(np.float64)) for a in (q, kc, vc)), heads, kv_heads, past_len).numpy()
    for b in range(bsz):
        got = prefill_attn_f64(oracle, q[b], kc[b], vc[b], heads, kv_heads, past_len, max_seq)
        assert np.isfinite(got).all()
        np.testing.assert_allclose(got, want[b], rtol=1e-9, atol=1e-9, err_msg=f"seq {b}")
