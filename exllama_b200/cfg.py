"""Classifier-free guidance on the device (DESIGN.md §4h): the reference's example_cfg.py, where each token comes from two prompts --
the prompt and a guidance prompt, stepped together with the same generated tokens -- whose penalised log-probabilities are mixed
as (1 - alpha) * l_prompt + alpha * l_guidance before the sampler (csrc/cfg.cu, include/exl_b200.h exl_cfg_mix).

    cfg.mix(logits, [(0, 1)], [1.5], [settings], history=hist, hist_lens=[L0 + j, L1 + j])   # in place; then sampling.sample(...)
    texts = cfg.generate_cfg(stack, embed, [(prompt, cfg_prompt)], alpha=1.5, eos_token_id=2)

Differences from the reference, which left-pads both prompts to one length in a batch-2 cache:
- prompts are not padded: each starts at cache position 0 of its own cache sequence (in the reference the pads shift the shorter
  prompt's positions and enter its penalty history);
- the stop token is kept, where the example breaks before appending it;
- the logits are the step's fp32 values.
"""
from __future__ import annotations

import torch

from . import capi, sampling


def mix(logits, pairs, alphas, settings, history=None, hist_lens=None):
    """exl_cfg_mix in place on logits [rows, vocab] fp32 (CUDA, unit stride along vocab): for pair k = (a, b), rows a and b are
    penalised over their own history with settings[k]'s penalty triple, log-softmaxed, and both become
    (1 - alphas[k]) * l_a + alphas[k] * l_b.  Rows in no pair are not touched.

    pairs     list of (a, b) row pairs, 1 .. 32 of them, no row in two pairs
    alphas    one float per pair
    settings  one sampling.Settings per pair (or one for every pair): only the repetition-penalty fields are used
    history   int64 [rows, hist_ld] token ids on the logits' device, newest last, or None (no penalty)
    hist_lens the tokens of each history row to use (host ints, default hist_ld each)

    Then sampling.sample of a mixed row with no history (and the request's bos id and banned list) draws the guided token.
    Returns logits."""
    rows, vocab = sampling.check_rows("cfg.mix", logits)
    pairs = [(int(a), int(b)) for a, b in pairs]
    n = len(pairs)
    alphas = [float(x) for x in alphas]
    settings = list(settings) if isinstance(settings, (list, tuple)) else [settings] * n
    if len(alphas) != n or len(settings) != n:
        raise ValueError(f"cfg.mix: {n} pairs, {len(alphas)} alphas and {len(settings)} settings")
    history, hist_ld, lens = sampling.history_args("cfg.mix", history, hist_lens, rows, logits.device)
    arr = (capi.ExlCfgPair * max(n, 1))()
    for k, ((a, b), alpha, s) in enumerate(zip(pairs, alphas, settings)):
        arr[k] = capi.ExlCfgPair(a, b, alpha, s.token_repetition_penalty_max, s.token_repetition_penalty_sustain,
                                 s.token_repetition_penalty_decay)
    with torch.cuda.device(logits.device):
        capi.check(capi.lib().exl_cfg_mix(capi._ptr(logits), rows, vocab, sampling.row_ld(logits), capi._ptr(history), hist_ld, lens,
                                          arr, n, capi._stream()))
    return logits


def generate_cfg(stack, embed, prompt_pairs, alpha, max_new_tokens=128, settings=None, eos_token_id=None, seed=0, banned=None):
    """example_cfg.generate_cfg over a list of (prompt, cfg_prompt) pairs (lists of ids): one guided request per pair through
    generate.BatchGenerator, with settings used as given (sample_current keeps min_p), no bos mask, eos_token_id as the stop id,
    seed seed + i for pair i, and max_new_tokens clipped to what the longer prompt leaves in max_seq.  Returns each first prompt
    followed by its tokens (host lists of ids)."""
    from . import generate                  # generate imports this module for mix
    s = settings if settings is not None else sampling.Settings()
    return generate.run_prompts(stack, embed, [generate.Request(p, 1, s, stop_ids=() if eos_token_id is None else (eos_token_id,),
                                                                seed=seed + i, banned=banned, cfg_prompt=q, cfg_alpha=alpha)
                                               for i, (p, q) in enumerate(prompt_pairs)], max_new_tokens)
