"""Generates tests/golden/beam_ref.npz by running the REFERENCE's own ExLlamaGenerator.beam_search (generator.py:384-700) on the CPU.

    EXLLAMA_REFERENCE=<reference checkout> python -m oracle.gen_golden_beam

generator.py imports cuda_ext, model and lora; stub modules stand in for them, so nothing is built:
  - the model's forward returns beam_oracle.seq_logits of the generator's whole sequence (seeded, a function of the tokens only);
  - ExLlamaCache has clone, roll_left, copy_states and current_seq_len, and holds nothing;
  - cuda_ext.ext_apply_rep_penalty_mask_cpu is oracle.apply_rep_penalty (bit-exact with the reference's rep_penalty.cpp);
  - torch.multinomial draws with a seeded torch.Generator.
A subclass of the generator records the first expansion's draw (every draw when beams == beam_length == 1) and the beam windows
after every expansion.  beam_length 1 with beams > 1 is not stored: the reference's emission indexes past the end of its sequence
there (generator.py:668, the sequence is only extended by to_sequence of a later expansion).  The reference runs in float64 (the stub's logits are
fp32 values).  A case is kept only if beam_oracle.run with the recorded draws reproduces the reference's emitted tokens and beam
windows after every expansion, and every decision it takes has a margin of at least 1e-6.  The fixture stores seeds, settings, prompts, the recorded draws, the emitted tokens and the beam windows.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch

from . import beam_oracle as B
from . import oracle as O

MARGIN = 1e-6


class _Cfg:
    pass


def reference_generator():
    ref = os.environ.get("EXLLAMA_REFERENCE")
    if not ref or not os.path.exists(os.path.join(ref, "generator.py")):
        sys.exit("EXLLAMA_REFERENCE must name a checkout of the reference")

    class Cache:
        def __init__(self, model, batch_size=1, max_seq_len=-1, copy_from=None):
            self.model, self.current_seq_len = model, 0

        def clone(self):
            c = Cache(self.model)
            c.current_seq_len = self.current_seq_len
            return c

        def roll_left(self):
            pass

        def copy_states(self, target, from_column, from_columns, to_column, to_columns, from_row, from_rows, to_row, to_rows):
            pass

    class Model:
        def __init__(self, seed, vocab, max_seq):
            self.seed, self.config = seed, _Cfg()
            self.config.vocab_size, self.config.max_seq_len = vocab, max_seq
            self.gen = None

        def forward(self, input_ids, cache, last_id_only=True, preprocess_only=False, lora=None, output_device=None, input_mask=None):
            cache.current_seq_len += input_ids.shape[-1]
            if preprocess_only:
                return None
            seq = self.gen.sequence[0].tolist()
            lg = B.seq_logits(self.seed, self.config.vocab_size, seq)
            return torch.from_numpy(lg.astype(np.float64)).view(1, 1, -1)

    def apply_pen(sequence, pmax, sustain, decay, logits):
        x = logits.view(-1).numpy().astype(np.float32)
        y = O.apply_rep_penalty(sequence.view(1, -1).numpy().astype(np.int64), pmax, sustain, decay, x[None])[0]
        logits.view(-1)[:] = torch.from_numpy(y.astype(np.float64))

    for name, attrs in (("cuda_ext", {"ext_apply_rep_penalty_mask_cpu": apply_pen}),
                        ("model", {"ExLlama": object, "ExLlamaCache": Cache}), ("lora", {"ExLlamaLora": object})):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
    sys.path.insert(0, ref)
    import generator
    return generator.ExLlamaGenerator, Model, Cache


def recording(Gen):
    """A subclass of the reference's generator that records the tokens of the first sample(num=beams) call (every sample() call's
    when beams == beam_length == 1), and the beam windows after every expansion: the first expansion's from those tokens, a later
    one's from the list it assigns to self.beams (an emission's assignment follows calls of Beam.cum_log_probs and is skipped)."""
    real_cum = Gen.Beam.cum_log_probs

    def cum_log_probs(beam):
        beam.generator.emitting = True
        return real_cum(beam)
    Gen.Beam.cum_log_probs = cum_log_probs

    class Rec(Gen):
        @property
        def beams(self):
            return self._beams

        @beams.setter
        def beams(self, v):
            self._beams = v
            if not v:
                return
            if getattr(self, "emitting", False):
                self.emitting = False
            else:
                self.windows.append([b.sequence[0].tolist() for b in v])

        def sample(self, logits, temperature, top_k, top_p, min_p, typical, num=1):
            tokens, probs = super().sample(logits, temperature, top_k, top_p, min_p, typical, num)
            degenerate = self.settings.beams == 1 and self.settings.beam_length == 1
            if not self.draws or degenerate:
                self.draws.append(tokens.view(-1).tolist())
                if not degenerate:
                    self.windows.append([[t] for t in tokens.view(-1).tolist()[:self.settings.beams]])
            return tokens, probs
    return Rec


def run_reference(Gen, Model, Cache, c, n_emit):
    """The reference's beam_search for one case: (emitted tokens, recorded draws, beam windows after each expansion)."""
    model = Model(c["seed"], c["vocab"], c["max_seq"])
    tok = types.SimpleNamespace(bos_token_id=c["bos"])
    g = recording(Gen)(model, tok, Cache(model))
    g.windows, g.draws = [], []
    model.gen = g
    s = g.settings
    st = c["settings"]
    s.temperature, s.top_k, s.top_p, s.min_p, s.typical = st["temperature"], st["top_k"], st["top_p"], st["min_p"], st["typical"]
    s.token_repetition_penalty_max, s.token_repetition_penalty_sustain = st["penalty_max"], st["sustain"]
    s.token_repetition_penalty_decay = st["decay"]
    s.beams, s.beam_length = c["beams"], c["beam_length"]
    tg = torch.Generator()
    tg.manual_seed(c["seed"])
    real = torch.multinomial
    torch.multinomial = lambda probs, num, *a, **kw: real(probs, num, generator=tg)
    try:
        g.gen_begin(torch.tensor([c["prompt"]], dtype=torch.long))
        g.begin_beam_search()
        emitted = []
        for _ in range(n_emit):
            t = g.beam_search()
            emitted.append(int(t.view(-1)[0]))
    finally:
        torch.multinomial = real
    return emitted, g.draws, g.windows


def main():
    Gen, Model, Cache = reference_generator()
    rng = np.random.default_rng(2027)
    cases = []
    kinds = [
        dict(temperature=0.95, top_k=40, top_p=0.65, min_p=0.0, typical=0.0, penalty_max=1.15, sustain=256, decay=128),
        dict(temperature=0.8, top_k=8, top_p=0.0, min_p=0.0, typical=0.0, penalty_max=1.0, sustain=-1, decay=0),
        dict(temperature=1.2, top_k=0, top_p=0.9, min_p=0.02, typical=0.0, penalty_max=1.1, sustain=-1, decay=0),
        dict(temperature=1.0, top_k=0, top_p=0.0, min_p=0.0, typical=0.5, penalty_max=1.0, sustain=-1, decay=0),
        dict(temperature=0.95, top_k=20, top_p=0.8, min_p=0.0, typical=0.7, penalty_max=1.3, sustain=8, decay=16),
    ]
    seed = 0
    for beams in range(1, 6):
        for beam_length in range(1, 7):
            if beam_length == 1 and beams > 1:
                continue
            for ki, st in enumerate(kinds):
                if (beams + beam_length + ki) % 2 and not (beams == 1 and beam_length == 1):
                    continue                                        # half the grid keeps the fixture small
                for attempt in range(8):
                    seed += 1
                    vocab = int(rng.choice([64, 200, 512]))
                    L = int(rng.integers(1, 12))
                    c = dict(seed=seed, vocab=vocab, settings=st, beams=beams, beam_length=beam_length, max_seq=64,
                             bos=int(rng.integers(vocab)) if seed % 2 else -1,
                             prompt=[int(t) for t in rng.integers(0, vocab, L)])
                    n_emit = 6
                    try:
                        emitted, draws, windows = run_reference(Gen, Model, Cache, c, n_emit)
                    except Exception as e:                          # noqa: BLE001  (a reference failure: try another seed)
                        print("reference failed", seed, e)
                        continue
                    c["draws"] = draws[0] if not (beams == 1 and beam_length == 1) else [d[0] for d in draws]
                    c["emitted"] = emitted
                    try:
                        r = B.run_case(c)
                    except (RuntimeError, AssertionError):
                        continue
                    if r["emitted"] != emitted or r["expansions"] != windows or B.min_margin(r) < MARGIN:
                        continue
                    c["expansions"] = windows
                    cases.append(c)
                    break
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "beam_ref.npz")
    np.savez_compressed(path, cases=np.array(json.dumps(cases)))
    print(f"{len(cases)} cases -> {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
