"""TEST INFRASTRUCTURE (CPU oracle) -- not part of the product path.

CPU restatement of the offline generator's MT beam search (`--beam-mt K --lenpen L`): the reference's
`SequenceGenerator.generate_decoder` (fairseq/examples/speech_to_speech/unity/sequence_generator.py:158-523) with
`BeamSearch.step` (fairseq/fairseq/search.py:104-146) and `finalize_hypos` (fairseq/fairseq/sequence_generator.py:630-739) at
beam_size = K, min_len 1, normalize_scores, no prefix, one sample at a time (samples of a batch only share the padding mask),
over the pinned MT decoder restatement `StreamSpeechOracle.mt_logits`.  The arithmetic follows the oracle's dtype: float32
restates the reference, float64 gives the margins of its decisions.

Candidates are ranked by score, and on exactly equal scores by the lower flat index beam * vocab + token (the rule of
ss_mt_beam_batch; torch.topk leaves the order of ties unspecified).  Pinned by oracle/gen_golden_beam.py against the reference's
own generate_decoder (tests/golden/mt_beam.npz).
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

from .streamspeech_oracle import StreamSpeechOracle


def early_eos_state_dict(sd: Dict[str, torch.Tensor], eos: int, scale: float) -> Dict[str, torch.Tensor]:
    """A copy of `sd` whose MT output row of eos (tied with its input embedding) is multiplied by `scale`.  With scale -0.2 the
    seeded synthetic checkpoint ranks eos among the best candidates within a few tokens, so that a beam search finalizes
    hypotheses early while its sample searches on (the unmodified checkpoint's eos rises only after ~30 tokens)."""
    out = dict(sd)
    emb = sd["target_unigram_decoder.embed_tokens.weight"].clone()
    emb[eos] *= scale
    out["target_unigram_decoder.embed_tokens.weight"] = emb
    out["target_unigram_decoder.output_projection.weight"] = emb
    return out


def mt_beam(o: StreamSpeechOracle, enc_out: torch.Tensor, beam: int, max_len_b: int, len_penalty: float = 1.0,
            max_decoder_positions: int = 1024, min_len: int = 1) -> Dict[str, object]:
    """enc_out [T, 1, C] of one sample.  Returns {"hyps": the K finalized hypotheses sorted by score (highest first, stable), each
    {"tokens": [... eos], "score": float, "positional_scores": [...]}, "margin": the smallest gap between consecutive finite
    scores among the 2K + 1 best candidates of any step (how far the search is from changing a decision)}."""
    c = o.cfg
    K, V, dt = int(beam), c.tgt_vocab, o.dtype
    max_len = min(int(max_len_b), max_decoder_positions - 1)
    assert min_len <= max_len
    tokens: List[List[int]] = [[c.eos]]
    cum: List[List[torch.Tensor]] = [[]]  # cumulative score after each step, per beam (0-d tensors of dtype dt)
    finalized: List[Dict[str, object]] = []
    margin = math.inf
    for step in range(max_len + 1):
        rows = len(tokens)  # 1 at step 0: lprobs[:, ::beam_size]
        toks = torch.tensor(tokens, dtype=torch.long)
        logits = o.mt_logits(toks, enc_out.expand(-1, rows, -1))[:, -1, :]
        lprobs = F.log_softmax(logits.to(dt), dim=-1)
        lprobs[lprobs != lprobs] = -math.inf
        lprobs[:, c.pad] = -math.inf
        if step >= max_len:
            lprobs[:, : c.eos] = -math.inf
            lprobs[:, c.eos + 1:] = -math.inf
        elif step < min_len:
            lprobs[:, c.eos] = -math.inf
        if step > 0:
            lprobs = lprobs + torch.stack([h[-1] for h in cum]).view(-1, 1)
        flat = lprobs.reshape(-1).numpy()
        idx = np.arange(flat.size)
        order = np.lexsort((idx, -flat.astype(np.float64)))[: 2 * K + 1]
        top = flat[order]
        fin = top[np.isfinite(top)]
        if fin.size > 1:
            margin = min(margin, float(np.min(fin[:-1].astype(np.float64) - fin[1:].astype(np.float64))))
        cand = [(int(i) // V, int(i) % V, lprobs.reshape(-1)[int(i)]) for i in order[: 2 * K]]
        # finalize eos among the first K (finalize_hypos), while fewer than K hypotheses are held
        for b, t, v in cand[:K]:
            if t == c.eos and math.isfinite(float(v)) and len(finalized) < K:
                pos = torch.stack(cum[b] + [v])
                pos = torch.cat([pos[:1], pos[1:] - pos[:-1]])
                finalized.append({"tokens": tokens[b][1:] + [c.eos], "score": float(v / ((step + 1) ** len_penalty)),
                                  "positional_scores": [float(x) for x in pos]})
        if len(finalized) == K or step >= max_len:
            break
        nxt = [(b, t, v) for b, t, v in cand if not (t == c.eos and math.isfinite(float(v)))][:K]
        tokens = [tokens[b] + [t] for b, t, _ in nxt]
        cum = [cum[b] + [v] for b, _, v in nxt]
    hyps = sorted(finalized, key=lambda h: -h["score"])  # (stable)
    return {"hyps": hyps, "margin": margin}
