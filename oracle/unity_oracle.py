"""TEST INFRASTRUCTURE (CPU oracle) -- not part of the product path.

CPU restatement of UnitY's second pass as `fairseq-generate --task speech_to_speech_modified --beam 1` runs it
(researches/translatotron/sequence_generator_multi_decoder.py:236-268):

  synthesizer_encoder(x, mt_decoder_padding_mask)      TransformerEncoderNoEmb: pre-LN layers, padded MT positions masked as keys,
                                                        no positions, final LayerNorm (StreamSpeechOracle.t2u_encoder, bidirectional)
  generator.generate_decoder(t2u_encoder_out)          fairseq/examples/speech_to_speech/unity/sequence_generator.py:158-523 with
                                                        BeamSearch at beam_size 1 (fairseq/search.py:104-146), min_len 1, unk
                                                        penalty 0, temperature 1, normalize_scores (finalize_hypos)

The unit decoder (TransformerUnitDecoder, n_frames_per_step 1) is fairseq's pre-LN TransformerDecoder: sqrt(dim)-scaled embedding
plus the sinusoidal row pad + 1 + step, self-attention over the tokens fed so far, cross-attention over the sample's T2U states,
FFN, final LayerNorm and the tied output projection.  Decoded incrementally with K / V caches (the incremental_state path), all rows
of a batch together; a row stops at its eos.  At beam 1 BeamSearch's choice is the best of log_softmax + cumulative score, lower
token index first on exactly equal scores (the rule of ss_unit_search_batch), eos finalizes.

`max_len` is the caller's min(int(max_len_a * src_tokens.size(1) + max_len_b), max_decoder_positions - 1): the batch's padded
source length (unity_max_len).  The arithmetic follows `dtype`: float32 restates the reference, float64 gives the margins.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from .streamspeech_oracle import StreamSpeechOracle, sinusoidal_table


def unity_max_len(max_len_a: float, max_len_b: int, padded_src_len: int, max_decoder_positions: int) -> int:
    """generate_decoder's max_len (unity/sequence_generator.py:182-194): src_len = src_tokens.size(1), the batch's padded length"""
    return min(int(max_len_a * padded_src_len + max_len_b), max_decoder_positions - 1)


class UnitYOracle:
    def __init__(self, cfg, model_sd: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float32, device="cpu"):
        assert cfg.unity and not cfg.uni_encoder
        self.cfg = cfg
        self.dtype = dtype
        self.o = StreamSpeechOracle(cfg, model_sd, None, None, chunk_size=None, dtype=dtype, device=device)
        self.device = self.o.device
        self.sd = self.o.sd
        # computed in fp32, then converted (what the engine loads as __const__.unit_pos_table)
        self.pos = sinusoidal_table(cfg.max_target_positions + cfg.pad + 1, cfg.unit_dim, cfg.pad).to(self.device, dtype)

    def t2u_encode(self, feats: torch.Tensor, lengths: Sequence[int]) -> torch.Tensor:
        """feats [B, S, D] (MT decoder features of [eos, hyp..., pad...]), lengths[b] = non-pad positions -> [B, S, D]"""
        B, S, _ = feats.shape
        pad = torch.arange(S).view(1, S) >= torch.tensor([int(n) for n in lengths]).view(B, 1)
        return self.o.t2u_encoder(feats.transpose(0, 1), pad if pad.any() else None).transpose(0, 1)

    def _lin(self, x, p):
        b = self.sd.get(p + ".bias")
        return F.linear(x, self.sd[p + ".weight"], b)

    def _ln(self, x, p):
        return F.layer_norm(x, (x.shape[-1],), self.sd[p + ".weight"], self.sd[p + ".bias"], 1e-5)

    def _attend(self, q, k, v, mask):
        """q [B, D], k / v [B, L, D], mask [B, L] (True = not a key) -> [B, D], heads of 64"""
        B, L, D = k.shape
        H = D // 64
        q = q.view(B, H, 1, 64)
        k = k.view(B, L, H, 64).transpose(1, 2)
        v = v.view(B, L, H, 64).transpose(1, 2)
        w = q @ k.transpose(-1, -2)  # q is already scaled
        if mask is not None:
            w = w.masked_fill(mask.view(B, 1, 1, L), -math.inf)
        w = torch.softmax(w, dim=-1)
        return (w @ v).reshape(B, D)

    def unit_search(self, t2u: torch.Tensor, lengths: Sequence[int], max_len: int, len_penalty: float = 1.0,
                    min_len: int = 1) -> List[Dict[str, object]]:
        """t2u [B, S, D] (t2u_encode's output), lengths[b] = the sample's keys.  One dict per sample: tokens (eos last),
        positional_scores, score, margins = the gap between the best candidate and the best finite one of a lower score at each step
        (how far the search is from changing that decision; exactly equal scores go to the lower index), margin = their minimum and
        ties = the steps whose best score was held by more than one token."""
        c, dt = self.cfg, self.dtype
        assert min_len <= max_len
        B, S, D = t2u.shape
        dev = self.device
        t2u = t2u.to(dev, dt)
        scale = 64 ** -0.5
        kpad = (torch.arange(S).view(1, S) >= torch.tensor([int(n) for n in lengths]).view(B, 1)).to(dev)
        cross = []
        for l in range(c.unit_layers):
            p = f"decoder.layers.{l}.encoder_attn"
            cross.append((self._lin(t2u, p + ".k_proj"), self._lin(t2u, p + ".v_proj")))
        E = self.sd["decoder.embed_tokens.weight"]
        selfk = [torch.zeros(B, 0, D, dtype=dt, device=dev) for _ in range(c.unit_layers)]
        selfv = [torch.zeros(B, 0, D, dtype=dt, device=dev) for _ in range(c.unit_layers)]
        tok = torch.full((B,), c.eos, dtype=torch.long, device=dev)
        out = [{"tokens": [], "cum": [], "score": None, "margin": math.inf, "margins": [], "ties": 0} for _ in range(B)]
        live = list(range(B))
        cum = torch.zeros(B, dtype=dt, device=dev)
        for step in range(max_len + 1):
            x = math.sqrt(D) * E[tok] + self.pos[c.pad + 1 + step]
            for l in range(c.unit_layers):
                p = f"decoder.layers.{l}"
                y = self._ln(x, p + ".self_attn_layer_norm")
                q = self._lin(y, p + ".self_attn.q_proj") * scale
                selfk[l] = torch.cat([selfk[l], self._lin(y, p + ".self_attn.k_proj").unsqueeze(1)], 1)
                selfv[l] = torch.cat([selfv[l], self._lin(y, p + ".self_attn.v_proj").unsqueeze(1)], 1)
                x = x + self._lin(self._attend(q, selfk[l], selfv[l], None), p + ".self_attn.out_proj")
                y = self._ln(x, p + ".encoder_attn_layer_norm")
                q = self._lin(y, p + ".encoder_attn.q_proj") * scale
                x = x + self._lin(self._attend(q, cross[l][0], cross[l][1], kpad), p + ".encoder_attn.out_proj")
                y = self._ln(x, p + ".final_layer_norm")
                x = x + self._lin(F.relu(self._lin(y, p + ".fc1")), p + ".fc2")
            logits = F.linear(self._ln(x, "decoder.layer_norm"), E)
            lp = F.log_softmax(logits, dim=-1)
            lp[lp != lp] = -math.inf
            lp[:, c.pad] = -math.inf
            if step >= max_len:
                lp[:, : c.eos] = -math.inf
                lp[:, c.eos + 1:] = -math.inf
            elif step < min_len:
                lp[:, c.eos] = -math.inf
            sc = lp + cum.view(-1, 1)
            nxt = tok.clone()
            keep = []
            for i, b in enumerate(live):
                row = sc[i].to(torch.float64)
                mx = row.max()
                tied = torch.nonzero(sc[i] == sc[i].max()).view(-1)
                best = int(tied[0])  # lowest index among exact ties
                out[b]["ties"] += len(tied) > 1
                below = row[row < mx]  # the gap to the best distinct score (exact ties are decided by the index, not arithmetic)
                second = float(below.max()) if below.numel() else -math.inf
                gap = float(mx) - second if math.isfinite(second) else math.inf
                out[b]["margins"].append(gap)
                out[b]["margin"] = min(out[b]["margin"], gap)
                out[b]["tokens"].append(best)
                out[b]["cum"].append(sc[i, best])
                if best == c.eos:  # finalize_hypos: positional scores are the steps' differences of the cumulative score
                    n = len(out[b]["tokens"])
                    cs = torch.stack(out[b].pop("cum"))
                    out[b]["positional_scores"] = [float(v) for v in torch.cat([cs[:1], cs[1:] - cs[:-1]])]
                    out[b]["score"] = float(cs[-1] / (n ** len_penalty))
                else:
                    keep.append(i)
                    nxt[i] = best
                    cum[i] = sc[i, best]
            if not keep:
                break
            idx = torch.tensor(keep, device=dev)
            live = [live[i] for i in keep]
            tok, cum, kpad = nxt[idx], cum[idx], kpad[idx]
            selfk = [k[idx] for k in selfk]
            selfv = [v[idx] for v in selfv]
            cross = [(k[idx], v[idx]) for k, v in cross]
        return out

    def generate_units(self, feats: torch.Tensor, lengths: Sequence[int], max_len: int, len_penalty: float = 1.0):
        """T2U encoder then the unit search of a batch (the oracle of the engine's last two UnitY stages)"""
        return self.unit_search(self.t2u_encode(feats, lengths), lengths, max_len, len_penalty)


def unity_generate(u: UnitYOracle, feats: torch.Tensor, lengths: Sequence[int], beam_mt: int, max_len_a: float, max_len_b: int,
                   max_len_b_mt: int = 200, len_penalty: float = 1.0) -> Dict[str, object]:
    """The whole batch as MultiDecoderSequenceGenerator._generate runs it (sequence_generator_multi_decoder.py:134-268): the offline
    encoder, the MT search per sample (beam_mt 1: greedy; else BeamSearch with len_penalty_mt = 1, finalized[b][0]), the MT decoder
    features of [eos, hyp..., pad...], the T2U encoder and the unit search with the batch's max_len.  feats [B, F, 80] zero padded."""
    from .mt_beam_oracle import mt_beam

    o, c = u.o, u.cfg
    enc = o.encoder(feats, torch.as_tensor([int(n) for n in lengths]))
    eo = enc["encoder_out"][0]
    pad_mask = enc["encoder_padding_mask"][0] if enc["encoder_padding_mask"] else None
    hyps = []
    for b in range(eo.shape[1]):
        Tb = int(enc["out_lengths"][b])
        if beam_mt == 1:
            h = o.mt_greedy(eo[:Tb, b:b + 1], None, -1, max_len_b=max_len_b_mt, max_decoder_positions=c.max_target_positions)
        else:
            h = mt_beam(o, eo[:Tb, b:b + 1], beam_mt, max_len_b_mt, 1.0, max_decoder_positions=c.max_target_positions)["hyps"][0]["tokens"]
        hyps.append([t for t in h if t != c.eos])
    S = max(len(h) for h in hyps) + 1
    prev = torch.tensor([[c.eos] + h + [c.pad] * (S - 1 - len(h)) for h in hyps], dtype=torch.long)
    x = o.mt_features(prev, eo, pad_mask)
    t2u_len = [len(h) + 1 for h in hyps]
    max_len = unity_max_len(max_len_a, max_len_b, int(feats.shape[1]), c.max_target_positions)
    return {"mt_hyps": hyps, "max_len": max_len, "units": u.unit_search(u.t2u_encode(x, t2u_len), t2u_len, max_len, len_penalty)}
