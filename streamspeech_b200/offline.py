"""Offline batched S2ST generation on the H100 engine (SURVEY.md §8 row O1).

Drop-in for the reference's `CTCMultiDecoderSequenceGenerator` as `fairseq-generate --task speech_to_speech_ctc` uses it
(researches/ctc_unity/sequence_generator_multi_decoder_ctc.py:163-331, built by tasks/speech_to_speech_ctc.py:21-49) with
`--beam-mt K --lenpen L --beam 1`, plus the batch-1 vocoder pass of `generate_waveform_from_code.py:40-78`:

    batched padded encoder (offline model: chunk_size None)                       ss_encoder_forward(B, lengths)
    ASR / ST CTC prints over all T rows of every sample (:206-246)                ss_ctc_greedy_batch
    MT search of the batch, max_len = max_len_b_mt (:251-260): K = 1 greedy        ss_mt_greedy_batch
      K >= 2 beam search, best finalized hypothesis finalized[b][0] (:262-279)    ss_mt_beam_batch
    prev_output_tokens_mt = [eos, hyp..., pad...] to the batch maximum (:262-271) host
    mt_decoder(features_only) on the padded batch (:287-291)                      ss_mt_features_batch
    T2U encoder -> CTC unit decoder -> CTC generate (:293-330)                    ss_t2u_unit_decode_batch
      with the unit hypothesis' scores (generate(scores=True))                    ss_t2u_unit_decode_batch_scored

Each stage is one call for the whole batch (the entry points split batches larger than their workspace budget into groups
themselves), so the host synchronisations of generate() do not grow with B.  Samples only interact through three quirks of the
reference, which the batched calls reproduce (oracle/offline_oracle.py is pinned against the reference modules on a padded batch):
  N1  the unit decoder's positional embedding is indexed by the BATCH axis: sample b gets position b + 2 at every step
      -> Engine.t2u_unit_decode_batch passes every sample's row (Engine.unit_position_row(b))
  N2  hypotheses keep the tokens emitted at padded T2U positions -> the pad tail is decoded too (n_pad_tail)
  N3  pad, unk and eos are masked before the arg-max (researches/ctc_unity/ctc_generator.py:56-58) -> mask_eos
The T2U beam (`--beam`) stays 1: the reference's CTC unit decoder does not search; max_len_a_mt stays 0.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch

from .engine import Engine, EngineError


class OfflineS2STGenerator:
    def __init__(self, engine: Engine, beam_size_mt: int = 1, beam_size: int = 1, max_len_a_mt: float = 0.0, max_len_b_mt: int = 200,
                 len_penalty: float = 1.0):
        if beam_size != 1:
            raise NotImplementedError("the H100 offline generator implements beam_size = 1 only (the CTC unit decoder does not search)")
        if int(beam_size_mt) != beam_size_mt or not 1 <= beam_size_mt <= 32:
            raise ValueError(f"beam_size_mt must be an integer in [1, 32], got {beam_size_mt}")
        if max_len_a_mt != 0.0:
            raise NotImplementedError("max_len_a_mt != 0 is not supported (the reference default is 0)")
        if not math.isfinite(len_penalty):
            raise ValueError(f"len_penalty must be finite, got {len_penalty}")
        self.engine = engine
        self.cfg = engine.cfg
        self.beam_size_mt = int(beam_size_mt)
        self.len_penalty = float(len_penalty)
        self.max_len_b_mt = int(max_len_b_mt)
        engine.set_chunk(None, None)  # offline model: full attention, symmetric convolutions (N10)

    @torch.inference_mode()
    def generate(self, src_tokens: torch.Tensor, src_lengths: Sequence[int], forced_mt: Optional[List[List[int]]] = None,
                 scores: bool = False) -> List[Dict[str, object]]:
        """src_tokens [B, F, 80] fbank + CMVN features on the engine's device (zero padded), src_lengths [B].
        Returns one dict per sample: asr_tokens / st_tokens (CTC prints), mt_tokens (hypothesis without eos), units (the
        reference's `finalized[b][0]["tokens"]`), unit_argmax (per-position arg-max, padded positions included) and
        mt_feats ([max_tgt_len, 512], device).  forced_mt: use these MT hypotheses instead of searching (tests).
        scores: each result also gets the unit hypothesis' scores as `fairseq-generate` prints them (ctc_generator.py:54-61):
        unit_positional_scores (fp32 [max_tgt_len * rate], pad-tail rows included) and unit_score (their fp32 sum)."""
        eng, c = self.engine, self.cfg
        if src_tokens.dim() != 3 or not src_tokens.is_cuda:
            raise EngineError("src_tokens must be a [B, F, feat_dim] CUDA tensor")
        B = src_tokens.shape[0]
        lengths = [int(x) for x in src_lengths]
        enc = eng.encoder(src_tokens.contiguous(), lengths)  # [B, T, C], padded rows included
        out_len = [eng.encoder_out_frames(n) for n in lengths]
        prints, _ = eng.ctc_greedy_batch(enc)  # padded frames are NOT trimmed (ctc_decoder.py:60-63)
        results: List[Dict[str, object]] = [{"asr_tokens": asr[0], "st_tokens": st[0]} for asr, st in prints]
        hyps: List[List[int]]
        if forced_mt is not None:
            hyps = [list(h) for h in forced_mt]
        elif self.beam_size_mt == 1:
            hyps = eng.mt_greedy_batch(enc, out_len, self.max_len_b_mt)  # all samples in one search
        else:
            nbest = eng.mt_beam_batch(enc, out_len, self.beam_size_mt, self.max_len_b_mt, self.len_penalty)
            hyps = [n[0]["tokens"] for n in nbest]
        max_tgt_len = max(len(h) for h in hyps) + 1  # hypothesis + eos (:262)
        n_pad = [max_tgt_len - (len(h) + 1) for h in hyps]
        prev = [[c.eos] + h + [c.pad] * n for h, n in zip(hyps, n_pad)]
        feats = eng.mt_features_batch(enc, out_len, prev)  # [B, max_tgt_len, mt_dim]
        if scores:
            units, argmax, lprob, _ = eng.t2u_unit_decode_batch_scored(feats, n_pad, mask_eos=True)  # N1, N2, N3
            for b in range(B):
                results[b].update(unit_positional_scores=lprob[b], unit_score=float(lprob[b].sum()))
        else:
            units, argmax, _ = eng.t2u_unit_decode_batch(feats, n_pad, mask_eos=True)  # N1, N2, N3
        for b in range(B):
            results[b].update(mt_tokens=hyps[b], units=units[b], unit_argmax=argmax[b], mt_feats=feats[b])
        return results

    def units_to_codes(self, units: Sequence[int]) -> List[int]:
        """dictionary indices -> vocoder codes: the unit dictionary is 4 specials, then "0" .. "999", then <blank>
        (tasks/speech_to_speech_ctc.py:15-17); what `tgt_dict.string()` + int() does in the reference's scripts"""
        n = self.cfg.vocoder.num_embeddings
        return [int(u) - 4 for u in units if 4 <= int(u) < 4 + n]

    def synthesize(self, codes: Sequence[int], dur_prediction: bool = True) -> torch.Tensor:
        """generate_waveform_from_code.py:58-71: one utterance, whole sequence.  `codes` are vocoder code indices (0..999)."""
        return self.synthesize_batch([codes], dur_prediction)[0]

    @torch.inference_mode()
    def synthesize_batch(self, codes_list: Sequence[Sequence[int]], dur_prediction: bool = True) -> List[torch.Tensor]:
        """synthesize() of every utterance in one vocoder durations call and one generate call; each waveform equals synthesize()'s
        bit for bit (views of one device buffer)."""
        return vocode_whole(self.engine, codes_list, dur_prediction)


class UnitYGenerator:
    """UnitY's `MultiDecoderSequenceGenerator` as `fairseq-generate --task speech_to_speech_modified --beam-mt K --beam 1` runs it
    (researches/translatotron/sequence_generator_multi_decoder.py:134-268) on the engine, one call per stage for the whole batch:

        batched padded encoder (UnitY: offline model; Uni-UnitY: future mask)         ss_encoder_forward(B, lengths)
        MT search, max_len = max_len_b_mt: K = 1 greedy, K >= 2 beam (finalized[b][0])  ss_mt_greedy_batch / ss_mt_beam_batch
        prev_output_tokens_mt = [eos, hyp..., pad...] to the batch maximum             host
        mt_decoder(features_only) on the padded batch                                 ss_mt_features_batch
        synthesizer_encoder(x, prev_output_tokens_mt == pad)                          ss_t2u_encode_batch
        unit search at beam 1, max_len = min(int(max_len_a * F + max_len_b),          ss_unit_search_batch
          max_target_positions - 1) with F the batch's PADDED fbank length

    There are no CTC prints (UnitY has no CTC heads); the D- text is the MT hypothesis.  A Uni-UnitY checkpoint
    (researches/uni_unity) runs the same stages with its encoder's future mask and a causal T2U encoder (cfg.uni_encoder), under
    fairseq's own MultiDecoderSequenceGenerator, which prints the MT text as "{text} (None-{id})" (generate.mt_print_line)."""

    def __init__(self, engine: Engine, beam_size_mt: int = 1, beam_size: int = 1, max_len_a_mt: float = 0.0, max_len_b_mt: int = 200,
                 max_len_a: float = 0.0, max_len_b: int = 200, len_penalty: float = 1.0):
        if not engine.cfg.unity:
            raise ValueError("UnitYGenerator needs a UnitY checkpoint (OfflineS2STGenerator runs StreamSpeech)")
        if beam_size != 1:
            raise NotImplementedError("the H100 UnitY generator implements the unit search at beam_size = 1 only")
        if int(beam_size_mt) != beam_size_mt or not 1 <= beam_size_mt <= 32:
            raise ValueError(f"beam_size_mt must be an integer in [1, 32], got {beam_size_mt}")
        if max_len_a_mt != 0.0:
            raise NotImplementedError("max_len_a_mt != 0 is not supported (the reference default is 0)")
        if not math.isfinite(len_penalty) or not math.isfinite(max_len_a):
            raise ValueError("len_penalty and max_len_a must be finite")
        self.engine = engine
        self.cfg = engine.cfg
        self.beam_size_mt = int(beam_size_mt)
        self.len_penalty = float(len_penalty)
        self.max_len_b_mt = int(max_len_b_mt)
        self.max_len_a, self.max_len_b = float(max_len_a), int(max_len_b)
        if self.cfg.unity_variant == "chunk_unity":
            raise NotImplementedError("Chunk-UnitY is a simultaneous model: it runs in the wait-k agents, not the offline generator")
        engine.set_chunk(*self.cfg.encoder_chunk())  # UnitY: the offline model; Uni-UnitY: a future mask, symmetric convolutions

    def unit_max_len(self, padded_frames: int) -> int:
        """generate_decoder's max_len (unity/sequence_generator.py:182-194) for a batch of `padded_frames` fbank frames"""
        return min(int(self.max_len_a * padded_frames + self.max_len_b), self.cfg.max_target_positions - 1)

    @torch.inference_mode()
    def generate(self, src_tokens: torch.Tensor, src_lengths: Sequence[int], scores: bool = False) -> List[Dict[str, object]]:
        """src_tokens [B, F, 80] on the engine's device (zero padded), src_lengths [B].  One dict per sample: mt_tokens (MT
        hypothesis without eos), units (the reference's finalized[b][0]["tokens"], eos last), unit_score and unit_positional_scores
        (fp32, one per unit; computed whatever `scores`, which is accepted for OfflineS2STGenerator's signature)."""
        eng, c = self.engine, self.cfg
        if src_tokens.dim() != 3 or not src_tokens.is_cuda:
            raise EngineError("src_tokens must be a [B, F, feat_dim] CUDA tensor")
        lengths = [int(x) for x in src_lengths]
        max_len = self.unit_max_len(int(src_tokens.shape[1]))
        if max_len < 1:
            raise ValueError("min_len cannot be larger than max_len, please adjust these!")
        enc = eng.encoder(src_tokens.contiguous(), lengths)
        out_len = [eng.encoder_out_frames(n) for n in lengths]
        if self.beam_size_mt == 1:
            hyps = eng.mt_greedy_batch(enc, out_len, self.max_len_b_mt)
        else:
            # (build_generator_dual_decoder passes --lenpen to the unit generator only: the MT generator keeps len_penalty_mt = 1)
            hyps = [n[0]["tokens"] for n in eng.mt_beam_batch(enc, out_len, self.beam_size_mt, self.max_len_b_mt, 1.0)]
        S = max(len(h) for h in hyps) + 1
        feats = eng.mt_features_batch(enc, out_len, [[c.eos] + h + [c.pad] * (S - 1 - len(h)) for h in hyps])
        t2u_len = [len(h) + 1 for h in hyps]
        t2u = eng.t2u_encode_batch(feats, t2u_len)
        units = eng.unit_search_batch(t2u, t2u_len, max_len, self.len_penalty)
        return [{"mt_tokens": h, "units": u["tokens"], "unit_score": u["score"], "unit_positional_scores": u["positional_scores"]}
                for h, u in zip(hyps, units)]


def vocode_whole(eng, codes_list: Sequence[Sequence[int]], dur_prediction: bool) -> List[torch.Tensor]:
    """Whole-sequence vocoder passes of the code sequences: one durations call, one host read of the cumsums, one generate call."""
    _, cums, _ = eng.vocoder_durations_ragged([[int(u) for u in c] for c in codes_list], dur_prediction)
    totals = [c[-1] for c in cums]
    return eng.vocoder_generate_ragged(totals, [0] * len(totals), totals, [0] * len(totals))
