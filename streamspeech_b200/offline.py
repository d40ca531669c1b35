"""Offline batched S2ST generation on the H100 engine (SURVEY.md §8 row O1).

Drop-in for the reference's `CTCMultiDecoderSequenceGenerator` as `fairseq-generate --task speech_to_speech_ctc` uses it
(researches/ctc_unity/sequence_generator_multi_decoder_ctc.py:163-331, built by tasks/speech_to_speech_ctc.py:21-49) with
`--beam-mt 1 --beam 1`, plus the batch-1 vocoder pass of `generate_waveform_from_code.py:40-78`:

    batched padded encoder (offline model: chunk_size None)                       ss_encoder_forward(B, lengths)
    ASR / ST CTC prints over all T rows of every sample (:206-246)                ss_ctc_greedy
    MT greedy search of the batch, max_len = max_len_b_mt (:251-260)              ss_mt_greedy_batch
    prev_output_tokens_mt = [eos, hyp..., pad...] to the batch maximum (:262-271) host
    mt_decoder(features_only) -> T2U encoder -> CTC unit decoder (:287-330)       ss_mt_features, ss_t2u_unit_decode

The reference runs the last three on the padded batch; utterances only interact through three quirks, which the per-sample
calls reproduce exactly (oracle/offline_oracle.py is pinned against the reference modules on a padded batch):
  N1  the unit decoder's positional embedding is indexed by the BATCH axis: sample b gets position b + 2 at every step
      -> Engine.set_unit_batch_index(b)
  N2  hypotheses keep the tokens emitted at padded T2U positions -> the pad tail is decoded too (n_pad_tail)
  N3  pad, unk and eos are masked before the arg-max (researches/ctc_unity/ctc_generator.py:56-58) -> mask_eos
Beam search over the MT decoder (beam_size_mt > 1) is not implemented: the constructor refuses it.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .engine import Engine, EngineError


class OfflineS2STGenerator:
    def __init__(self, engine: Engine, beam_size_mt: int = 1, beam_size: int = 1, max_len_a_mt: float = 0.0, max_len_b_mt: int = 200):
        if beam_size_mt != 1 or beam_size != 1:
            raise NotImplementedError("the H100 offline generator implements beam_size_mt = beam_size = 1 (greedy) only")
        if max_len_a_mt != 0.0:
            raise NotImplementedError("max_len_a_mt != 0 is not supported (the reference default is 0)")
        self.engine = engine
        self.cfg = engine.cfg
        self.max_len_b_mt = int(max_len_b_mt)
        engine.set_chunk(None, None)  # offline model: full attention, symmetric convolutions (N10)

    @torch.inference_mode()
    def generate(self, src_tokens: torch.Tensor, src_lengths: Sequence[int], forced_mt: Optional[List[List[int]]] = None) -> List[Dict[str, object]]:
        """src_tokens [B, F, 80] fbank + CMVN features on the engine's device (zero padded), src_lengths [B].
        Returns one dict per sample: asr_tokens / st_tokens (CTC prints), mt_tokens (hypothesis without eos), units (the
        reference's `finalized[b][0]["tokens"]`), unit_argmax (per-position arg-max, padded positions included) and
        mt_feats ([max_tgt_len, 512], device).  forced_mt: use these MT hypotheses instead of searching (tests)."""
        eng, c = self.engine, self.cfg
        if src_tokens.dim() != 3 or not src_tokens.is_cuda:
            raise EngineError("src_tokens must be a [B, F, feat_dim] CUDA tensor")
        B = src_tokens.shape[0]
        lengths = [int(x) for x in src_lengths]
        enc = eng.encoder(src_tokens.contiguous(), lengths)  # [B, T, C], padded rows included
        T = enc.shape[1]
        out_len = [eng.encoder_out_frames(n) for n in lengths]
        results: List[Dict[str, object]] = []
        for b in range(B):
            eb = enc[b].contiguous()
            am = torch.zeros(T, dtype=torch.int64, device=eb.device)
            asr, _ = eng.ctc_greedy_rows(0, eb, 0, am)       # padded frames are NOT trimmed (ctc_decoder.py:60-63)
            st, _ = eng.ctc_greedy_rows(1, eb, 0, am)
            results.append({"asr_tokens": asr, "st_tokens": st})
        hyps: List[List[int]]
        if forced_mt is not None:
            hyps = [list(h) for h in forced_mt]
        else:
            hyps = eng.mt_greedy_batch(enc, out_len, self.max_len_b_mt)  # all samples in one search
        for b in range(B):
            results[b]["mt_tokens"] = hyps[b]
        max_tgt_len = max(len(h) for h in hyps) + 1  # hypothesis + eos (:262)
        try:
            for b in range(B):
                n_pad = max_tgt_len - (len(hyps[b]) + 1)
                prev = [c.eos] + hyps[b] + [c.pad] * n_pad
                feats = eng.mt_features(enc[b, : out_len[b]].contiguous(), prev)
                eng.set_unit_batch_index(b)  # N1
                r = eng.t2u_unit_decode(feats.contiguous(), n_pad_tail=n_pad, mask_eos=True)  # N2, N3
                results[b]["units"] = eng.units_to_host(r)
                results[b]["unit_argmax"] = r["argmax"].tolist()
                results[b]["mt_feats"] = feats
        finally:
            eng.set_unit_batch_index(0)
        return results

    def units_to_codes(self, units: Sequence[int]) -> List[int]:
        """dictionary indices -> vocoder codes: the unit dictionary is 4 specials, then "0" .. "999", then <blank>
        (tasks/speech_to_speech_ctc.py:15-17); what `tgt_dict.string()` + int() does in the reference's scripts"""
        n = self.cfg.vocoder.num_embeddings
        return [int(u) - 4 for u in units if 4 <= int(u) < 4 + n]

    @torch.inference_mode()
    def synthesize(self, codes: Sequence[int], dur_prediction: bool = True) -> torch.Tensor:
        """generate_waveform_from_code.py:58-71: one utterance, whole sequence.  `codes` are vocoder code indices (0..999)."""
        eng = self.engine
        codes = torch.tensor([int(u) for u in codes], dtype=torch.long, device=eng.device)
        _, cum = eng.vocoder_durations(codes, dur_prediction)
        total = int(cum[-1].item())
        return eng.vocoder_generate(total, 0, total, 0)
