"""TEST INFRASTRUCTURE (CPU oracle) -- not part of the product path.

CPU restatement of the reference's wait-k-stride-n agents on a UnitY checkpoint (agent/speech_to_speech.wait-k-stride-n.agent.py
and agent/speech_to_text.wait-k-stride-n.agent.py, policy() :358-581 and reset() :290-296), in float32 as the reference runs:

  gate                 src_seg_num = len(source) // (segment_size * rate / 1000), subword / unit counts of k1, n, k2, n2,
                       unit_per_subword (READ while a count is below 1 and the source is open, -1 once it has ended)
  features / encoder   online_features of the whole source, the offline (bidirectional) encoder on the whole prefix
  MT                   greedy generate_decoder with the previous hypothesis as prefix and max_len = prefix + new tokens, or
                       min(F + 200, max_decoder_positions - 1) once the source has ended (no incremental state)
  S2ST                 MT decoder features of [eos, tokens...], synthesizer_encoder, the unit search from BOS (UnitYOracle) with
                       the absolute unit count as max_len, the vocoder on all units and the samples of the new units
  S2TT                 " ".join of the subword symbols, the text delta

`rate` is the source's sample rate (16 kHz here: the fixture's sources are 16 kHz and the reference's convert_waveform is then
the identity).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .agent_oracle import OracleAction
from .streamspeech_oracle import StreamSpeechOracle, online_features
from .unity_oracle import UnitYOracle


class _OracleWaitk:
    def __init__(self, cfg, sd, gcmvn, vsd=None, lagging_k1=3, lagging_k2=1, stride_n=1, stride_n2=1, unit_per_subword=15,
                 segment_size=320, sample_rate=16000, symbols=None, unit_symbols=None, dtype=torch.float32):
        self.cfg = cfg
        self.o = StreamSpeechOracle(cfg, sd, vsd, gcmvn, chunk_size=None, dtype=dtype)
        self.k1, self.k2, self.n, self.n2, self.ups = lagging_k1, lagging_k2, stride_n, stride_n2, unit_per_subword
        self.segment_size, self.rate = segment_size, sample_rate
        self.symbols = symbols if symbols is not None else str
        self.max_decoder_positions = cfg.max_target_positions
        self.reset()

    def reset(self):
        self.source: List[float] = []
        self.source_finished = False
        self.target_finished = False
        self.src_seg_num = 0
        self.tgt_subwords_indices: Optional[List[int]] = None
        self.unit: Optional[List[int]] = None
        self.tgt_text = ""

    def push(self, samples, finished: bool = False):
        self.source.extend(samples)
        self.source_finished = finished

    def unit_tokens(self, subword_tokens):
        return ((subword_tokens - self.k2) // self.n2) * self.n2 * self.ups

    def gate(self, trace):
        fin = self.source_finished
        src_seg_num = int(len(self.source) // (self.segment_size * self.rate / 1000))
        if (src_seg_num <= self.src_seg_num or src_seg_num < self.k1) and not fin:
            return None
        self.src_seg_num = src_seg_num
        subword_tokens = ((src_seg_num - self.k1) // self.n) * self.n
        new_sub = subword_tokens - len(self.tgt_subwords_indices) if self.tgt_subwords_indices is not None else subword_tokens
        new_unit = self.unit_tokens(subword_tokens)
        if (new_sub < 1 or new_unit < 1) and not fin:
            return None
        if fin:
            new_sub = new_unit = -1
        trace["new_subword_tokens"], trace["new_unit_tokens"] = new_sub, new_unit
        return new_sub, new_unit

    def translate(self, new_sub, trace):
        """features, encoder, MT: (hypothesis with its eos, encoder output, fbank frames) or None for READ"""
        feature = online_features(torch.tensor(self.source, dtype=torch.float32), self.o.gcmvn)
        F = int(feature.size(0))
        if F == 0 and not self.source_finished:
            return None
        eo = self.o.encoder(feature.unsqueeze(0), torch.tensor([F]))["encoder_out"][0]
        max_len_b = min(F + 200, self.max_decoder_positions - 1)
        margins = []
        hyp = self.o.mt_greedy(eo, self.tgt_subwords_indices, new_sub, max_len_b=max_len_b, max_decoder_positions=self.max_decoder_positions,
                               margins=margins)
        trace["mt_margin"] = min(margins)
        self.tgt_subwords_indices = hyp[:-1]
        trace["mt_tokens"] = list(hyp[:-1])
        return hyp, eo, F


class OracleWaitkS2STAgent(_OracleWaitk):
    def __init__(self, cfg, sd, gcmvn, vsd, dur_prediction=True, **kw):
        super().__init__(cfg, sd, gcmvn, vsd, **kw)
        self.u = UnitYOracle(cfg, sd, self.o.dtype)
        self.dur_prediction = dur_prediction

    def policy(self) -> OracleAction:
        c, trace = self.cfg, {}
        fin = self.source_finished
        g = self.gate(trace)
        if g is None:
            return OracleAction("read", trace=trace)
        new_sub, _ = g
        r = self.translate(new_sub, trace)
        if r is None:
            return OracleAction("read", trace=trace)
        hyp, eo, F = r
        new_unit = self.unit_tokens(len(self.tgt_subwords_indices))
        if new_unit < 1 and not fin:
            return OracleAction("read", trace=trace)
        if fin:
            new_unit = -1
        tmp = hyp[:-1] if hyp[-1] == c.eos else hyp
        prev = torch.tensor([[c.eos] + tmp + [c.pad] * (len(hyp) - 1 - len(tmp))], dtype=torch.long)
        x = self.o.mt_features(prev, eo)  # [1, S, D]
        S = len(hyp)
        max_len = new_unit if new_unit != -1 else min(F + 200, self.max_decoder_positions - 1)
        out = self.u.unit_search(self.u.t2u_encode(x, [S]), [S], max_len)[0]
        trace["unit_margin"] = out["margin"]
        toks = out["tokens"]
        tmp = toks[:-1] if toks[-1] == c.eos else toks
        unit = [t - 4 for t in tmp]  # the unit dictionary's symbols: 4 specials, then "0".."999"
        assert all(u >= 0 for u in unit), "a special symbol among the units: the reference's int(symbol) raises"
        trace["units"] = list(unit)
        cur_unit = unit if self.unit is None else unit[len(self.unit):]
        if len(unit) < 1 or len(cur_unit) < 1:
            if not fin:
                return OracleAction("read", trace=trace)
            return OracleAction("write", wav=[], finished=True, seg_finished=True, trace=trace)
        wav, dur = self.o.vocoder(unit, self.dur_prediction)
        n = int(dur[:, -len(cur_unit):].sum()) * 320
        trace["dur"] = dur.view(-1).tolist()
        self.unit = unit
        if new_sub == -1 and new_unit == -1:
            self.target_finished = True
            self.reset()
        return OracleAction("write", wav=wav[-n:].tolist(), finished=self.target_finished, seg_finished=self.source_finished, trace=trace)


class OracleWaitkS2TTAgent(_OracleWaitk):
    def policy(self) -> OracleAction:
        trace = {}
        g = self.gate(trace)
        if g is None:
            return OracleAction("read", trace=trace)
        new_sub, _ = g
        r = self.translate(new_sub, trace)
        if r is None:
            return OracleAction("read", trace=trace)
        text = " ".join(self.symbols(t) for t in self.tgt_subwords_indices)
        new_text = text[len(self.tgt_text):]
        self.tgt_text = text
        if self.source_finished and new_sub == -1:
            self.target_finished = True
            self.reset()
        return OracleAction("write", wav=new_text, finished=self.target_finished, trace=trace)
