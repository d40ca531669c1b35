"""Generate tests/golden/unity_generate.npz from the reference's own UnitY code (build container only, CPU, a few minutes).

Run:  python -m oracle.gen_golden_unity      (needs /root/reference)

The fixture of `python -m streamspeech_b200.generate --task speech_to_speech_modified` (researches/unitY/test_scripts/pred.sh):

  model       the modules UnityConformerModelModified.build_model assembles (fairseq s2s_conformer_unity.py:125-211), each from
              the reference's own class, with the seeded synthetic UnitY state dict loaded strictly:
                encoder      fairseq's S2TConformerEncoder (speech_to_text/s2t_conformer.py, run from its own class body) with
                             fairseq's Conv1dSubsampler and ConformerEncoderLayer (--attn-type espnet --pos-enc-type rel_pos,
                             --conv-version s2t_transformer, the argparse default that pred.sh's training run kept)
                MT decoder   fairseq's TransformerDecoderBase (models/transformer/transformer_decoder.py), 4 x 512
                T2U encoder  fairseq's TransformerEncoderNoEmb (speech_to_speech/modules/transformer_encoder.py)
                unit decoder fairseq's TransformerUnitDecoder (s2s_transformer.py, its own class body) over StackedEmbedding
              The module classes load through oracle.ref_loader's stub recipe; the model object around them is a stand-in with
              the attributes MultiDecoderSequenceGenerator reads (UnityConformerModelModified itself needs fairseq's hydra-based
              registry, which is not installed).
  generator   researches/translatotron/sequence_generator_multi_decoder.py:MultiDecoderSequenceGenerator and fairseq's
              examples/speech_to_speech/unity/sequence_generator.py:SequenceGenerator, both imported unchanged, built as
              SpeechToSpeechTaskModified.build_generator_dual_decoder builds them (--beam 1, --max-len-a, --max-len-b, --lenpen 1)
  split       nine synthetic utterances of 0.8-4 s (raw fbank in steps of 1/32 as int16, gcmvn stats); batches by
              streamspeech_b200.generate.make_batches (pinned to fairseq's own batching by tests/golden/offline_generate.npz)
  settings    (--max-tokens, --beam-mt, --max-len-b) in SETTINGS: batches of unequal length, --beam-mt 1 and 4, and a small
              --max-len-b so that some samples run to the forced eos of max_len = int(1 * F_padded + max_len_b)

For each setting it records the `D-` prints (stdout), the results-file lines (T- / H- / D- / P- with generate.py's format
strings, Dictionary.string from its own source) and every sample's units, positional scores and score; it asserts that the
float32 oracle (oracle.unity_oracle.unity_generate) reproduces the MT hypotheses and units exactly and the scores within 1e-5,
and that both kinds of ending occur, before writing.
"""
from __future__ import annotations

import contextlib
import io
import math
import os
import sys
import types
from typing import Any, Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import GOLD, REF, FakeDict, extract_class, extract_functions, sub_state, transformer_cfg  # noqa: E402
from oracle.gen_golden_agent import load_file_module, load_reference_generators  # noqa: E402
from oracle.streamspeech_oracle import online_features  # noqa: E402
from oracle.unity_oracle import UnitYOracle, unity_generate  # noqa: E402
from streamspeech_b200 import generate as G  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402

DURATIONS = [2.0, 4.0, 1.0, 3.0, 0.8, 2.6, 1.5, 3.5, 1.2]
NPY_SAMPLES = (0, 4, 7)
RAW_SCALE = 32
MAX_LEN_B_MT = 60
SETTINGS = [(900, 1, 200), (900, 4, 200), (1500, 1, 10), (10000, 4, 10), (700, 4, 40)]


def load_reference_classes():
    """The reference's module and generator classes, unchanged (see the module docstring)."""
    search, _ = load_reference_generators()
    fm = sys.modules["fairseq.modules"]
    from fairseq.modules.multihead_attention import MultiheadAttention

    fm.MultiheadAttention = MultiheadAttention
    from fairseq.modules.transformer_layer import TransformerDecoderLayer, TransformerEncoderLayer

    fm.TransformerEncoderLayer, fm.TransformerDecoderLayer = TransformerEncoderLayer, TransformerDecoderLayer
    fm.transformer_layer = sys.modules["fairseq.modules.transformer_layer"]
    from fairseq.modules.espnet_multihead_attention import (ESPNETMultiHeadedAttention, RelPositionMultiHeadedAttention,
                                                            RotaryPositionMultiHeadedAttention)

    fm.ESPNETMultiHeadedAttention = ESPNETMultiHeadedAttention
    fm.RelPositionMultiHeadedAttention = RelPositionMultiHeadedAttention
    fm.RotaryPositionMultiHeadedAttention = RotaryPositionMultiHeadedAttention
    from fairseq.modules.conformer_layer import ConformerEncoderLayer
    from fairseq.models.speech_to_speech.modules.stacked_embedding import StackedEmbedding
    from fairseq.models.speech_to_speech.modules.transformer_encoder import TransformerEncoderNoEmb
    from fairseq.modules.positional_encoding import RelPositionalEncoding
    import fairseq.utils as futils

    conv = load_file_module("_ref_s2t_convolution", REF + "/fairseq/fairseq/models/speech_to_text/modules/convolution.py")
    td = load_file_module("fairseq.models.transformer.transformer_decoder", REF + "/fairseq/fairseq/models/transformer/transformer_decoder.py")
    from fairseq.models.fairseq_encoder import FairseqEncoder

    def _lengths_to_padding_mask(lens):
        return torch.arange(int(lens.max())).view(1, -1) >= lens.view(-1, 1)

    s2t_reorder = extract_functions(REF + "/fairseq/fairseq/models/speech_to_text/s2t_transformer.py", "S2TTransformerEncoder",
                                    ["reorder_encoder_out"], {"torch": torch, "Dict": Dict, "List": List})
    S2TConformerEncoder = extract_class(REF + "/fairseq/fairseq/models/speech_to_text/s2t_conformer.py", "S2TConformerEncoder", {
        "torch": torch, "math": math, "FairseqEncoder": FairseqEncoder, "Conv1dSubsampler": conv.Conv1dSubsampler,
        "Conv2dSubsampler": conv.Conv2dSubsampler, "RelPositionalEncoding": RelPositionalEncoding, "PositionalEmbedding": None,
        "ConformerEncoderLayer": ConformerEncoderLayer, "lengths_to_padding_mask": _lengths_to_padding_mask,
        "logger": types.SimpleNamespace(info=lambda *a, **k: None),
        "S2TTransformerEncoder": types.SimpleNamespace(reorder_encoder_out=s2t_reorder["reorder_encoder_out"])})
    TransformerUnitDecoder = extract_class(REF + "/fairseq/fairseq/models/speech_to_speech/s2s_transformer.py", "TransformerUnitDecoder", {
        "TransformerDecoder": td.TransformerDecoderBase, "Linear": lambda i, o, bias=True: nn.Linear(i, o, bias), "Optional": Optional,
        "Dict": Dict, "List": List, "Any": Any, "Tensor": torch.Tensor, "torch": torch, "utils": futils})
    unity = load_file_module("examples.speech_to_speech.unity.sequence_generator",
                             REF + "/fairseq/examples/speech_to_speech/unity/sequence_generator.py")
    for name in ("examples", "examples.speech_to_speech", "examples.speech_to_speech.unity"):
        m = sys.modules.setdefault(name, types.ModuleType(name))
        m.__path__ = []
    sys.modules["examples.speech_to_speech.unity"].sequence_generator = unity
    sys.modules["examples.speech_to_speech.unity.sequence_generator"] = unity
    mdsg = load_file_module("_ref_sequence_generator_multi_decoder", REF + "/researches/translatotron/sequence_generator_multi_decoder.py")
    return dict(search=search, S2TConformerEncoder=S2TConformerEncoder, TransformerDecoderBase=td.TransformerDecoderBase,
                TransformerEncoderNoEmb=TransformerEncoderNoEmb, TransformerUnitDecoder=TransformerUnitDecoder, StackedEmbedding=StackedEmbedding,
                MultiDecoderSequenceGenerator=mdsg.MultiDecoderSequenceGenerator)


class RefUnitY(nn.Module):
    """The attributes of UnityConformerModelModified that MultiDecoderSequenceGenerator and the unity SequenceGenerator read."""

    mt_task_name = "target_unigram"
    t2u_augmented_cross_attn = False

    def __init__(self, cfg: ModelConfig, sd, R):
        super().__init__()
        NS = types.SimpleNamespace
        eargs = NS(encoder_freezing_updates=0, encoder_embed_dim=cfg.enc_dim, no_scale_embedding=False, conv_version="s2t_transformer",
                   input_feat_per_channel=cfg.feat_dim, input_channels=1, conv_channels=cfg.conv_channels,
                   conv_kernel_sizes=f"{cfg.conv_kernel},{cfg.conv_kernel}", pos_enc_type="rel_pos", max_source_positions=cfg.max_source_positions,
                   dropout=0.1, encoder_ffn_embed_dim=cfg.enc_ffn, encoder_attention_heads=cfg.enc_heads, encoder_layers=cfg.enc_layers,
                   depthwise_conv_kernel_size=cfg.dw_kernel, attn_type="espnet", fp16=False)
        self.encoder = R["S2TConformerEncoder"](eargs)
        self.encoder.load_state_dict(sub_state(sd, "encoder."), strict=True)
        mt_cfg = transformer_cfg(cfg, cfg.enc_dim, cfg.mt_dim, cfg.mt_ffn, cfg.mt_heads, cfg.mt_layers, cfg.max_target_positions)
        mt = R["TransformerDecoderBase"](mt_cfg, FakeDict(cfg.tgt_vocab), nn.Embedding(cfg.tgt_vocab, cfg.mt_dim, padding_idx=cfg.pad))
        _load(mt, sd, "target_unigram_decoder.")
        self.target_unigram_decoder = mt
        t2u_args = NS(**vars(transformer_cfg(cfg, cfg.unit_dim, cfg.unit_dim, cfg.unit_ffn, cfg.unit_heads, cfg.t2u_layers, cfg.max_target_positions)))
        t2u_args.encoder_ffn_embed_dim, t2u_args.encoder_attention_heads, t2u_args.encoder_layers = cfg.unit_ffn, cfg.unit_heads, cfg.t2u_layers
        t2u_args.layernorm_embedding = False
        self.synthesizer_encoder = R["TransformerEncoderNoEmb"](t2u_args)
        self.synthesizer_encoder.load_state_dict(sub_state(sd, "synthesizer_encoder."), strict=True)
        u_cfg = transformer_cfg(cfg, cfg.unit_dim, cfg.unit_dim, cfg.unit_ffn, cfg.unit_heads, cfg.unit_layers, cfg.max_target_positions)
        emb = R["StackedEmbedding"](cfg.unit_vocab, cfg.unit_dim, cfg.pad, num_stacked=1)
        self.decoder = R["TransformerUnitDecoder"](u_cfg, FakeDict(cfg.unit_vocab), emb)
        _load(self.decoder, sd, "decoder.")

    def max_decoder_positions(self):  # FairseqEncoderDecoderModel: the unit decoder's max_positions()
        return self.decoder.max_positions()

    def get_normalized_probs(self, net_output, log_probs, sample=None):
        logits = net_output[0].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)


def _load(m, sd, prefix):
    """load_state_dict of a decoder whose `version` buffer and tied output projection are extra or shared; every key must land"""
    sub = sub_state(sd, prefix)
    assert set(sub) <= set(m.state_dict()), sorted(set(sub) - set(m.state_dict()))[:5]
    m.load_state_dict(sub, strict=False)
    for k, v in sub.items():
        assert torch.equal(m.state_dict()[k], v), k


def main():
    assert ref_loader.available(), "reference tree missing"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    R = load_reference_classes()
    import fairseq.utils as futils

    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    gcmvn = synth.make_gcmvn(cfg)
    model = RefUnitY(cfg, sd, R).eval()
    oracle = UnitYOracle(cfg, sd, torch.float32)
    q = [np.round(online_features(synth.make_audio(d, seed=300 + i), None).numpy() * RAW_SCALE).astype(np.int16) for i, d in enumerate(DURATIONS)]
    raw = [x.astype(np.float32) / np.float32(RAW_SCALE) for x in q]
    feats = [G.apply_cmvn(r, (gcmvn["mean"], gcmvn["std"])).astype(np.float32) for r in raw]
    n_frames = [int(f.shape[0]) for f in raw]
    gold = {f"raw_{i}": x for i, x in enumerate(q)}
    gold.update(gcmvn_mean=gcmvn["mean"], gcmvn_std=gcmvn["std"], raw_scale=np.array(RAW_SCALE), n_frames=np.array(n_frames),
                npy_samples=np.array(NPY_SAMPLES), tgt_n_frames=np.zeros(len(DURATIONS), dtype=np.int64),
                settings=np.array(SETTINGS), max_len_b_mt=np.array(MAX_LEN_B_MT))
    fns = extract_functions(REF + "/fairseq/fairseq/data/dictionary.py", "Dictionary", ["string", "unk_string"],
                            {"torch": torch, "utils": futils, "data_utils": types.SimpleNamespace(post_process=lambda s, b: s)})

    class RefDict(Dictionary):  # Dictionary.string / unk_string from their own source
        unk_word = "<unk>"
        string = fns["string"]
        unk_string = fns["unk_string"]

    rd = RefDict([str(i) for i in range(cfg.unit_vocab - 4)])
    tdict = Dictionary.synthetic(cfg.tgt_vocab)
    early = forced = ragged = 0
    for k, (max_tokens, beam_mt, max_len_b) in enumerate(SETTINGS):
        batches = G.make_batches(n_frames, [0] * len(n_frames), max_tokens, None, 1, (6000, 1024), False)
        gen = R["MultiDecoderSequenceGenerator"]([model], rd, tdict, beam_size=1, beam_size_mt=beam_mt, max_len_a=1, max_len_b=max_len_b,
                                                 max_len_a_mt=0, max_len_b_mt=MAX_LEN_B_MT, min_len=1, normalize_scores=True, len_penalty=1.0,
                                                 unk_penalty=0.0, temperature=1.0, match_source_len=False, no_repeat_ngram_size=0)
        stdout, lines = [], []
        for bi, batch in enumerate(batches):
            lens = torch.tensor([n_frames[i] for i in batch])
            x = torch.zeros(len(batch), int(lens.max()), cfg.feat_dim)
            for b, i in enumerate(batch):
                x[b, :n_frames[i]] = torch.from_numpy(feats[i])
            sample = {"id": torch.tensor(batch), "net_input": {"src_tokens": x, "src_lengths": lens}}
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                fin = gen.generate([model], sample)
            stdout += buf.getvalue().splitlines()
            mine = unity_generate(oracle, x, lens.tolist(), beam_mt, 1.0, max_len_b, MAX_LEN_B_MT)
            ragged |= len(batch) > 1 and len({len(h) for h in mine["mt_hyps"]}) > 1
            for b, i in enumerate(batch):
                h = fin[b][0]
                units = h["tokens"].tolist()
                m = mine["units"][b]
                assert units == m["tokens"], (k, bi, b, units[:12], m["tokens"][:12])
                assert abs(float(h["score"]) - m["score"]) < 1e-5, (k, bi, b)
                # positional scores are differences of fp32 cumulative scores: about one ulp of the cumulative sum each
                bar = 1e-5 + 2.4e-7 * abs(m["score"]) * len(units)
                assert np.abs(h["positional_scores"].numpy() - np.array(m["positional_scores"])).max() < bar, (k, bi, b)
                early += len(units) < mine["max_len"] + 1
                forced += len(units) == mine["max_len"] + 1
                hypo_str = rd.string(torch.tensor(units), None, extra_symbols_to_ignore={rd.eos()})
                target_str = rd.string(torch.tensor([rd.eos()]), None, escape_unk=True, extra_symbols_to_ignore={rd.eos()})
                score = h["score"] / math.log(2)
                pos = h["positional_scores"].clone().div_(math.log(2)).tolist()
                lines += ["T-{}\t{}".format(i, target_str), "H-{}\t{}\t{}".format(i, score, hypo_str), "D-{}\t{}\t{}".format(i, score, hypo_str),
                          "P-{}\t{}".format(i, " ".join(map(lambda v: "{:.4f}".format(v), pos)))]
                gold[f"s{k}_units_{i}"] = np.array(units, dtype=np.int64)
                gold[f"s{k}_score_{i}"] = np.array(float(h["score"]))
                gold[f"s{k}_positional_{i}"] = h["positional_scores"].numpy().astype(np.float32)
            mt_text = [ln for ln in buf.getvalue().splitlines()]
            assert mt_text == ["D-{}\t{}".format(i, G.ctc_text(tdict, h)) for i, h in zip(batch, mine["mt_hyps"])], (k, bi)
            print(f"setting {k}: batch {bi} samples {batch} F {int(lens.max())} unit lengths {[len(fin[b][0]['tokens']) for b in range(len(batch))]}")
        gold[f"s{k}_stdout"] = np.array(stdout)
        gold[f"s{k}_file_lines"] = np.array(lines)
        gold[f"s{k}_n_batches"] = np.array(len(batches))
    assert forced and ragged, (early, forced, ragged)
    gold["n_early_eos"], gold["n_forced_eos"] = np.array(early), np.array(forced)
    path = os.path.join(GOLD, "unity_generate.npz")
    np.savez_compressed(path, **gold)
    print("wrote", path, os.path.getsize(path), "bytes;", early, "early eos,", forced, "forced eos")


if __name__ == "__main__":
    main()
