"""Generate tests/golden/unity_variants.npz from the reference's own Uni-UnitY and Chunk-UnitY code (build container only, CPU).

Run:  python -m oracle.gen_golden_unity_variants      (needs /root/reference)

The model object is oracle.gen_golden_unity's RefUnitY (fairseq's MT decoder and TransformerUnitDecoder, which the uni_unity and
chunk_unity models also build: their own transformer_decoder.py differs only by a training-time streaming_config that inference
never passes) with the seeded synthetic state dict of synth.make_unity_checkpoint(variant) and the variant's own modules in place of
the encoder and the T2U encoder, every module loaded strictly:

  uni_unity    UniS2TConformerEncoder (researches/uni_unity/models/s2t_conformer.py, run from its own class body) with uni_unity's
               Conv1dSubsampler and UniConformerEncoderLayer, --uni-encoder; uni_unity's UniTransformerEncoderNoEmb (causal)
  chunk_unity  ChunkS2TConformerEncoder (oracle.gen_golden.build_reference_encoder: chunk_unity's own _forward and
               buffered_chunk_mask over ChunkConformerEncoderLayer and chunk_unity's Conv1dSubsampler) at --chunk-size 8, the
               training value for the attention mask and the convolutions; uni_unity's UniTransformerEncoderNoEmb (causal)

Fixtures:
  generate     researches/uni_unity/test_scripts/pred.sh on Uni-UnitY: `fairseq-generate --user-dir researches/uni_unity --task
               speech_to_speech_modified`, whose task inherits fairseq's build_generator_dual_decoder (fairseq/tasks/
               speech_to_speech.py): examples/speech_to_speech/unity/sequence_generator_multi_decoder.py and its SequenceGenerator,
               imported unchanged.  The split and batching are gen_golden_unity's; GEN_SETTINGS below.  Recorded: the MT prints
               ("{text} (None-{id})"), the results-file lines and every sample's units, positional scores and score
  waitk        both wait-k agents' policy() / reset() from their own source (oracle.gen_golden_waitk.run_setting) on each model
               with the settings of tests/golden/waitk_policy.npz; one waveform (WAV_KEPT), the sample count of every write

Before writing, oracle.unity_variant_oracle (float32) must reproduce every print, unit, score and wait-k action.
"""
from __future__ import annotations

import contextlib
import io
import math
import os
import sys
import types
from typing import Dict, List

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden_waitk as W  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import GOLD, REF, extract_class, extract_functions, sub_state, transformer_cfg  # noqa: E402
from oracle.gen_golden import build_reference_encoder  # noqa: E402
from oracle.gen_golden_agent import load_file_module  # noqa: E402
from oracle.gen_golden_unity import DURATIONS, MAX_LEN_B_MT, RAW_SCALE, RefUnitY, load_reference_classes  # noqa: E402
from oracle.streamspeech_oracle import online_features  # noqa: E402
from oracle.unity_oracle import unity_generate  # noqa: E402
from oracle.unity_variant_oracle import VariantUnitYOracle, VariantWaitkS2STAgent, VariantWaitkS2TTAgent  # noqa: E402
from streamspeech_b200 import generate as G  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402

GEN_SETTINGS = [(900, 1, 200), (10000, 4, 10), (700, 4, 40)]  # (--max-tokens, --beam-mt, --max-len-b), as gen_golden_unity
VARIANTS = ("uni_unity", "chunk_unity")
# The one wait-k waveform stored: the first WRITE of this setting.  A waveform is the vocoder's on the call's units and durations, which
# every call stores exactly, and the vocoder is the same for every model of the family (pinned to the reference's CodeGenerator by
# waitk_policy.npz and vocoder.npz); every other WRITE stores its sample count, and the tests recompute its samples with the float32
# oracle's vocoder, which run_setting has just asserted within 1e-5 of the reference's on every call.
WAV_KEPT = ("uni_unity", "s2st_default")


def variant_encoders(cfg: ModelConfig, sd):
    """(encoder, T2U encoder) of the variant from the reference's own modules, loaded strictly"""
    ref_loader.load_full()
    from uni_unity.modules.transformer_encoder import UniTransformerEncoderNoEmb

    NS = types.SimpleNamespace
    t2u_args = NS(**vars(transformer_cfg(cfg, cfg.unit_dim, cfg.unit_dim, cfg.unit_ffn, cfg.unit_heads, cfg.t2u_layers, cfg.max_target_positions)))
    t2u_args.encoder_ffn_embed_dim, t2u_args.encoder_attention_heads, t2u_args.encoder_layers = cfg.unit_ffn, cfg.unit_heads, cfg.t2u_layers
    t2u_args.uni_encoder = cfg.uni_encoder
    t2u = UniTransformerEncoderNoEmb(t2u_args)
    t2u.load_state_dict(sub_state(sd, "synthesizer_encoder."), strict=True)
    if cfg.unity_variant == "chunk_unity":
        return build_reference_encoder(cfg, sd, cfg.chunk_size, cfg.chunk_size), t2u.eval()
    from uni_unity.modules.conformer_layer import UniConformerEncoderLayer
    from uni_unity.modules.convolution import Conv1dSubsampler
    from fairseq.models.fairseq_encoder import FairseqEncoder
    from fairseq.modules.positional_encoding import RelPositionalEncoding
    import fairseq.utils as futils

    reorder = extract_functions(REF + "/fairseq/fairseq/models/speech_to_text/s2t_transformer.py", "S2TTransformerEncoder",
                                ["reorder_encoder_out"], {"torch": torch, "Dict": Dict, "List": List})
    Enc = extract_class(REF + "/researches/uni_unity/models/s2t_conformer.py", "UniS2TConformerEncoder", {
        "torch": torch, "math": math, "FairseqEncoder": FairseqEncoder, "Conv1dSubsampler": Conv1dSubsampler, "Conv2dSubsampler": None,
        "RelPositionalEncoding": RelPositionalEncoding, "PositionalEmbedding": None, "UniConformerEncoderLayer": UniConformerEncoderLayer,
        "lengths_to_padding_mask": lambda lens: torch.arange(int(lens.max())).view(1, -1) >= lens.view(-1, 1), "utils": futils,
        "logger": types.SimpleNamespace(info=lambda *a, **k: None),
        "S2TTransformerEncoder": types.SimpleNamespace(reorder_encoder_out=reorder["reorder_encoder_out"])})
    eargs = NS(encoder_freezing_updates=0, encoder_embed_dim=cfg.enc_dim, no_scale_embedding=False, conv_version="s2t_transformer",
               input_feat_per_channel=cfg.feat_dim, input_channels=1, conv_channels=cfg.conv_channels,
               conv_kernel_sizes=f"{cfg.conv_kernel},{cfg.conv_kernel}", pos_enc_type="rel_pos", max_source_positions=cfg.max_source_positions,
               dropout=0.1, encoder_ffn_embed_dim=cfg.enc_ffn, encoder_attention_heads=cfg.enc_heads, encoder_layers=cfg.enc_layers,
               depthwise_conv_kernel_size=cfg.dw_kernel, attn_type="espnet", fp16=False, uni_encoder=cfg.uni_encoder)
    enc = Enc(eargs)
    enc.load_state_dict(sub_state(sd, "encoder."), strict=True)
    return enc.eval(), t2u.eval()


def chunk_encoder_class():
    """ChunkS2TConformerEncoder's forward (its _forward) and reorder_encoder_out (S2TTransformerEncoder's) around
    oracle.gen_golden.build_reference_encoder's module, as a FairseqEncoder the generators call"""
    from fairseq.models.fairseq_encoder import FairseqEncoder

    reorder = extract_functions(REF + "/fairseq/fairseq/models/speech_to_text/s2t_transformer.py", "S2TTransformerEncoder",
                                ["reorder_encoder_out"], {"torch": torch, "Dict": Dict, "List": List})

    class ChunkEncoder(FairseqEncoder):
        def __init__(self, enc):
            super().__init__(None)
            self.enc = enc

        def forward(self, src_tokens, src_lengths, return_all_hiddens=False):
            return self.enc._forward(src_tokens, src_lengths, return_all_hiddens)

        reorder_encoder_out = reorder["reorder_encoder_out"]

    return ChunkEncoder


def build_model(variant: str, R):
    state = synth.make_unity_checkpoint(variant, seed=0)
    cfg = ModelConfig.from_checkpoint(state)
    sd = state["model"]
    model = RefUnitY(ModelConfig.unity_default(), sd, R)  # MT decoder, unit decoder (and UnitY's modules, replaced below)
    enc, t2u = variant_encoders(cfg, sd)
    model.encoder = enc if variant == "uni_unity" else chunk_encoder_class()(enc)
    model.synthesizer_encoder = t2u
    return cfg, sd, model.eval()


def fairseq_generator_class():
    """fairseq's own MultiDecoderSequenceGenerator (examples/speech_to_speech/unity), over the unity SequenceGenerator that
    load_reference_classes registered"""
    return load_file_module("_ref_fairseq_sequence_generator_multi_decoder",
                            REF + "/fairseq/examples/speech_to_speech/unity/sequence_generator_multi_decoder.py").MultiDecoderSequenceGenerator


def run_generate(cfg, sd, model, gold, report):
    import fairseq.utils as futils

    MDSG = fairseq_generator_class()
    oracle = VariantUnitYOracle(cfg, sd, torch.float32)
    gcmvn = synth.make_gcmvn(cfg)
    q = [np.round(online_features(synth.make_audio(d, seed=300 + i), None).numpy() * RAW_SCALE).astype(np.int16) for i, d in enumerate(DURATIONS)]
    raw = [x.astype(np.float32) / np.float32(RAW_SCALE) for x in q]
    feats = [G.apply_cmvn(r, (gcmvn["mean"], gcmvn["std"])).astype(np.float32) for r in raw]
    n_frames = [int(f.shape[0]) for f in raw]
    fns = extract_functions(REF + "/fairseq/fairseq/data/dictionary.py", "Dictionary", ["string", "unk_string"],
                            {"torch": torch, "utils": futils, "data_utils": types.SimpleNamespace(post_process=lambda s, b: s)})

    class RefDict(Dictionary):
        unk_word = "<unk>"
        string = fns["string"]
        unk_string = fns["unk_string"]

    rd = RefDict([str(i) for i in range(cfg.unit_vocab - 4)])
    tdict = Dictionary.synthetic(cfg.tgt_vocab)
    gold["gen_settings"] = np.array(GEN_SETTINGS)
    gold["gen_max_len_b_mt"] = np.array(MAX_LEN_B_MT)
    gold["gen_n_frames"] = np.array(n_frames)
    early = forced = 0
    for k, (max_tokens, beam_mt, max_len_b) in enumerate(GEN_SETTINGS):
        batches = G.make_batches(n_frames, [0] * len(n_frames), max_tokens, None, 1, (6000, 1024), False)
        gen = MDSG([model], rd, tdict, beam_size=1, beam_size_mt=beam_mt, max_len_a=1, max_len_b=max_len_b, max_len_a_mt=0,
                   max_len_b_mt=MAX_LEN_B_MT, min_len=1, normalize_scores=True, len_penalty=1.0, unk_penalty=0.0, temperature=1.0,
                   match_source_len=False, no_repeat_ngram_size=0)
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
            assert buf.getvalue().splitlines() == [G.mt_print_line(cfg, i, G.ctc_text(tdict, h)) for i, h in zip(batch, mine["mt_hyps"])], (k, bi)
            for b, i in enumerate(batch):
                h = fin[b][0]
                units = h["tokens"].tolist()
                m = mine["units"][b]
                assert units == m["tokens"], (k, bi, b, units[:12], m["tokens"][:12])
                assert abs(float(h["score"]) - m["score"]) < 1e-5, (k, bi, b)
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
                gold[f"gen{k}_units_{i}"] = np.array(units, dtype=np.int64)
                gold[f"gen{k}_score_{i}"] = np.array(float(h["score"]))
                gold[f"gen{k}_positional_{i}"] = h["positional_scores"].numpy().astype(np.float32)
        gold[f"gen{k}_stdout"] = np.array(stdout)
        gold[f"gen{k}_file_lines"] = np.array(lines)
        gold[f"gen{k}_n_batches"] = np.array(len(batches))
    assert forced, (early, forced)
    report["generate"] = f"{early} early eos, {forced} forced eos"
    # the split is tests/golden/unity_generate.npz's (the same durations, seeds and quantisation): its checksums, not a second copy
    gold["gen_raw_sums"] = np.array([[int(x.astype(np.int64).sum()), int((x.astype(np.int64) ** 2).sum())] for x in q], dtype=np.int64)
    gold["gen_raw_scale"] = np.array(RAW_SCALE)


def run_waitk(variant, cfg, sd, model, gold, report, R):
    gcmvn = synth.make_gcmvn(cfg)
    vsd_wn = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True)
    W.OracleWaitkS2STAgent, W.OracleWaitkS2TTAgent = VariantWaitkS2STAgent, VariantWaitkS2TTAgent  # run_setting's oracle classes
    for s in W.SETTINGS:
        out = W.run_setting(s, model, cfg, sd, gcmvn, vsd_wn, R, report)  # asserts the oracle's waveform within 1e-5 of the reference's
        # the samples are the vocoder's on the stored units and durations: their count pins the tail window
        writes = sorted((k for k in out if k.endswith("_wav")), key=lambda k: int(k[len("call"):-len("_wav")]))
        for k in writes[1 if (variant, s[0]) == WAV_KEPT else 0:]:
            out[k[:-len("_wav")] + "_wav_n"] = np.array(len(out.pop(k)))
        gold.update({f"{variant}_{s[0]}_{k}": v for k, v in out.items()})
        report[f"{variant} {s[0]}"] = report.pop(s[0])


def main():
    assert ref_loader.available(), "reference tree missing"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    R = load_reference_classes()
    report, gold = {}, {"variants": np.array(VARIANTS), "waitk_tags": np.array([s[0] for s in W.SETTINGS])}
    for variant in VARIANTS:
        cfg, sd, model = build_model(variant, R)
        if variant == "uni_unity":
            run_generate(cfg, sd, model, gold, report)
        run_waitk(variant, cfg, sd, model, gold, report, R)
    path = os.path.join(GOLD, "unity_variants.npz")
    np.savez_compressed(path, **gold)
    for k, v in report.items():
        print(f"{k:28s} {v}")
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
