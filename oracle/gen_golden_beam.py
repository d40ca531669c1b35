"""Generate tests/golden/mt_beam.npz from the reference's own beam search (build container only, CPU).

Run:  python -m oracle.gen_golden_beam        (needs /root/reference)

The reference's unity `SequenceGenerator` (fairseq/examples/speech_to_speech/unity/sequence_generator.py, imported unchanged
from its file on top of the unchanged fairseq.sequence_generator / fairseq.search that oracle.gen_golden_agent loads) runs
`generate_decoder` with BeamSearch at beam K on the reference MT decoder (TransformerDecoderBase with incremental states), as
tasks/speech_to_speech_ctc.py:21-49 builds the offline MT generator (beam_size_mt = K, len_penalty = --lenpen, max_len_a 0,
min_len 1, normalize_scores), on the reference encoder's output for a padded batch of four short utterances of the seeded
synthetic offline checkpoint.  For K in {2, 5} and len_penalty in {1.0, 0.6} it asserts that

  - oracle.mt_beam_oracle.mt_beam in float32 returns the reference's n-best of every sample: same tokens, same order, scores
    and positional scores within 1e-5;
  - the float64 restatement selects the same hypotheses (its smallest score gap at a selection boundary is stored as
    margin_k{K}_lp{L}, to diagnose a later failure);
  - the batch covers a sample whose best beam hypothesis differs from its greedy one, and hypotheses finalized at the forced
    eos of max_len.

The synthetic checkpoint's MT distributions are nearly flat (about -8.3 nats per token against log(1/6000) = -8.7) and its
eos rises only after ~30 tokens, where the float64 margins at the selection boundaries shrink to a few ulp of the cumulative
scores; MAX_LEN_B_MT = 8 keeps its decisions at least 6e-5 apart in float64, and every hypothesis there ends at the forced eos.
A second set of cases ("early_", max_len_b EARLY_MAX_LEN_B) runs the same search on the checkpoint with eos's output row
scaled by EOS_ROW_SCALE (oracle.mt_beam_oracle.early_eos_state_dict; the encoder is untouched, so the same encoder rows
apply): there eos ranks among the best candidates after a few tokens, and the script asserts that some sample finalizes
hypotheses before max_len while it searches on and finalizes a longer one later (hypothesis lengths [2, 2, 2, 2, 9] and
[2, 2, 2, 9, 9] at K = 5: four or three finalized at step 1, the rest at step 8 < max_len).  Those cases run the slot offset of
hypotheses finalized at a later step, the skipping of finite eos candidates when the new beams are chosen, positional scores
from reordered histories, and the length normalization over hypotheses of different lengths.  Their hypotheses come out in
finalization order under both len_penalty values (scales -0.05 .. -0.3 gave no sample where a later, longer hypothesis
outranks an earlier one).  The fixture stores each sample's reference encoder rows, so that the GPU test isolates the search.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import GOLD, REF, build_reference_decoders, build_reference_encoder  # noqa: E402
from oracle.gen_golden_agent import FakeStreamSpeechModel, load_file_module, load_reference_generators  # noqa: E402
from oracle.mt_beam_oracle import early_eos_state_dict, mt_beam  # noqa: E402
from oracle.streamspeech_oracle import StreamSpeechOracle, online_features  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402

SECONDS = (0.9, 0.5, 1.3, 0.7)
SEEDS = (41, 42, 43, 44)
MAX_LEN_B_MT = 8
EOS_ROW_SCALE = -0.2
EARLY_MAX_LEN_B = 12
BEAMS = (2, 5)
LEN_PENALTIES = (1.0, 0.6)


def offline_cfg() -> ModelConfig:
    cfg = ModelConfig()
    cfg.uni_encoder = False
    return cfg


def main():
    assert ref_loader.available(), "reference tree missing"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    cfg = offline_cfg()
    sd = synth.make_model_state_dict(cfg, seed=0)
    gcmvn = synth.make_gcmvn(cfg)
    fl = [online_features(synth.make_audio(s, seed=k), gcmvn) for s, k in zip(SECONDS, SEEDS)]
    lens = torch.tensor([f.size(0) for f in fl])
    feats = torch.zeros(len(fl), int(lens.max()), cfg.feat_dim)
    for b, f in enumerate(fl):
        feats[b, : f.size(0)] = f
    B = len(fl)

    search, _ = load_reference_generators()
    unity = load_file_module("_ref_unity_sequence_generator", REF + "/fairseq/examples/speech_to_speech/unity/sequence_generator.py")
    enc = build_reference_encoder(cfg, sd, None, None)
    d = Dictionary.synthetic(cfg.tgt_vocab)
    enc_out = enc._forward(feats, lens)
    eo = enc_out["encoder_out"][0]  # [T, B, C]
    pad = enc_out["encoder_padding_mask"][0] if enc_out["encoder_padding_mask"] else None
    T_b = [int(eo.size(0) - pad[b].sum()) if pad is not None else eo.size(0) for b in range(B)]
    gold = {"enc_lengths": np.array(T_b, dtype=np.int32), "max_len_b_mt": np.array(MAX_LEN_B_MT), "beams": np.array(BEAMS),
            "len_penalties": np.array(LEN_PENALTIES, dtype=np.float64), "eos_row_scale": np.array(EOS_ROW_SCALE),
            "early_max_len_b_mt": np.array(EARLY_MAX_LEN_B)}
    for b in range(B):
        gold[f"enc_{b}"] = eo[: T_b[b], b].numpy()

    src = torch.zeros(B, eo.size(0) * 4, cfg.feat_dim)
    sample = {"id": torch.arange(B), "net_input": {"src_tokens": src, "src_lengths": lens}}

    def run_cases(model_sd, prefix, max_len_b):
        """the reference's n-best for every (K, len_penalty) on model_sd, pinned to the restatements; per-sample lengths"""
        model = FakeStreamSpeechModel(enc, build_reference_decoders(cfg, model_sd)).eval()
        o32 = StreamSpeechOracle(cfg, model_sd, None, gcmvn, chunk_size=None, conv_chunk_size=None)
        o64 = StreamSpeechOracle(cfg, model_sd, None, gcmvn, chunk_size=None, conv_chunk_size=None, dtype=torch.float64)
        out = {}
        for K in BEAMS:
            for lp in LEN_PENALTIES:
                gen = unity.SequenceGenerator([model], d, beam_size=K, max_len_a=0, max_len_b=max_len_b, max_len=0, min_len=1,
                                              normalize_scores=True, len_penalty=lp, unk_penalty=0.0, temperature=1.0,
                                              match_source_len=False, no_repeat_ngram_size=0, search_strategy=search.BeamSearch(d),
                                              eos=d.eos(), symbols_to_strip_from_output=None)
                fin = gen.generate_decoder([enc_out], src, lens, sample, None, None, None, aux_task_name="target_unigram")
                margin = np.inf
                tag = f"{prefix}k{K}_lp{lp}"
                for b in range(B):
                    ref = fin[b]
                    assert len(ref) == K, (tag, b, len(ref))
                    mine = mt_beam(o32, eo[: T_b[b], b:b + 1], K, max_len_b, lp)
                    hi = mt_beam(o64, eo[: T_b[b], b:b + 1], K, max_len_b, lp)
                    margin = min(margin, hi["margin"])
                    for i, (r, m, h) in enumerate(zip(ref, mine["hyps"], hi["hyps"])):
                        rt = r["tokens"].tolist()
                        assert rt == m["tokens"], (tag, b, i, rt, m["tokens"])
                        assert rt == h["tokens"], (tag, b, i, "float64", rt, h["tokens"])
                        assert abs(float(r["score"]) - m["score"]) < 1e-5, (tag, b, i)
                        assert np.abs(r["positional_scores"].numpy() - np.array(m["positional_scores"])).max() < 1e-5, (tag, b, i)
                        gold[f"{tag}_tokens_{b}_{i}"] = np.array(rt, dtype=np.int64)
                        gold[f"{tag}_score_{b}_{i}"] = np.array(float(r["score"]), dtype=np.float32)
                        gold[f"{tag}_pos_{b}_{i}"] = r["positional_scores"].numpy().astype(np.float32)
                    out[(K, lp, b)] = [r["tokens"].tolist() for r in ref]
                    print(tag, b, "lengths", [len(r["tokens"]) for r in ref], "scores", [round(float(r["score"]), 4) for r in ref])
                gold[f"margin_{tag}"] = np.array(margin)
                print(tag, "float64 margin", margin)
        return out

    o32 = StreamSpeechOracle(cfg, sd, None, gcmvn, chunk_size=None, conv_chunk_size=None)
    greedy = [o32.mt_greedy(eo[: T_b[b], b:b + 1], None, -1, max_len_b=MAX_LEN_B_MT) for b in range(B)]
    plain = run_cases(sd, "", MAX_LEN_B_MT)
    differs_from_greedy = any(h[0] != greedy[b] for (_, _, b), h in plain.items())
    forced = any(len(t) == MAX_LEN_B_MT + 1 for h in plain.values() for t in h)
    early_sd = early_eos_state_dict(sd, cfg.eos, EOS_ROW_SCALE)
    ear = run_cases(early_sd, "early_", EARLY_MAX_LEN_B)
    # finalized before max_len while the sample searched on: a shorter hypothesis next to a longer one of the same sample
    early = any(min(map(len, h)) < max(map(len, h)) < EARLY_MAX_LEN_B + 1 for h in ear.values())
    print("coverage: differs from greedy", differs_from_greedy, "forced eos", forced, "early", early)
    assert differs_from_greedy, "no sample's best beam hypothesis differs from greedy: pick other seeds"
    assert forced, "no hypothesis finalized at the forced eos: pick other seeds"
    assert early, "no sample finalized hypotheses at two steps before max_len: pick another EOS_ROW_SCALE"
    np.savez_compressed(os.path.join(GOLD, "mt_beam.npz"), **gold)
    print("wrote", os.path.join(GOLD, "mt_beam.npz"), os.path.getsize(os.path.join(GOLD, "mt_beam.npz")), "bytes")


if __name__ == "__main__":
    main()
