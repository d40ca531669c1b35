"""Generate tests/golden/offline_generate.npz from the REAL reference code (build container only, CPU, a few minutes).

Run:  python -m oracle.build_ref_ext && python -m oracle.gen_golden_generate      (needs /root/reference)

The fixture of `python -m streamspeech_b200.generate` (fairseq-generate --task speech_to_speech_ctc on a data split):

  split       ten synthetic utterances of 1-4.5 s (synth.make_audio), two of them of equal length; raw fbank (the oracle's Kaldi
              fbank, rounded to steps of 1/32 so that the fixture stays small) and the SHA-256 of the fp32 features after GlobalCMVN,
              run from its own source (feature_transforms/global_cmvn.py) with the synthetic gcmvn stats
  batching    SpeechToTextDataset.ordered_indices from its own source, data_utils.batch_by_size from its own source over
              batch_by_size_vec compiled from data_utils_fast.pyx (oracle/build_ref_ext.py), the collater's torch.sort, at several
              --max-tokens / --batch-size / --required-batch-size-multiple settings
  BLEU        fairseq's bleu Scorer from its own source over clib/libbleu (ctypes), on random unit sequences with unks and pads
  generation  per batch of the --max-tokens setting the tests run: the reference modules chained as in gen_golden_offline.py,
              ending in the reference CTCSequenceGenerator.generate, whose positional_scores and score are kept; the unit strings
              from fairseq's Dictionary.string; the lines with generate.py's format strings

and asserts that oracle/offline_oracle.py reproduces every batch's prints and units before writing the fixture.
"""
from __future__ import annotations

import ctypes
import hashlib
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import (FakeDict, GOLD, REF, build_reference_decoders, build_reference_encoder, extract_class,  # noqa: E402
                               extract_functions)
from oracle.offline_oracle import offline_generate  # noqa: E402
from oracle.streamspeech_oracle import StreamSpeechOracle, online_features  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402

DURATIONS = [2.0, 4.5, 3.0, 1.0, 1.8, 3.5, 1.2, 3.0, 2.6, 1.5]  # manifest order; #2 and #7 have equal n_frames
NPY_SAMPLES = (0, 3, 5, 8)                                      # stored as .npy, the others in one zip
MAX_TOKENS = 900                                                # the front door's run: 4 batches of 2, 3, 4 and 1 samples
MAX_LEN_B_MT = 60
RAW_SCALE = 32                                                  # raw fbank in steps of 1/32 (int16 counts in the fixture)
BATCH_SETTINGS = [(900, -1, 1), (1200, -1, 1), (10000, -1, 1), (800, -1, 1), (-1, 3, 1), (1500, -1, 2), (2000, 4, 3), (-1, 4, 8), (1000, 2, 1)]


def offline_cfg() -> ModelConfig:
    cfg = ModelConfig()
    cfg.uni_encoder = False
    return cfg


def reference_batching(n_frames, settings):
    """ordered_indices + batch_by_size (+ batch_by_size_vec compiled from its .pyx) + the collater's sort, from the reference"""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import data_utils_fast  # noqa: E402  (oracle/build_ref_ext.py)

    fq = REF + "/fairseq/fairseq"
    ordered = extract_functions(fq + "/data/audio/speech_to_text_dataset.py", "SpeechToTextDataset", ["ordered_indices"], {"np": np})
    class _DS:
        shuffle = False

        def __init__(self):
            self.n_frames = list(n_frames)

        def __len__(self):
            return len(self.n_frames)

    order = ordered["ordered_indices"](_DS())
    import ast

    src = open(fq + "/data/data_utils.py").read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "batch_by_size"][0]
    pkg = types.ModuleType("fairseq.data")
    pkg.data_utils_fast = data_utils_fast
    saved = {k: sys.modules.get(k) for k in ("fairseq.data", "fairseq.data.data_utils_fast")}
    sys.modules["fairseq.data"], sys.modules["fairseq.data.data_utils_fast"] = pkg, data_utils_fast
    ns = {"np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "data_utils.py:batch_by_size", "exec"), ns)
    out = {}
    try:
        for mt, bs, mult in settings:
            nt = np.array([n_frames[i] for i in order], dtype=np.int64)
            batches = ns["batch_by_size"](order.astype(np.int64), None, num_tokens_vec=nt, max_tokens=mt if mt > 0 else None,
                                          max_sentences=bs if bs > 0 else None, required_batch_size_multiple=mult)
            coll = []
            for b in batches:
                nf = torch.tensor([n_frames[i] for i in b], dtype=torch.long)
                _, o = nf.sort(descending=True)  # the collater (speech_to_speech_dataset.py)
                coll.append(torch.tensor(b, dtype=torch.long).index_select(0, o).tolist())
            out[(mt, bs, mult)] = coll
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return order, out


def reference_bleu(pairs, pad, eos, unk):
    """fairseq's bleu Scorer (scoring/bleu.py) from its own source over clib/libbleu compiled into oracle/_ref/"""
    lib = types.ModuleType("fairseq.libbleu")
    lib.__file__ = os.path.join(ROOT, "oracle", "_ref", "libbleu.so")
    sys.modules["fairseq.libbleu"] = lib
    sys.modules["fairseq"].libbleu = lib
    glb = {"ctypes": ctypes, "math": math, "sys": sys, "torch": torch, "register_scorer": lambda *a, **k: (lambda c: c),
           "BleuConfig": None, "BaseScorer": object}
    BleuStat = extract_class(REF + "/fairseq/fairseq/scoring/bleu.py", "BleuStat", glb)
    glb["BleuStat"] = BleuStat
    Scorer = extract_class(REF + "/fairseq/fairseq/scoring/bleu.py", "Scorer", glb)
    s = Scorer(types.SimpleNamespace(pad=pad, eos=eos, unk=unk))
    for ref, pred in pairs:
        s.add(torch.IntTensor(ref), torch.IntTensor(pred))
    return s.result_string()


def main():
    assert ref_loader.available(), "reference tree missing"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    ref_loader.load_full()
    import fairseq.utils as futils
    from typing import Dict, List, Optional

    cfg = offline_cfg()
    sd = synth.make_model_state_dict(cfg, seed=0)
    gcmvn = synth.make_gcmvn(cfg)
    gold = {}

    # ---- split: raw fbank, then the reference GlobalCMVN
    # raw fbank rounded to multiples of 1/RAW_SCALE and stored as int16 counts (keeps the fixture small); the split holds raw / RAW_SCALE
    # (exact in fp32) as fp32 .npy files
    q = [np.round(online_features(synth.make_audio(d, seed=100 + i), None).numpy() * RAW_SCALE).astype(np.int16) for i, d in enumerate(DURATIONS)]
    raw = [x.astype(np.float32) / np.float32(RAW_SCALE) for x in q]
    n_frames = [int(f.shape[0]) for f in raw]
    assert n_frames[2] == n_frames[7], n_frames
    GlobalCMVN = extract_class(REF + "/fairseq/fairseq/data/audio/feature_transforms/global_cmvn.py", "GlobalCMVN",
                               {"np": np, "AudioFeatureTransform": object, "register_audio_feature_transform": lambda n: (lambda c: c)})
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        np.savez(os.path.join(tmp, "gcmvn.npz"), mean=gcmvn["mean"], std=gcmvn["std"])
        cmvn = GlobalCMVN(os.path.join(tmp, "gcmvn.npz"))
        feats = [torch.from_numpy(cmvn(f)).float().numpy() for f in raw]  # + the dataset's .float()
    for i, (r, f) in enumerate(zip(raw, feats)):
        gold[f"raw_{i}"] = q[i]
        gold[f"feats_sha256_{i}"] = np.array(hashlib.sha256(np.ascontiguousarray(f).tobytes()).hexdigest())
        assert f.dtype == np.float32
    gold["gcmvn_mean"], gold["gcmvn_std"] = gcmvn["mean"], gcmvn["std"]
    gold["raw_scale"] = np.array(RAW_SCALE)
    gold["n_frames"] = np.array(n_frames)
    gold["npy_samples"] = np.array(NPY_SAMPLES)
    rng = np.random.default_rng(5)
    gold["tgt_n_frames"] = rng.integers(20, 300, len(DURATIONS))

    # ---- batching from fairseq's own code
    order, batchings = reference_batching(n_frames, BATCH_SETTINGS)
    gold["ordered_indices"] = np.asarray(order)
    gold["batch_settings"] = np.array(BATCH_SETTINGS)
    for k, (setting, batches) in enumerate(batchings.items()):
        gold[f"batches_{k}"] = np.array([j for b in batches for j in b])
        gold[f"batch_sizes_{k}"] = np.array([len(b) for b in batches])

    # ---- BLEU over unit ids (refs end in eos, some unks and pads; one lone-eos ref as --target-is-code gives)
    udict = Dictionary.units(cfg.unit_vocab - 5)
    pairs = []
    for k in range(12):
        n = int(rng.integers(1, 40))
        ref = list(rng.integers(4, 30, n)) + [udict.eos()]
        if k % 3 == 0:
            ref[int(rng.integers(0, n))] = udict.unk()
        pred = [int(t) for t in ref[:-1]]
        pred = [t if rng.random() < 0.7 else int(rng.integers(4, 30)) for t in pred][: max(1, n - int(rng.integers(0, 5)))]
        if k == 5:
            ref = [udict.eos()]
        if k == 7:
            ref = [udict.pad(), udict.pad()] + ref
        pairs.append((ref, pred))
    gold["bleu_pairs"] = np.array([" ".join(map(str, r)) + "|" + " ".join(map(str, p)) for r, p in pairs])
    gold["bleu_result"] = np.array(reference_bleu(pairs, udict.pad(), udict.eos(), udict.unk()))

    # ---- generation at --max-tokens MAX_TOKENS: reference modules per batch
    enc = build_reference_encoder(cfg, sd, None, None)
    mods = build_reference_decoders(cfg, sd)
    glb = {"torch": torch, "nn": nn, "math": math, "utils": futils, "List": List, "Dict": Dict, "Optional": Optional, "Tensor": torch.Tensor}
    RefCTC = extract_class(REF + "/researches/ctc_unity/ctc_decoder.py", "CTCDecoder", glb)
    RefUnitCTC = extract_class(REF + "/researches/ctc_unity/ctc_generator.py", "CTCSequenceGenerator", glb)
    fns = extract_functions(REF + "/fairseq/fairseq/data/dictionary.py", "Dictionary", ["string", "unk_string"],
                            {"torch": torch, "utils": futils, "data_utils": types.SimpleNamespace(post_process=lambda s, b: s)})

    class RefDict(Dictionary):  # the unit dictionary with fairseq Dictionary.string / unk_string from their own source
        unk_word = "<unk>"
        string = fns["string"]
        unk_string = fns["unk_string"]

    rd = RefDict([str(i) for i in range(cfg.unit_vocab - 5)] + ["<blank>"])
    assert len(rd) == cfg.unit_vocab

    class FakeModel(nn.Module):
        def __init__(self):
            super().__init__()
            self.source_unigram_decoder = mods["source_unigram"]
            self.ctc_target_unigram_decoder = mods["ctc_target_unigram"]
            self.decoder = mods["unit"]

        def max_decoder_positions(self):
            return 1200

        def get_normalized_probs(self, net_output, log_probs, sample=None):
            logits = net_output[0].float()
            return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)

    fake = FakeModel()
    orc = StreamSpeechOracle(cfg, sd, None, gcmvn, chunk_size=None, conv_chunk_size=None)
    gen_batches = batchings[(MAX_TOKENS, -1, 1)]
    assert len(gen_batches) >= 3 and max(len(b) for b in gen_batches) > 1, gen_batches
    sdict, tdict = Dictionary.synthetic(cfg.src_vocab), Dictionary.synthetic(cfg.tgt_vocab)

    def text(d, toks):  # the generator's print rule (sequence_generator_multi_decoder_ctc.py:216-225)
        t = "".join([d[c] for c in toks])
        t = t.replace("_", " ").replace("▁", " ").replace("<unk>", " ").replace("<s>", "").replace("</s>", "")
        return t[1:] if len(t) > 0 and t[0] == " " else t

    stdout, results, ragged = [], [], False
    for bi, batch in enumerate(gen_batches):
        fl = [torch.from_numpy(feats[i]) for i in batch]
        lens = torch.tensor([f.size(0) for f in fl])
        x = torch.zeros(len(fl), int(lens.max()), cfg.feat_dim)
        for b, f in enumerate(fl):
            x[b, :f.size(0)] = f
        mine = offline_generate(orc, x, lens, max_len_b_mt=MAX_LEN_B_MT)
        enc_out = enc._forward(x, lens)
        lines = {"A": [], "S": [], "D": []}
        for name, key, d in (("source_unigram", "A", sdict), ("ctc_target_unigram", "S", tdict)):
            hyp = RefCTC(FakeDict(6000), [fake]).generate(enc_out, aux_task_name=name)
            for b, i in enumerate(batch):
                assert hyp[b][0]["tokens"].tolist() == mine["asr" if key == "A" else "st"][b]["tokens"], (bi, name, b)
                lines[key].append("{}-{}\t{}".format(key, i, text(d, hyp[b][0]["tokens"].int().tolist())))
        prev = mine["prev_output_tokens_mt"]
        mt_lens = [len(h) for h in mine["mt_hyps"]]
        ragged |= len(batch) > 1 and len(set(mt_lens)) > 1
        for b, i in enumerate(batch):
            h = list(mine["mt_hyps"][b])
            if h and h[-1] == cfg.eos:
                h = h[:-1]
            lines["D"].append("D-{}\t{}".format(i, text(tdict, h)))
        stdout += lines["A"] + lines["S"] + lines["D"]
        ref_feats, _ = mods["mt"](prev, encoder_out=enc_out, features_only=True)
        pad_mask = prev.eq(cfg.pad) if prev.eq(cfg.pad).any() else None
        t2u_ref = mods["t2u"](ref_feats.transpose(0, 1), pad_mask)
        hyp = RefUnitCTC(FakeDict(cfg.unit_vocab, blank=cfg.unit_blank), [fake]).generate(t2u_ref)
        for b, i in enumerate(batch):
            assert hyp[b][0]["tokens"].tolist() == mine["units"][b]["tokens"], (bi, b)
            h = hyp[b][0]
            units = h["tokens"].int().tolist()
            hypo_str = rd.string(torch.tensor(units), None, extra_symbols_to_ignore={rd.eos()})
            target_tokens = torch.tensor([rd.eos()])  # --target-is-code: encode_line("", append_eos=True) of the empty target
            target_str = rd.string(target_tokens.int(), None, escape_unk=True, extra_symbols_to_ignore={rd.eos()})
            score = h["score"] / math.log(2)
            pos = h["positional_scores"].clone().div_(math.log(2)).tolist()
            results.append({"id": i, "T": "T-{}\t{}".format(i, target_str), "H": "H-{}\t{}\t{}".format(i, score, hypo_str),
                            "D": "D-{}\t{}\t{}".format(i, score, hypo_str), "P": "P-{}\t{}".format(i, " ".join(map(lambda v: "{:.4f}".format(v), pos))),
                            "units": units, "score": h["score"], "positional": h["positional_scores"].numpy().astype(np.float32),
                            "target": target_tokens.int().tolist()})
        print(f"batch {bi}: samples {batch}, MT lengths {mt_lens}")
    assert ragged, "the fixture should have a batch of several samples with ragged MT lengths"
    bleu_pairs = [(r["target"], r["units"]) for r in results]
    gold["gen_max_tokens"] = np.array(MAX_TOKENS)
    gold["max_len_b_mt"] = np.array(MAX_LEN_B_MT)
    gold["stdout"] = np.array(stdout)
    gold["file_lines"] = np.array([r[k] for r in results for k in "THDP"] +
                                  ["Generate test with beam=1: " + reference_bleu(bleu_pairs, rd.pad(), rd.eos(), rd.unk())])
    for r in results:
        gold[f"units_{r['id']}"] = np.array(r["units"], dtype=np.int64)
        gold[f"score_{r['id']}"] = np.array(r["score"])
        gold[f"positional_{r['id']}"] = r["positional"]
    path = os.path.join(GOLD, "offline_generate.npz")
    np.savez_compressed(path, **gold)
    print("\n".join(stdout[:4]))
    print("\n".join(gold["file_lines"][:4].tolist()), "\n", gold["file_lines"][-1])
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
