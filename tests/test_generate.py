"""`python -m streamspeech_b200.generate` (fairseq-generate --task speech_to_speech_ctc on a data split) and the scored unit arg-max
under it, against tests/golden/offline_generate.npz (oracle/gen_golden_generate.py: fairseq's own ordering, batching, BLEU and
CTCSequenceGenerator scores).  CPU: reading, batching, BLEU, formatting, checkpoint settings, refusals.  GPU: the kernel against
float64, the front door end to end against the fixture, and the waveform pipeline."""
import argparse
import hashlib
import json
import math
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest
import torch

from streamspeech_b200 import generate as G
from streamspeech_b200.dictionary import Dictionary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "offline_generate.npz")
UNIT_BATCH_ROWS = 32768  # SS_UNIT_BATCH_ROWS (include/streamspeech_b200.h)
MAX_TOKENS = 900         # --max-tokens of the fixture's generation run (gen_max_tokens)


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLD))


def write_split(g, root):
    """The fixture's split on disk: raw fbank (int16 counts of 1 / raw_scale in the fixture) as fp32 .npy files and as fp32 .npy entries
    of one stored zip, gcmvn stats, config yaml"""
    scale = np.float32(int(g["raw_scale"]))
    n = len(g["n_frames"])
    os.makedirs(root, exist_ok=True)
    np.savez(os.path.join(root, "gcmvn.npz"), mean=g["gcmvn_mean"], std=g["gcmvn_std"])
    with open(os.path.join(root, "config_gcmvn.yaml"), "w") as f:
        f.write(f"global_cmvn:\n  stats_npz_path: {os.path.join(root, 'gcmvn.npz')}\ninput_channels: 1\ninput_feat_per_channel: 80\n"
                "transforms:\n  '*':\n  - global_cmvn\n  _train:\n  - global_cmvn\n  - specaugment\n")
    zpath = os.path.join(root, "fbank80.zip")
    npy = set(g["npy_samples"].tolist())
    with zipfile.ZipFile(zpath, "w", compression=zipfile.ZIP_STORED) as z:
        for i in range(n):
            if i not in npy:
                with z.open(f"utt{i}.npy", "w") as e:
                    np.save(e, g[f"raw_{i}"].astype(np.float32) / scale)
    paths = {}
    with zipfile.ZipFile(zpath) as z:
        for info in z.infolist():
            off = info.header_offset + 30 + len(info.filename.encode()) + len(info.extra)
            paths[int(info.filename[3:-4])] = f"{zpath}:{off}:{info.file_size}"
    for i in npy:
        p = os.path.join(root, f"utt{i}.npy")
        np.save(p, g[f"raw_{i}"].astype(np.float32) / scale)
        paths[i] = p
    with open(os.path.join(root, "test.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\n")
        for i in range(n):
            f.write(f"utt{i}\t{paths[i]}\t{int(g['n_frames'][i])}\t5 17 17 940\t{int(g['tgt_n_frames'][i])}\n")
    return root


# ----------------------------------------------------------------------------------------------------------------------------- CPU

def test_reading_and_cmvn_equal_fixture(g, tmp_path):
    root = write_split(g, str(tmp_path))
    args = G.parse_args([root, "--config-yaml", "config_gcmvn.yaml", "--path", "synthetic", "--beam", "1", "--max-tokens", "1200",
                         "--target-is-code"])
    split = G.Split(args, G.load_config_yaml(args), 1024)
    assert [int(r["src_n_frames"]) for r in split.rows] == g["n_frames"].tolist()
    for i in range(len(split.rows)):
        x = split.features(i)
        assert x.dtype == np.float32 and hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest() == str(g[f"feats_sha256_{i}"]), i
    assert split.target(0) == ""  # --target-is-code: the reference's creator replaces the target by ""


def test_batching_equals_fairseq(g):
    n_frames, tgt = g["n_frames"].tolist(), g["tgt_n_frames"].tolist()
    assert len(set(n_frames)) < len(n_frames)  # ties in n_frames
    assert G.ordered_indices(n_frames).tolist() == g["ordered_indices"].tolist()
    for k, (mt, bs, mult) in enumerate(g["batch_settings"].tolist()):
        got = G.make_batches(n_frames, tgt, mt if mt > 0 else None, bs if bs > 0 else None, mult, (6000, 1024), False)
        assert [len(b) for b in got] == g[f"batch_sizes_{k}"].tolist(), (mt, bs, mult)
        assert [i for b in got for i in b] == g[f"batches_{k}"].tolist(), (mt, bs, mult)


def test_size_filter():
    with pytest.raises(ValueError, match="Size of sample #1 is invalid"):
        G.make_batches([100, 7000, 50], [5, 5, 5], 10000, None, 1, (6000, 1024), False)
    assert G.make_batches([100, 7000, 50], [5, 5, 2000], 10000, None, 1, (6000, 1024), True) == [[0]]


def test_bleu_equals_libbleu(g):
    d = Dictionary.units(1000)
    s = G.BleuScorer(d.pad(), d.eos(), d.unk())
    for pair in g["bleu_pairs"].tolist():
        ref, pred = pair.split("|")
        s.add([int(t) for t in ref.split()], [int(t) for t in pred.split()])
    assert s.result_string() == str(g["bleu_result"])


def test_line_formatting_equals_fixture(g):
    d = Dictionary.units(1000)
    ids = [int(line.split("\t")[0][2:]) for line in g["file_lines"].tolist()[0::4][:-1]]
    lines = []
    s = G.BleuScorer(d.pad(), d.eos(), d.unk())
    for i in ids:
        units = g[f"units_{i}"].tolist()
        tt = G.encode_line(d, "")
        lines += G.hypothesis_lines(i, G.unit_string(d, tt, escape_unk=True), G.unit_string(d, units), float(g[f"score_{i}"]), g[f"positional_{i}"])
        s.add(tt, units)
    lines.append("Generate test with beam=1: " + s.result_string())
    assert lines == g["file_lines"].tolist()


def test_text_rule():
    d = Dictionary(["▁le", "_chat", "noir", "<blank>"])
    # <s>=0 <pad>=1 </s>=2 <unk>=3 ▁le=4 _chat=5 noir=6
    assert G.ctc_text(d, [4, 5, 6]) == "le chatnoir"
    assert G.ctc_text(d, [0, 6, 3, 4, 2]) == "noir  le"
    assert G.ctc_text(d, []) == ""
    assert G.unit_string(Dictionary.units(1000), [0, 4, 3, 1003, 2]) == "0 <unk> 999"


def test_checkpoint_settings():
    assert G.offline_settings({"cfg": {"model": {"uni_encoder": False, "chunk_size": 999999}}}, 1024) == (False, None)
    assert G.offline_settings({"args": argparse.Namespace(uni_encoder=True, chunk_size=1024)}, 1024) == (True, None)
    assert G.offline_settings({"cfg": {"model": {}}}, 1024) == (False, None)
    with pytest.raises(ValueError, match="--chunk-size 8:"):
        G.offline_settings({"cfg": {"model": {"uni_encoder": True, "chunk_size": 8}}}, 1024)


@pytest.mark.parametrize("flags,msg", [(["--beam", "5"], "--beam 5"), (["--beam", "1", "--nbest", "2"], "--nbest 2"),
                                       (["--beam", "1", "--max-len-a-mt", "1"], "--max-len-a-mt"), (["--beam", "1", "--cpu"], "--cpu"),
                                       (["--beam", "1", "--task", "speech_to_text"], "speech_to_speech_ctc")])
def test_refused_flags(flags, msg, capsys):
    with pytest.raises(SystemExit):
        G.parse_args(["DATA", "--path", "synthetic", "--max-tokens", "1000"] + flags)
    assert msg in capsys.readouterr().err


def test_refused_inputs(g, tmp_path):
    with pytest.raises(ValueError, match="waveform sources"):
        G.read_features("a.wav")
    with pytest.raises(ValueError, match="waveform sources"):
        G.read_features("a.flac")
    root = write_split(g, str(tmp_path))
    with open(os.path.join(root, "long.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\nbig\tx.npy\t5000\t\t10\n")
    args = G.parse_args([root, "--config-yaml", "config_gcmvn.yaml", "--path", "synthetic", "--beam", "1", "--max-tokens", "10000",
                         "--gen-subset", "long"])
    with pytest.raises(ValueError, match="sample big: 5000 source frames.*at most 4096"):
        G.Split(args, G.load_config_yaml(args), 1024)
    with open(os.path.join(root, "wav.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\nw\tx.wav\t50\t\t10\n")
    args.gen_subset = "wav"
    with pytest.raises(ValueError, match="sample w: source x.wav"):
        G.Split(args, G.load_config_yaml(args), 1024)


# ----------------------------------------------------------------------------------------------------------------------------- GPU

def offline_engine():
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    cfg.uni_encoder = False
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, None)
    e.set_chunk(None, None)
    return e


def ref_lprob(logits: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return torch.log_softmax(logits.double().cpu(), dim=-1).gather(1, idx.cpu()[:, None])[:, 0]


# Largest |lprob - fp64 log_softmax| measured on the H100 (80 GB HBM3, 700 W, 1980 MHz max SM clock): 1.9e-6 on the edge rows of
# test_argmax_lprob_kernel_edges, 3.3e-7 on the unit logits of test_scored_entry_point_matches_unscored
LPROB_BAR = 1e-5


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_argmax_lprob_kernel_edges():
    """argmax_lprob_rows against fp64 log_softmax of the same fp32 logits, indices bit-identical to argmax_rows: a masked column
    holding the row maximum, exact ties, a very large spread, plain rows"""
    e = offline_engine()
    try:
        V = 1005
        gen = torch.Generator().manual_seed(3)
        x = torch.randn(64, V, generator=gen) * 4
        x[0:8, 1] = 50.0            # pad holds the maximum (masked)
        x[8:16, 2] = 60.0           # eos holds the maximum (masked only with 3 masked columns)
        x[16:24, 700] = 30.0        # exact tie, lower index must win
        x[16:24, 900] = 30.0
        x[24:32, :] = -1e4          # very large spread: one live column, the rest underflow
        x[24:32, 500] = 1e3
        x[32:40, 10:] = 7.25        # a row of equal values
        x[40:48] *= 100
        worst = 0.0
        for n_masked in (2, 3):
            xd = x.cuda()
            i0, _ = e.op_argmax_rows(xd, n_masked, False)
            i1, lp = e.op_argmax_rows(xd, n_masked, True)
            assert torch.equal(i0, i1)
            masked = [1, 3, 2][:n_masked]
            assert not any(int(v) in masked for v in i1.tolist())
            assert (i1[16:24] == 700).all()
            ref = ref_lprob(x, i1)
            worst = max(worst, float((lp.cpu().double() - ref).abs().max()))
        print(f"argmax_lprob_rows worst |lprob - fp64| = {worst:.3e}")
        assert worst < LPROB_BAR, worst
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_scored_entry_point_matches_unscored():
    """ss_t2u_unit_decode_batch_scored: arg-max and units bit-identical to ss_t2u_unit_decode_batch with pad tails and in more than
    one SS_UNIT_BATCH_ROWS group; for one sample its lprob matches fp64 log_softmax of the call's unit logits"""
    e = offline_engine()
    try:
        gen = torch.Generator().manual_seed(11)
        S = 40
        B = UNIT_BATCH_ROWS // (S * 25) + 3  # two groups
        x = (torch.randn(B, S, 512, generator=gen) * 0.5).cuda().contiguous()
        pads = [(b * 7) % 9 for b in range(B)]
        u0, a0, _ = e.t2u_unit_decode_batch(x, pads, mask_eos=True)
        u1, a1, lp, dev = e.t2u_unit_decode_batch_scored(x, pads, mask_eos=True)
        assert u0 == u1 and a0 == a1
        assert all(bool(torch.isfinite(t).all()) and float(t.max()) <= 0 for t in lp)
        assert dev["lprob"].shape == (B, S * 25)
        # one sample: the debug logits of the same arithmetic (ss_t2u_unit_decode is this call with B = 1)
        x1 = x[:1].contiguous()
        r = e.t2u_unit_decode(x1[0].contiguous(), n_pad_tail=pads[0], mask_eos=True, debug=True)
        _, a1s, lp1, _ = e.t2u_unit_decode_batch_scored(x1, pads[:1], mask_eos=True)
        assert a1s[0] == r["argmax"].tolist()
        err = float((lp1[0].double() - ref_lprob(r["logits"], r["argmax"])).abs().max())
        print(f"scored entry point, one sample: worst |lprob - fp64| = {err:.3e}")
        assert err < LPROB_BAR, err
    finally:
        e.close()


def run_front_door(root, out, extra=()):
    cmd = [sys.executable, "-m", "streamspeech_b200.generate", root, "--user-dir", "researches/ctc_unity", "--config-yaml", "config_gcmvn.yaml",
           "--task", "speech_to_speech_ctc", "--target-is-code", "--target-code-size", "1000", "--vocoder", "code_hifigan",
           "--path", "synthetic", "--gen-subset", "test", "--beam", "1", "--max-len-a", "1", "--max-len-b-mt", "60",
           "--max-tokens", str(MAX_TOKENS), "--required-batch-size-multiple", "1", "--results-path", out, *extra]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    with open(os.path.join(out, "generate-test.txt")) as f:
        return p.stdout.splitlines(), f.read().splitlines()


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_front_door_end_to_end(g, tmp_path):
    assert int(g["gen_max_tokens"]) == MAX_TOKENS
    root = write_split(g, str(tmp_path / "data"))
    out = str(tmp_path / "res")
    stdout, lines = run_front_door(root, out)
    assert stdout == g["stdout"].tolist()
    exp = g["file_lines"].tolist()
    assert len(lines) == len(exp) and lines[-1] == exp[-1]
    worst_p = 0.0
    for got, want in zip(lines[:-1], exp[:-1]):
        kind = got[0]
        gf, wf = got.split("\t"), want.split("\t")
        assert gf[0] == wf[0]
        if kind == "T":
            assert got == want
        elif kind in "HD":
            assert gf[2] == wf[2]
            rows = len(g[f"positional_{int(gf[0][2:])}"])
            assert abs(float(gf[1]) - float(wf[1])) * math.log(2) < 1e-5 * rows, (got[:80], want[:80])
        else:
            a, b = np.array(gf[1].split(), dtype=np.float64), np.array(wf[1].split(), dtype=np.float64)
            assert a.shape == b.shape
            worst_p = max(worst_p, float(np.abs(a - b).max()))
    assert worst_p < 2e-4, worst_p
    # the reference script's grep / cut lines
    units = sorted(((int(l.split("\t")[0][2:]), l.split("\t")[2]) for l in lines if l.startswith("D-")))
    assert [u for _, u in units] == [G.unit_string(Dictionary.units(1000), g[f"units_{i}"].tolist()) for i, _ in units]

    # the units equal OfflineS2STGenerator.generate on the same batches, greedy and --beam-mt 4
    from streamspeech_b200.offline import OfflineS2STGenerator

    args = G.parse_args([root, "--config-yaml", "config_gcmvn.yaml", "--path", "synthetic", "--beam", "1", "--max-tokens", str(MAX_TOKENS),
                         "--required-batch-size-multiple", "1", "--target-is-code"])
    split = G.Split(args, G.load_config_yaml(args), 1024)
    assert len(split.batches) >= 3 and max(len(b) for b in split.batches) > 1
    e = offline_engine()
    try:
        for beam, file_lines in ((1, lines), (4, run_front_door(root, str(tmp_path / "res4"), ("--beam-mt", "4"))[1])):
            gen = OfflineS2STGenerator(e, beam_size_mt=beam, max_len_b_mt=60)
            d_lines = {int(l.split("\t")[0][2:]): l.split("\t")[2] for l in file_lines if l.startswith("D-")}
            for batch in split.batches:
                res = G.run_batch(gen, split, batch)
                plain = gen.generate(torch.stack([torch.nn.functional.pad(torch.from_numpy(split.features(i)),
                                                                          (0, 0, 0, max(split.src_n_frames[j] for j in batch) - split.src_n_frames[i]))
                                                  for i in batch]).cuda(), [split.src_n_frames[i] for i in batch])
                for i, r, p in zip(batch, res, plain):
                    assert r["units"] == p["units"], (beam, i)
                    assert d_lines[i] == G.unit_string(Dictionary.units(1000), p["units"]), (beam, i)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_front_door_to_waveforms(g, tmp_path):
    """generate-test.txt | grep "^D-" | sed 's/^D-//ig' | sort -nk1 | cut -f3 -> generate_waveform_from_code: one finite waveform each"""
    root = write_split(g, str(tmp_path / "data"))
    out = str(tmp_path / "res")
    _, lines = run_front_door(root, out)
    d = sorted((int(l.split("\t")[0][2:]), l.split("\t")[2]) for l in lines if l.startswith("D-"))
    unit_file = os.path.join(out, "generate-test.unit")
    with open(unit_file, "w") as f:
        f.write("".join(u + "\n" for _, u in d))
    wav_dir = os.path.join(out, "pred_wav")
    from streamspeech_b200.config import VocoderConfig

    vcfg = os.path.join(out, "vocoder_config.json")
    with open(vcfg, "w") as f:
        json.dump(VocoderConfig().to_json_dict(), f)
    p = subprocess.run([sys.executable, "-m", "streamspeech_b200.generate_waveform_from_code", "--in-code-file", unit_file, "--vocoder", "synthetic",
                        "--vocoder-cfg", vcfg, "--results-path", wav_dir, "--dur-prediction"], cwd=ROOT, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    from streamspeech_b200.evaluate import read_wav

    wavs = sorted(os.listdir(wav_dir))
    assert len(wavs) == len(d)
    for w in wavs:
        x, _ = read_wav(os.path.join(wav_dir, w))
        assert len(x) > 0 and np.isfinite(x).all()
