"""UnitY offline generation on the H100: the unit-search kernel (ss_unit_search_batch) and the T2U encoder (ss_t2u_encode_batch)
against the float64 oracle (oracle/unity_oracle.py) with margin-aware token checks, the `--task speech_to_speech_modified` front door
on a split written to disk, its units through the waveform pipeline, and a UnitY handle refusing the CTC and stream-pool entries."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.unity_oracle import UnitYOracle
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARGIN = 1e-4  # float64 decisions closer than this may go either way in fp32


@pytest.fixture(scope="module")
def unity():
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, None, None, device=0)
    yield cfg, sd, eng, UnitYOracle(cfg, sd, torch.float64)
    eng.close()


def _states(B, S, lens, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, 512, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = 1e3 * torch.randn(S - n, 512, generator=g)  # rows that are not keys: any leak would show
    return x


def long_search_state_dict(cfg):
    """the synthetic UnitY weights with eos's output row set to zero: its logit is 0 at every step, below the best unit's"""
    sd = synth.make_unity_state_dict(cfg, seed=1)
    e = sd["decoder.embed_tokens.weight"].clone()
    e[cfg.eos] = 0.0
    sd["decoder.embed_tokens.weight"] = sd["decoder.output_projection.weight"] = e
    return sd


def _check_rows(got, want, cfg):
    for b, (a, r) in enumerate(zip(got, want)):
        n = next((i for i, m in enumerate(r["margins"]) if m < MARGIN), len(r["margins"]))
        assert a["tokens"][:n] == r["tokens"][:n], (b, n)
        if n == len(r["margins"]):
            assert a["tokens"] == r["tokens"], b
            assert abs(a["score"] - r["score"]) < 2e-4 * max(1.0, abs(r["score"])), (b, a["score"], r["score"])
            # positional scores are differences of fp32 cumulative scores (finalize_hypos): each carries about one ulp of the
            # cumulative sum, 5e-4 at -5500 after 1100 steps
            pos = a["positional_scores"].double().numpy()
            bar = 2e-4 + 2.4e-7 * abs(r["score"]) * len(r["tokens"])
            assert np.abs(pos - np.array(r["positional_scores"])).max() < bar, b
            assert a["tokens"][-1] == cfg.eos


@pytest.mark.parametrize("B,max_len", [(1, 60), (8, 60), (8, 300), (32, 60), (33, 60)])
def test_unit_search_against_fp64(unity, B, max_len):
    """1 row, a full launch group, and 33 rows (two groups); ragged T2U lengths; early eos and the forced eos at max_len"""
    cfg, _, eng, o64 = unity
    S = 14
    lens = [S - (b * 5) % S for b in range(B)]
    x = _states(B, S, lens, seed=B)
    got = eng.unit_search_batch(x.cuda().contiguous(), lens, max_len)
    want = o64.unit_search(x, lens, max_len)
    _check_rows(got, want, cfg)
    n = [len(r["tokens"]) for r in want]
    if B >= 8 and max_len == 60:
        assert min(n) < max_len + 1 and max(n) == max_len + 1 and len(set(n)) > 2  # early eos, forced eos, different ends


def test_unit_search_past_1024_positions(unity):
    """self-attention over more than 1024 cached entries: rows that never rank eos first run to the forced eos at step 1100"""
    cfg, _, _, _ = unity
    from streamspeech_b200.engine import Engine

    sd = long_search_state_dict(cfg)
    eng = Engine(cfg, sd, None, None, device=0)
    try:
        lens = [9, 4]
        x = _states(2, 9, lens, seed=11)
        got = eng.unit_search_batch(x.cuda().contiguous(), lens, 1100)
        want = UnitYOracle(cfg, sd, torch.float64).unit_search(x, lens, 1100)
        assert max(len(r["tokens"]) for r in want) > 1025
        _check_rows(got, want, cfg)
    finally:
        eng.close()


def test_t2u_encoder_against_fp64(unity):
    cfg, _, eng, o64 = unity
    lens = [12, 7, 1, 12, 3]
    x = _states(5, 12, lens, seed=3)
    got = eng.t2u_encode_batch(x.cuda().contiguous(), lens).cpu().double()
    want = o64.t2u_encode(x, lens)
    for b, n in enumerate(lens):
        err = (got[b, :n] - want[b, :n]).abs().max() / want[b, :n].abs().max()
        assert err < 1e-5, (b, float(err))


def test_refusals(unity):
    from streamspeech_b200.engine import EngineError

    cfg, _, eng, _ = unity
    enc = torch.zeros(1, 8, cfg.enc_dim, device="cuda")
    with pytest.raises(EngineError, match="no CTC heads"):
        eng.ctc_greedy_batch(enc)
    with pytest.raises(EngineError, match="no CTC heads"):
        eng.ctc_greedy(0, enc[0])
    eng.pool_create(2, 4)
    with pytest.raises(EngineError, match="no CTC heads"):
        eng.pool_step([0], ctc_heads=0)
    x = torch.zeros(2, 4, 512, device="cuda")
    with pytest.raises(EngineError, match="outside"):
        eng.unit_search_batch(x, [4, 5], 10)
    with pytest.raises(EngineError, match="position table"):
        eng.unit_search_batch(x, [4, 4], 1200)
    with pytest.raises(EngineError, match="max_len"):
        eng.unit_search_batch(x, [4, 4], 0)


def test_streamspeech_handle_refuses_unit_search():
    from streamspeech_b200.engine import Engine, EngineError

    cfg = ModelConfig().tiny()
    eng = Engine(cfg, synth.make_model_state_dict(cfg, seed=0), None, None, device=0)
    try:
        with pytest.raises(EngineError, match="no autoregressive unit decoder"):
            eng.unit_search_batch(torch.zeros(1, 4, 512, device="cuda"), [4], 10)
    finally:
        eng.close()


def write_unity_split(root, n=7, seed=0):
    g = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    frames = [int(x) for x in g.integers(60, 400, n)]
    with open(os.path.join(root, "test.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\n")
        for i, F in enumerate(frames):
            p = os.path.join(root, f"utt{i}.npy")
            np.save(p, g.standard_normal((F, 80)).astype(np.float32))
            f.write(f"utt{i}\t{p}\t{F}\t\t0\n")
    return frames


def test_front_door_end_to_end(tmp_path, capsys):
    """pred.sh's flags on a written split: stdout only D- lines, the results file T/H/D/P + BLEU, and its D- units through
    generate_waveform_from_code (one finite waveform per sample) and asr_bleu (a score line).  The outputs themselves are compared
    with the reference's in tests/test_unity_golden.py."""
    import json

    from streamspeech_b200 import asr_bleu
    from streamspeech_b200 import generate as G
    from streamspeech_b200.config import VocoderConfig
    from streamspeech_b200.evaluate import read_wav

    data = str(tmp_path / "data")
    write_unity_split(data)
    out = str(tmp_path / "out")
    argv = [data, "--task", "speech_to_speech_modified", "--target-is-code", "--target-code-size", "1000", "--path", "synthetic",
            "--gen-subset", "test", "--beam-mt", "4", "--beam", "1", "--max-len-a", "1", "--max-len-b", "20", "--max-tokens", "900",
            "--required-batch-size-multiple", "1", "--results-path", out]
    split = G.main(argv)
    stdout = capsys.readouterr().out.splitlines()
    assert stdout and all(line.startswith("D-") for line in stdout)
    assert sorted(int(line.split("\t")[0][2:]) for line in stdout) == list(range(7))
    lines = open(os.path.join(out, "generate-test.txt")).read().splitlines()
    assert lines[-1].startswith("Generate test with beam=1: BLEU4 = ")
    assert [line[0] for line in lines[:-1]] == list("THDP") * 7
    assert len(split.batches) > 1 and any(len(b) > 1 for b in split.batches)
    import json

    from streamspeech_b200 import asr_bleu
    from streamspeech_b200.config import VocoderConfig
    from streamspeech_b200.evaluate import read_wav

    d = sorted((int(l.split("\t")[0][2:]), l.split("\t")[2]) for l in lines if l.startswith("D-"))
    codes, wav_dir, vcfg = os.path.join(out, "generate-test.unit"), os.path.join(out, "pred_wav"), os.path.join(out, "vocoder.json")
    with open(codes, "w") as f:
        f.write("".join(u + "\n" for _, u in d))
    with open(vcfg, "w") as f:
        json.dump(VocoderConfig().to_json_dict(), f)
    r = subprocess.run([sys.executable, "-m", "streamspeech_b200.generate_waveform_from_code", "--in-code-file", codes, "--vocoder",
                        "synthetic", "--vocoder-cfg", vcfg, "--results-path", wav_dir, "--dur-prediction"], cwd=ROOT, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    wavs = sorted(os.listdir(wav_dir))
    assert len(wavs) == 7
    for w in wavs:
        x, _ = read_wav(os.path.join(wav_dir, w))
        assert len(x) > 0 and np.isfinite(x).all()
    ref = tmp_path / "test.txt"
    ref.write_text("".join(f"reference sentence {i}\n" for i in range(7)))
    _, bleu = asr_bleu.main(["--lang", "en", "--audio_dirpath", wav_dir, "--reference_path", str(ref), "--reference_format", "txt",
                             "--asr-model", "synthetic", "--results_dirpath", str(tmp_path / "asr")])
    assert capsys.readouterr().out.splitlines()[-1] == str(bleu)
