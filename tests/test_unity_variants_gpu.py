"""GPU: Uni-UnitY and Chunk-UnitY on the engine.

- Uni-UnitY's encoder (ss_encoder_forward with attention chunk 1 and conv chunk 0: a future mask, symmetric convolutions) against the
  float64 restatement of tests/test_encoder_fp64.py at T = 1, 63, 64, 65 and 1024, alone and in padded batches, with that file's bars.
- Chunk-UnitY's incremental encoder in the wait-k agent's call pattern: at every call the rows are within the streaming bar of the
  float64 full-prefix chunk encoder, and the rows that an earlier call reported final are bit-identical to what that call wrote.
- The `--user-dir researches/uni_unity` generate front door against tests/golden/unity_variants.npz with the tolerances of
  tests/test_unity_golden.py, and both wait-k agents on both models against the same fixture action by action (tokens, units and
  durations exact, waveform within 1e-3 of the reference's: the one stored WRITE, else the float32 oracle's vocoder on the stored units;
  a differing unit decision only at a float64 near tie, as in tests/test_waitk_gpu.py).
- The CTC entry points still refuse a UnitY-family handle.
"""
import argparse
import importlib.util
import io
import math
import os

import numpy as np
import pytest
import torch

from oracle.unity_variant_oracle import VariantWaitkS2STAgent, VariantWaitkS2TTAgent
from streamspeech_b200 import generate as G
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.simuleval_compat import SpeechSegment

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARGIN = 1e-4
ENC_TOL = {"stream": 4e-5, "fp32": 7e-5, "tc": 2e-4}  # tests/test_encoder_fp64.py's bars
UMMA_MIN_ROWS = 128


def _load(name):
    spec = importlib.util.spec_from_file_location(f"_uv_{name}", os.path.join(ROOT, "tests", f"{name}.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def g():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "unity_variants.npz")))


@pytest.fixture(scope="module")
def split():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "unity_generate.npz")))


@pytest.fixture(scope="module")
def fp64():
    return _load("test_encoder_fp64")


def _engine(variant, **kw):
    from streamspeech_b200.engine import Engine

    state = synth.make_unity_checkpoint(variant, seed=0)
    cfg = ModelConfig.from_checkpoint(state)
    return cfg, state["model"], Engine(cfg, state["model"], None, synth.make_gcmvn(cfg), **kw)


def test_uni_unity_encoder_vs_fp64(fp64):
    """T = 1, 63, 64, 65, 1024 alone, and padded batches (B = 3 and 4) whose samples span those lengths"""
    cfg, sd, e = _engine("uni_unity")
    try:
        e.set_option("umma_min_rows", UMMA_MIN_ROWS)
        e.set_chunk(*cfg.encoder_chunk())
        assert cfg.encoder_chunk() == (1, 0)
        ref = fp64.Ref64(cfg, sd, synth.make_gcmvn(cfg))
        feats = e.fbank(synth.make_audio(41.0, seed=17).cuda().contiguous())[:4094].contiguous()
        worst = fp64.Worst()
        for F_ in (3, 252, 256, 260, 4094):
            T = fp64.out_frames(F_)
            out = e.encoder(feats[:F_].unsqueeze(0).contiguous())
            want = ref.encoder(feats[:F_], None, 1, None)[0]
            worst.add("tc" if T >= UMMA_MIN_ROWS else "fp32", fp64.maxdiff(out[0], want), f"T={T}")
        for F_, lengths in ((260, [260, 1, 252, 256]), (4094, [4094, 256, 3])):
            B = len(lengths)
            x = torch.zeros(B, F_, cfg.feat_dim, device="cuda")
            for b, n in enumerate(lengths):
                x[b, :n] = feats[:n]
            out = e.encoder(x, lengths)
            want = ref.encoder(x, lengths, 1, None)
            for b, n in enumerate(lengths):
                m = fp64.out_frames(n)
                tc = B * fp64.out_frames(F_) >= UMMA_MIN_ROWS
                worst.add("tc" if tc else "fp32", fp64.maxdiff(out[b, :m], want[b, :m]), f"F={F_} B={B} b={b} length={n}")
        fp64.report("uni_unity_encoder_fp64", **worst.as_dict())
        worst.check(ENC_TOL)
    finally:
        e.close()


def test_chunk_unity_stream_vs_fp64_and_final_rows(fp64):
    """the agent's call pattern (320 ms of new source per call, the whole prefix's fbank rows): every row within the streaming bar
    of the float64 chunk encoder of the prefix; rows below an earlier call's T_final bit-identical to that call's output"""
    cfg, sd, e = _engine("chunk_unity")
    try:
        c = cfg.chunk_size
        e.set_chunk(*cfg.encoder_chunk())
        ref = fp64.Ref64(cfg, sd, synth.make_gcmvn(cfg))
        wav = synth.make_audio(8.0, seed=5).cuda().contiguous()
        feats = e.fbank(wav)
        buf = torch.zeros(1024, cfg.enc_dim, device="cuda")
        e.encoder_stream_reset()
        worst, prev, n_final = fp64.Worst(), None, 0
        for n in range(5120, wav.numel() + 5120, 5120):
            F_ = e.num_fbank_frames(min(n, wav.numel()))
            T, t_final = e.encoder_stream_step(feats[:F_].contiguous(), buf)
            assert t_final % c == 0 and t_final <= T
            if prev is not None:
                assert torch.equal(buf[:n_final], prev[:n_final]), F_
            worst.add("stream", fp64.maxdiff(buf[:T], ref.encoder(feats[:F_], None, c, c)[0]), f"F={F_}")
            prev, n_final = buf[:T].clone(), t_final
        assert n_final > 0
        fp64.report("chunk_unity_stream_fp64", **worst.as_dict())
        worst.check(ENC_TOL)
    finally:
        e.close()


def test_ctc_entry_points_refuse_the_variants():
    from streamspeech_b200.engine import EngineError

    for variant in ("uni_unity", "chunk_unity"):
        cfg, _, e = _engine(variant)
        try:
            enc = torch.zeros(8, cfg.enc_dim, device="cuda")
            with pytest.raises(EngineError, match="CTC heads"):
                e.ctc_greedy(0, enc)
        finally:
            e.close()


def test_uni_unity_front_door_against_fixture(g, split, tmp_path):
    """`python -m streamspeech_b200.generate --user-dir researches/uni_unity` on the fixture's split for every setting: the
    "(None-id)" MT prints and the results file's texts / units identical, scores within test_unity_golden's tolerances"""
    data = _load("test_generate").write_split(split, str(tmp_path / "data"))
    for k, (mt, beam_mt, mlb) in enumerate(g["gen_settings"].tolist()):
        out = str(tmp_path / f"out{k}")
        buf = io.StringIO()
        G.main([data, "--user-dir", "researches/uni_unity", "--config-yaml", "config_gcmvn.yaml", "--task", "speech_to_speech_modified",
                "--target-is-code", "--target-code-size", "1000", "--path", "synthetic", "--gen-subset", "test", "--beam-mt", str(beam_mt),
                "--beam", "1", "--max-len-a", "1", "--max-len-b", str(mlb), "--max-len-b-mt", str(int(g["gen_max_len_b_mt"])),
                "--max-tokens", str(mt), "--required-batch-size-multiple", "1", "--results-path", out], stdout=buf)
        assert buf.getvalue().splitlines() == g[f"gen{k}_stdout"].tolist(), k
        got = open(os.path.join(out, "generate-test.txt")).read().splitlines()
        want = g[f"gen{k}_file_lines"].tolist()
        assert len(got) == len(want) + 1 and got[-1].startswith("Generate test with beam=1: BLEU4 = ")
        for a, b in zip(got, want):
            fa, fb = a.split("\t"), b.split("\t")
            assert fa[0] == fb[0], (k, a[:60], b[:60])
            if fa[0][0] in "HD":
                assert fa[2] == fb[2], (k, fa[0])
                n = len(fb[2].split()) + 1
                assert abs(float(fa[1]) - float(fb[1])) * math.log(2) < 1e-5 * n, (k, fa[0], fa[1], fb[1])
            elif fa[0][0] == "P":
                pa, pb = np.array(fa[1].split(), dtype=np.float64), np.array(fb[1].split(), dtype=np.float64)
                assert pa.shape == pb.shape
                assert np.abs(pa - pb).max() < 2e-4 + 2.4e-7 * abs(pb.sum()) * math.log(2), (k, fa[0])
            else:
                assert a == b


def _setting(g, p):
    k1, k2, n, n2, ups, seg, chunk, seed = g[f"{p}_setting"].tolist()
    return dict(k1=k1, k2=k2, n=n, n2=n2, ups=ups, seg=seg, chunk=chunk, seed=seed, kind=str(g[f"{p}_kind"]), seconds=float(g[f"{p}_seconds"]))


def _float64_unit_margin(variant, s, wav, upto):
    cfg = ModelConfig.from_checkpoint(synth.make_unity_checkpoint(variant))
    sd = synth.make_unity_state_dict(cfg, seed=0)
    kw = dict(lagging_k1=s["k1"], lagging_k2=s["k2"], stride_n=s["n"], stride_n2=s["n2"], unit_per_subword=s["ups"], segment_size=s["seg"],
              dtype=torch.float64)
    o = (VariantWaitkS2STAgent(cfg, sd, synth.make_gcmvn(cfg), synth.make_vocoder_state_dict(cfg.vocoder, 1), **kw) if s["kind"] == "s2st"
         else VariantWaitkS2TTAgent(cfg, sd, synth.make_gcmvn(cfg), **kw))
    step = 16 * s["chunk"]
    for ci, i in enumerate(range(0, len(wav), step)):
        o.push(wav[i:i + step].tolist(), finished=i + step >= len(wav))
        tr = o.policy().trace
        if ci == upto:
            return tr.get("unit_margin", np.inf)


def _vocoder_oracle():
    """the float32 oracle's CodeHiFiGAN with duration prediction on the synthetic vocoder (the fixture generator's weights)"""
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg = ModelConfig.unity_default()
    return StreamSpeechOracle(cfg, {}, synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True), None, chunk_size=None)


def _reference_wav(g, key, voc):
    """the reference's samples of a WRITE: stored for one call of the fixture; for every other call the last wav_n samples of the
    float32 oracle's vocoder on the call's stored units, which the fixture generator held within 1e-5 of the reference's on every
    call (its durations must be the stored ones)"""
    if key + "_wav" in g:
        return g[key + "_wav"]
    n = int(g[key + "_wav_n"])
    if n == 0:
        return np.zeros(0, dtype=np.float32)
    wav, dur = voc.vocoder(g[key + "_units"].tolist(), True)
    assert dur.view(-1).tolist() == g[key + "_dur"].tolist(), key
    return wav[-n:].numpy().astype(np.float32)


@pytest.mark.parametrize("variant", ["uni_unity", "chunk_unity"])
@pytest.mark.parametrize("tag", ["s2st_default", "s2st_k5n2", "s2tt_default", "s2tt_k5n2"])
def test_waitk_agent_reproduces_the_reference_policy(g, variant, tag):
    from streamspeech_b200.waitk import WaitkS2STAgent, WaitkS2TTAgent, add_waitk_args

    p = f"{variant}_{tag}"
    s = _setting(g, p)
    parser = argparse.ArgumentParser()
    add_waitk_args(parser)
    args = parser.parse_args(["--model-path", "synthetic", "--user-dir", f"researches/{variant}", "--data-bin", ".", "--vocoder", "synthetic",
                              "--vocoder-cfg", "none", "--dur-prediction", "--lagging-k1", str(s["k1"]), "--lagging-k2", str(s["k2"]),
                              "--stride-n", str(s["n"]), "--stride-n2", str(s["n2"]), "--unit-per-subword", str(s["ups"]),
                              "--segment-size", str(s["seg"])])
    agent = WaitkS2STAgent(args) if s["kind"] == "s2st" else WaitkS2TTAgent(args)
    assert agent.cfg.unity_variant == variant and agent.incremental == (variant == "chunk_unity")
    wav = synth.make_audio(s["seconds"], seed=s["seed"])
    step = 16 * s["chunk"]
    kinds, flags, texts = g[f"{p}_kinds"], g[f"{p}_flags"], g[f"{p}_texts"]
    worst, n_write, finals = 0.0, 0, []
    voc = _vocoder_oracle() if s["kind"] == "s2st" else None
    try:
        for ci, i in enumerate(range(0, len(wav), step)):
            fin = i + step >= len(wav)
            agent.push(SpeechSegment(content=wav[i:i + step].tolist(), sample_rate=16000, finished=fin))
            action = agent.policy()
            tr = agent.trace
            finals.append(agent._enc_final)
            for k in ("mt_tokens", "units"):
                key = f"{p}_call{ci}_{k}"
                if key in g and k in tr and list(tr[k]) != g[key].tolist():
                    m = _float64_unit_margin(variant, s, wav, ci)
                    assert k == "units" and m < MARGIN, (p, ci, k, "differs away from a tie")
                    pytest.skip(f"{p}: call {ci} is a float64 near tie ({m:.2e}); the trajectories part there")
            for k in ("new_subword_tokens", "new_unit_tokens", "mt_tokens", "units", "dur"):
                key = f"{p}_call{ci}_{k}"
                assert (key in g) == (k in tr), (key, sorted(tr))
                if key in g:
                    assert np.array(tr[k]).reshape(-1).tolist() == g[key].reshape(-1).tolist(), key
            assert action.is_read() == (kinds[ci] == 0), (p, ci)
            if action.is_read():
                continue
            n_write += 1
            if s["kind"] == "s2st":
                seg = action.content
                assert [action.finished, seg.finished] == flags[ci].tolist(), (p, ci)
                ref = _reference_wav(g, f"{p}_call{ci}", voc)
                assert len(seg.content) == len(ref), (p, ci)
                if len(ref):
                    worst = max(worst, float(np.abs(np.asarray(seg.content, dtype=np.float32) - ref).max()))
            else:
                assert action.content == str(texts[ci]) and action.finished == bool(flags[ci][0]), (p, ci)
        assert ci + 1 == len(kinds) and n_write == int(kinds.sum())
        assert worst < 1e-3, (p, worst)
        # Chunk-UnitY encodes incrementally: final rows appear; Uni-UnitY's rows never become final
        assert (max(finals) > 0) == (variant == "chunk_unity"), finals
    finally:
        agent.engine.close()
