"""GPU, end to end: `python -m streamspeech_b200.evaluate` runs the S2ST agent over a short synthetic source list, then
`python -m streamspeech_b200.asr_bleu` scores its wavs/ in both variants on the synthetic Large-shape transcriber.  The transcripts, the
files and the printed score line must equal what the oracle pipeline gives on the same WAVs: read_wav, remove_silence (pinned to the
reference's own code by tests/golden/asr_w2v.npz), the float64 oracle forward pass, the beam-1 rule, _get_tokens (pinned to torchaudio's
own), the letter post-processing and the BLEU restatement."""
import os

import pytest
import torch

from oracle import asr_oracle as ao
from streamspeech_b200 import asr_bleu, synth
from streamspeech_b200 import evaluate as ev
from streamspeech_b200.asr import SPECIALS, ASRTranscriber, remove_silence
from streamspeech_b200.sacrebleu_compat import corpus_bleu

pytestmark = pytest.mark.gpu

AGENT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents",
                     "speech_to_speech.streamspeech.agent.py")
SECONDS = [2.1, 3.4, 1.6, 2.8]
REFS = ["so on and so on", "the end", "o no", "son of a son"]
STRIDES = [s for (_, _, s) in synth.W2V_CONV_LAYERS]
KERNELS = [k for (_, k, _) in synth.W2V_CONV_LAYERS]
TIE_MARGIN = 1e-2  # the engine and the fp64 oracle may pick different letters only where the fp64 top two are this close (as test_asr_gpu)


def oracle_transcripts(files, rm, sd64, vocab, engine):
    """per file: the oracle pipeline's transcript (None: shorter than one frame).  The engine's per-frame arg-max (ASRTranscriber, the
    transcriber the CLI builds) must equal the fp64 one except at near-ties; at those frames the engine's letter is the expected one."""
    out, ties = [], 0
    for fp in files:
        x, _ = ev.read_wav(fp)
        if rm:
            x = remove_silence(x)
        if ao.num_frames(len(x), KERNELS, STRIDES) <= 0:
            out.append(None)
            continue
        e = ao.forward(sd64, torch.from_numpy(x), STRIDES, normalize=True, dtype=torch.float64, device="cuda")["emissions"]
        m = e.clone()
        m[:, ao.UNK] = float("-inf")
        top2 = m.topk(2, dim=1).values
        margin = (top2[:, 0] - top2[:, 1]).cpu()
        bp = ao.best_path(e)
        _, am = engine.transcribe_tokens([x])[0]
        diff = [t for t in range(len(bp)) if am[t] != bp[t]]
        assert all(float(margin[t]) < TIE_MARGIN for t in diff), [(t, float(margin[t])) for t in diff]
        ties += len(diff)
        out.append(ao.letters(ao.get_tokens(am if diff else bp), vocab))
    return out, ties


def test_evaluate_then_asr_bleu_equals_the_oracle_pipeline(tmp_path, capsys):
    paths = []
    for i, sec in enumerate(SECONDS):
        p = tmp_path / f"utt{i}.wav"
        from streamspeech_b200.generate_waveform_from_code import write_wav

        write_wav(str(p), synth.make_audio(sec, seed=900 + i).numpy(), 16000)
        paths.append(str(p))
    (tmp_path / "src.txt").write_text("\n".join(paths) + "\n")
    (tmp_path / "tgt.txt").write_text("\n".join(REFS) + "\n")
    out = tmp_path / "eval"
    ev.main(["--agent", AGENT, "--source", str(tmp_path / "src.txt"), "--target", str(tmp_path / "tgt.txt"), "--output", str(out),
             "--source-segment-size", "320", "--streams", "2", "--model-path", "synthetic", "--data-bin", ".", "--vocoder", "synthetic",
             "--vocoder-cfg", "none", "--dur-prediction", "--sample-rate", "16000"])
    wavs = out / "wavs"
    files = asr_bleu.extract_audio_for_eval(str(wavs), "n_pred.wav")
    assert len(files) == len(SECONDS)
    sd64 = {k: v.to("cuda", torch.float64) for k, v in synth.make_w2v_ctc_state_dict().items()}
    vocab = SPECIALS + [ln.split()[0] for ln in synth.w2v_letter_dict().splitlines()]
    engine = ASRTranscriber("synthetic", None, 0)
    capsys.readouterr()

    base = ["--lang", "en", "--audio_dirpath", str(wavs), "--reference_path", str(tmp_path / "tgt.txt"), "--reference_format", "txt",
            "--asr-model", "synthetic"]
    # default variant
    want, ties = oracle_transcripts(files, False, sd64, vocab, engine)
    print(f"default variant: {ties} frames took the engine's letter at a near-tie")
    want = [w if w is not None else "" for w in want]
    tr, bleu = asr_bleu.main(base + ["--results_dirpath", str(tmp_path / "res")])
    assert tr == want
    assert any(want)  # the synthetic transcriber writes letters
    ref_bleu = corpus_bleu(want, [REFS])
    assert str(bleu) == str(ref_bleu)
    assert capsys.readouterr().out.splitlines()[-1] == str(ref_bleu)
    assert (wavs / "pred.txt").read_text() == "\n".join(want)
    assert (tmp_path / "res" / "txt_en_bleu.txt").read_text() == ref_bleu.format(width=2)
    # rm_silence variant
    (wavs / "pred.txt").unlink()
    want_rm, ties = oracle_transcripts(files, True, sd64, vocab, engine)
    argv = base + ["--rm-silence", "--results_dirpath", str(tmp_path / "res_rm"), "--transcripts_path", str(tmp_path / "t.txt")]
    if any(w is None for w in want_rm):  # an output the silence rule empties: the reference's transcriber fails, and so does this one
        with pytest.raises(ValueError, match="fewer than one encoder frame"):
            asr_bleu.main(argv)
        return
    tr, bleu = asr_bleu.main(argv)
    assert tr == want_rm
    ref_bleu = corpus_bleu(want_rm, [REFS])
    assert str(bleu) == str(ref_bleu)
    assert capsys.readouterr().out.splitlines()[-1] == str(ref_bleu)
    assert (tmp_path / "t.txt").read_text() == "".join(t + "\n" for t in want_rm)
    assert (tmp_path / "res_rm" / "txt_en_bleu.txt").read_text() == ref_bleu.format(width=2)
    assert not (wavs / "pred.txt").exists()
