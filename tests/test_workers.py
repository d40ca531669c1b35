"""streamspeech_b200.workers, the `--devices` worker pool, with stub jobs and no CUDA: the flag and its refusals on every front door,
results in key order whatever order the workers finish in, a worker's error ending the run with no child left behind, and
evaluate's instance log merged in index order under --start-index / --end-index."""
import json
import multiprocessing
import os
import signal
import subprocess
import sys
import time
from contextlib import closing

import pytest

from streamspeech_b200 import asr_bleu
from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import generate as G
from streamspeech_b200 import workers
from test_evaluate import AGENT_DIR, ASR, LENGTHS, RecordingAgent, _no_elapsed, _source_list

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------------- flags

def test_devices_are_parsed_with_repeats():
    assert workers.parse_devices("0") == [0]
    assert workers.parse_devices("0,0") == [0, 0]
    assert workers.parse_devices("3,1,0,1") == [3, 1, 0, 1]


@pytest.mark.parametrize("text", ["", "a", "0,", ",0", "0,,1", "-1", "1.5", "0;1", "0 1"])
def test_malformed_device_lists_are_refused(text):
    with pytest.raises(Exception, match="comma-separated list of CUDA device indices"):
        workers.parse_devices(text)


def _evaluate_argv(tmp_path, *extra, out="out"):
    return ["--agent", os.path.join(AGENT_DIR, ASR), "--source", str(tmp_path / "src.txt"), "--target", str(tmp_path / "tgt.txt"),
            "--output", str(tmp_path / out), "--model-path", "synthetic", "--data-bin", ".", *extra]


def test_every_front_door_takes_devices_and_refuses_it_with_its_device_flag(tmp_path, capsys):
    args = ev.parse_args(_evaluate_argv(tmp_path, "--devices", "0,0", "--streams", "4"))
    assert args.devices == [0, 0] and args.device_index == 0 and args.streams == 4
    args = ev.parse_args(_evaluate_argv(tmp_path, "--device-index", "1"))
    assert args.devices is None and args.device_index == 1
    assert ev.parse_args(_evaluate_argv(tmp_path)).device_index == 0
    assert ev.parse_score_only_args(["--score-only", "--output", "o", "--devices", "1,0"]).devices == [1, 0]
    assert G.parse_args(["D", "--path", "synthetic", "--beam", "1", "--max-tokens", "9", "--devices", "0,0,0"]).devices == [0, 0, 0]
    assert asr_bleu.parse_args(["--lang", "en", "--devices", "0,1"]).devices == [0, 1]
    assert asr_bleu.parse_args(["--lang", "en"]).device == 0 and asr_bleu.parse_args(["--lang", "en"]).devices is None
    refusals = [
        (lambda: ev.parse_args(_evaluate_argv(tmp_path, "--devices", "0,1", "--device-index", "0")), "--device-index"),
        (lambda: ev.parse_score_only_args(["--score-only", "--output", "o", "--devices", "0", "--device-index", "1"]), "--device-index"),
        (lambda: G.parse_args(["D", "--path", "synthetic", "--beam", "1", "--max-tokens", "9", "--device-index", "0", "--devices", "0"]),
         "--device-index"),
        (lambda: asr_bleu.parse_args(["--lang", "en", "--device", "0", "--devices", "0,0"]), "--device"),
    ]
    for parse, flag in refusals:
        with pytest.raises(SystemExit):
            parse()
        assert f"--devices and {flag} exclude each other" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        ev.parse_args(_evaluate_argv(tmp_path, "--devices", "0,x"))
    assert "argument --devices" in capsys.readouterr().err


# ------------------------------------------------------------------------------------------------------------------------- stub jobs
# module-level, so that the spawned workers find them by name

def sleepy_job(device, payload, next_item, emit):
    for key, seconds in iter(next_item, None):
        time.sleep(seconds)
        emit(key, {"key": key, "pid": os.getpid(), "finished": time.time()})


def first_last_job(device, payload, next_item, emit):
    """key 0 finishes only after every other key has: the worker that holds it waits for the file the last key writes"""
    for key, last in iter(next_item, None):
        if key == 0:
            deadline = time.time() + 120
            while not os.path.exists(payload) and time.time() < deadline:
                time.sleep(0.01)
        emit(key, {"key": key, "pid": os.getpid(), "finished": time.time()})
        if key == last:
            open(payload, "w").close()


def failing_job(device, payload, next_item, emit):
    for key, _ in iter(next_item, None):
        if key == payload:
            raise ValueError(f"refused file {key}.wav")
        time.sleep(0.05)
        emit(key, key)


def stuck_job(device, payload, next_item, emit):
    for key, _ in iter(next_item, None):
        emit(key, key)
        time.sleep(600)


def pid_job(device, payload, next_item, emit):
    for key, _ in iter(next_item, None):
        emit(key, os.getpid())
        time.sleep(600)


def _alive(pid):
    """the process exists and is not a zombie"""
    try:
        with open(f"/proc/{pid}/stat") as f:
            return f.read().rsplit(")", 1)[1].split()[0] not in ("Z", "X")
    except FileNotFoundError:
        return False


@pytest.mark.parametrize("sig", [signal.SIGTERM, signal.SIGHUP, signal.SIGKILL], ids=["sigterm", "sighup", "sigkill"])
def test_no_worker_outlives_a_command_ended_by_a_signal(sig):
    code = ("import sys; sys.path[:0] = [{root!r}, {tests!r}]; import test_workers as t; from streamspeech_b200 import workers\n"
            "for _, pid in workers.run([0, 0], t.pid_job, None, [(k, None) for k in range(6)]): print(pid, flush=True)"
            ).format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    p = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        pids = [int(p.stdout.readline()) for _ in range(2)]  # each worker holds an item and sleeps
        assert len(set(pids)) == 2 and all(_alive(pid) for pid in pids)
        p.send_signal(sig)
        p.wait(timeout=60)
    finally:
        if p.poll() is None:
            p.kill()
            p.wait()
    if sig != signal.SIGKILL:
        assert p.returncode == 128 + sig, p.stderr.read()[-2000:]
    deadline = time.time() + 10
    while any(_alive(pid) for pid in pids) and time.time() < deadline:
        time.sleep(0.05)
    assert not any(_alive(pid) for pid in pids)


def test_results_come_back_in_key_order_whatever_order_the_workers_finish_in(tmp_path):
    items = [(k, 7) for k in range(8)]
    with closing(workers.run([0, 0, 0], first_last_job, str(tmp_path / "last_done"), items)) as results:
        got = list(results)
    assert [k for k, _ in got] == list(range(8)) and all(r["key"] == k for k, r in got)
    finished = [r["finished"] for _, r in got]
    assert finished[0] > max(finished[1:])  # key 0 finished last
    assert len({r["pid"] for _, r in got}) >= 2 and os.getpid() not in {r["pid"] for _, r in got}
    assert multiprocessing.active_children() == []


def test_keys_keep_the_order_of_the_items_not_their_sort_order():
    items = [(k, 0.01 * (k % 3)) for k in (7, 2, 9, 0, 5)]
    assert [k for k, _ in workers.run([0, 0], sleepy_job, None, items)] == [7, 2, 9, 0, 5]
    assert list(workers.run([0], sleepy_job, None, [])) == []
    assert multiprocessing.active_children() == []


def test_a_worker_error_stops_every_worker_and_names_its_device():
    with pytest.raises(workers.WorkerFailed, match=r"worker on device 3 failed: ValueError: refused file 5\.wav"):
        with closing(workers.run([3], failing_job, 5, [(k, None) for k in range(20)])) as results:
            for _ in results:
                pass
    assert multiprocessing.active_children() == []
    with pytest.raises(workers.WorkerFailed, match=r"failed: ValueError: refused file 2\.wav"):
        list(workers.run([0, 1, 0], failing_job, 2, [(k, None) for k in range(40)]))
    assert multiprocessing.active_children() == []


def test_a_worker_error_exits_the_command_non_zero_with_its_message():
    code = ("import sys; sys.path[:0] = [{root!r}, {tests!r}]; import test_workers as t; from streamspeech_b200 import workers; "
            "list(workers.run([0, 0], t.failing_job, 3, [(k, None) for k in range(10)]))").format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert p.returncode != 0
    assert "WorkerFailed: worker on device 0 failed: ValueError: refused file 3.wav" in p.stderr


def test_a_caller_that_stops_early_leaves_no_child_behind():
    results = workers.run([0, 0], stuck_job, None, [(k, None) for k in range(4)])
    with closing(results):
        assert next(results)[0] == 0
    assert multiprocessing.active_children() == []


# ------------------------------------------------------------------------------------------------------------ evaluate's log merge

class StubEngine:
    def close(self):
        pass


class ClosingAgent(RecordingAgent):
    engine = StubEngine()


def stub_agents(args, max_seconds):
    return [ClosingAgent(j, []) for j in range(args.streams)], None, "text"


def stub_evaluate_job(device, payload, next_item, emit):
    """evaluate's worker with recording agents in place of the GPU agents"""
    ev.build_agents = stub_agents
    ev._evaluate_job(device, payload, next_item, emit)


@pytest.mark.parametrize("start,end,streams", [(0, -1, 1), (2, 8, 2), (7, -1, 3), (3, 3, 1)])
def test_instance_log_is_merged_in_index_order(tmp_path, monkeypatch, capsys, start, end, streams):
    _source_list(tmp_path, LENGTHS)
    flags = ["--start-index", str(start), "--end-index", str(end), "--streams", str(streams), "--sample-rate", "16000",
             "--source-segment-size", "320"]
    if start != end:
        flags += ["--quality-metrics", "BLEU", "--latency-metrics", "AL", "AP", "NumChunks", "RTF"]
    monkeypatch.setattr(ev, "build_agents", stub_agents)
    ev.main(_evaluate_argv(tmp_path, *flags, out="single"))
    monkeypatch.setattr(ev, "build_agents", lambda *a, **k: pytest.fail("the parent builds no agent"))
    monkeypatch.setattr(ev, "_evaluate_job", stub_evaluate_job)
    run = ev.main(_evaluate_argv(tmp_path, *flags, "--devices", "0,0,0", out="multi"))
    printed = [json.loads(x) for x in capsys.readouterr().out.splitlines() if x.startswith("{")]
    assert "devices" not in printed[0] and printed[-1]["devices"] == "0,0,0" and printed[-1]["streams"] == streams
    assert list(printed[-1]) == list(printed[0])[:2] + ["devices"] + list(printed[0])[2:]
    want = list(ev.get_indices(start, end, len(LENGTHS)))
    lines = (tmp_path / "multi" / "instances.log").read_text().splitlines()
    assert [json.loads(x)["index"] for x in lines] == want
    ref = (tmp_path / "single" / "instances.log").read_text().splitlines()
    assert [_no_elapsed(x) for x in lines] == [_no_elapsed(x) for x in ref]
    assert (tmp_path / "multi" / "config.yaml").read_text() == "source_type: speech\ntarget_type: speech\n"
    if start != end:
        assert list(run.kept) == want
        for name in ("scores.tsv", "metrics.tsv"):
            assert (tmp_path / "multi" / name).read_bytes() == (tmp_path / "single" / name).read_bytes()
    assert multiprocessing.active_children() == []
