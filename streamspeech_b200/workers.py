"""Worker processes for the front doors' `--devices LIST`: one process per entry, each with its own engine on that CUDA device.

The front doors (evaluate, generate, asr_bleu) split their work into keyed items: an instance index, a batch, a group of files.
`run` starts one `spawn` process per device, every worker pulls items from one shared queue as it frees up (so ragged items balance
themselves), and the parent receives each result with its key and yields the results in the order of the items, which is the order
the single-process run writes them in.  Processes rather than threads: the agents' per-call host work runs in Python and would
serialise on the GIL.  The parent builds no engine and does not initialise CUDA; each worker builds its engine from the same
arguments (a checkpoint file, or the seeded synthetic one), so no weights are sent between processes.

A worker that raises stops the run: the parent terminates the other workers, joins every child and raises WorkerFailed naming the
worker's device and repeating its error.  A KeyboardInterrupt in the parent does the same (workers ignore SIGINT, so the parent alone
decides), and so do SIGTERM and SIGHUP while `run` is active (they raise SystemExit(128 + signal) in the parent, as a scheduler or
`timeout` ending the command expects).  A parent killed outright (SIGKILL) cannot clean up, so each worker also watches its parent: on
Linux the kernel kills it when the parent dies (PR_SET_PDEATHSIG), elsewhere it exits at its next wait for an item.  No child outlives
the command.
"""
from __future__ import annotations

import argparse
import ctypes
import multiprocessing as mp
import os
import pickle
import queue
import signal
import sys
import threading
import traceback
from typing import Any, Callable, Iterator, List, Optional, Sequence, Tuple

# How long the parent waits for a message before it checks that every worker is still alive, and a worker waits for an item before
# it checks that its parent is
_POLL_SECONDS = 1.0
_PR_SET_PDEATHSIG = 1  # <linux/prctl.h>


class WorkerFailed(RuntimeError):
    """a worker raised, or died, before the run finished"""


def parse_devices(text: str) -> List[int]:
    """`--devices 0,1` -> [0, 1]: CUDA device indices (relative to CUDA_VISIBLE_DEVICES), one worker each; repeats allowed"""
    parts = text.split(",")
    if not text or any(not p.strip().isdigit() for p in parts):
        raise argparse.ArgumentTypeError(f"{text!r}: a comma-separated list of CUDA device indices, e.g. 0,1 or 0,0")
    return [int(p) for p in parts]


def add_devices_arg(parser: argparse.ArgumentParser):
    parser.add_argument("--devices", type=parse_devices, default=None, metavar="LIST",
                        help="comma-separated CUDA device indices: one worker process per entry, each with its own engine on that "
                             "device (repeats run several workers on one GPU); results are written in the single-process order")


def parse_with_devices(parser: argparse.ArgumentParser, argv: Optional[Sequence[str]], device_flag: str) -> argparse.Namespace:
    """parser.parse_args(argv), refusing --devices together with the single-device flag (device_flag, e.g. --device-index)"""
    action = next((a for a in parser._actions if device_flag in a.option_strings), None)
    if action is None:  # the parser does not know the flag yet (evaluate without --agent): it refuses argv itself
        return parser.parse_args(argv)
    default, action.default = action.default, None
    try:
        args = parser.parse_args(argv)
    finally:
        action.default = default
    if getattr(args, action.dest) is not None and args.devices is not None:
        parser.error(f"--devices and {device_flag} exclude each other: --devices names every device a worker runs on")
    if getattr(args, action.dest) is None:
        setattr(args, action.dest, default)
    return args


def _die_with_parent(parent_pid: int):
    """have the kernel SIGKILL this worker when the parent dies (Linux), and exit now if it already has"""
    if sys.platform.startswith("linux"):
        try:
            ctypes.CDLL(None, use_errno=True).prctl(_PR_SET_PDEATHSIG, int(signal.SIGKILL), 0, 0, 0)
        except (OSError, AttributeError):
            pass
    if os.getppid() != parent_pid:
        os._exit(1)


def _raise_system_exit(signum, frame):
    raise SystemExit(128 + signum)


def _worker(device: int, job: Callable, payload: Any, tasks, results, parent_pid: int):
    signal.signal(signal.SIGINT, signal.SIG_IGN)
    _die_with_parent(parent_pid)
    exhausted = False

    def next_item() -> Optional[Tuple[Any, Any]]:
        nonlocal exhausted
        if exhausted:
            return None
        while True:
            try:
                item = tasks.get(timeout=_POLL_SECONDS)
                break
            except queue.Empty:
                if os.getppid() != parent_pid:  # the parent died without stopping this worker
                    os._exit(1)
        exhausted = item is None
        return item

    def emit(key, value):
        results.put(("result", key, pickle.dumps(value)))  # pickled here, so an unpicklable result is this worker's error

    try:
        job(device, payload, next_item, emit)
    except BaseException as e:  # noqa: BLE001 (every failure is reported to the parent)
        traceback.print_exc()
        results.put(("error", device, "".join(traceback.format_exception_only(type(e), e)).strip()))
        return
    results.put(("done", device, None))


def run(devices: Sequence[int], job: Callable, payload: Any, items: Sequence[Tuple[Any, Any]]) -> Iterator[Tuple[Any, Any]]:
    """Run `job(device, payload, next_item, emit)` in one spawned process per entry of devices, over the (key, item) pairs of items,
    and yield (key, result) in the order of items.  next_item() returns the next (key, item) of the shared queue, or None once the
    queue is empty; emit(key, result) sends a result.  job, payload, items and results must pickle (job a module-level function).
    Use it under contextlib.closing (or run it to the end), so that the workers are stopped when the caller stops early."""
    if not items:
        return
    ctx = mp.get_context("spawn")
    tasks, results = ctx.Queue(), ctx.Queue()
    keys = [k for k, _ in items]
    for it in items:
        tasks.put(it)
    for _ in devices:
        tasks.put(None)
    procs = [ctx.Process(target=_worker, args=(d, job, payload, tasks, results, os.getpid()), daemon=True) for d in devices]
    started: List = []
    handlers = {}
    if threading.current_thread() is threading.main_thread():  # signal handlers can only be set there
        for sig in (signal.SIGTERM, signal.SIGHUP):
            handlers[sig] = signal.signal(sig, _raise_system_exit)
    try:
        for p in procs:
            p.start()
            started.append(p)
        pending, pos, finished = {}, 0, 0
        while pos < len(keys):
            try:
                kind, key, value = results.get(timeout=_POLL_SECONDS)
            except queue.Empty:
                for d, p in zip(devices, procs):
                    if p.exitcode not in (None, 0):
                        raise WorkerFailed(f"worker on device {d} exited with code {p.exitcode}") from None
                continue
            if kind == "error":
                raise WorkerFailed(f"worker on device {key} failed: {value}")
            if kind == "done":
                finished += 1  # a worker's results reach the queue before its "done"
                if finished == len(procs):
                    raise WorkerFailed(f"the workers finished without results for {len(keys) - pos - len(pending)} items")
                continue
            pending[key] = value
            while pos < len(keys) and keys[pos] in pending:
                yield keys[pos], pickle.loads(pending.pop(keys[pos]))
                pos += 1
        for p in started:
            p.join()
    finally:
        for sig in handlers:  # a second signal does not cut the clean-up short
            signal.signal(sig, signal.SIG_IGN)
        for p in started:
            if p.is_alive():
                p.terminate()
        for p in started:
            p.join()
        for q in (tasks, results):
            q.cancel_join_thread()
            q.close()
        for sig, handler in handlers.items():
            signal.signal(sig, handler)
