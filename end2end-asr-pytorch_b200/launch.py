"""Data-parallel launcher for the reference's train.py and test.py: one process per GPU, in place of `--parallel`
(nn.DataParallel).

    python -m b200asr.launch [--quiet-ranks[=DIR]] train.py <train.py flags> [--parallel] [--device-ids 0 1 ...]
    python -m b200asr.launch [--quiet-ranks[=DIR]] test.py <test.py flags> [--device-ids 0 1 ...]

One child per entry of `--device-ids` (ids of the GPUs this process sees), or one per visible GPU without the flag.  Each
child sees only its own GPU (CUDA_VISIBLE_DEVICES), so train.py's `model.cuda(0)` and the trainer's `src.cuda()` land on
it, and gets the rendezvous environment (RANK, LOCAL_RANK, WORLD_SIZE, LOCAL_WORLD_SIZE, MASTER_ADDR, MASTER_PORT) plus
B200ASR_DIST_BACKEND: "nccl" when every rank has a GPU of its own, "gloo" when a GPU is listed twice (NCCL refuses two ranks
on one device).  The children run the script with `--parallel` and `--device-ids` removed, so the model is not wrapped in
nn.DataParallel and checkpoints carry no `module.` prefix.  `b200asr.install()` in the script joins the process group.
Ranks > 0 run with `--name <name>.rank<r>` (the reference's default name is `model`): train.py opens its log file
`log/<name>` in truncating mode before anything else, so ranks sharing one name would truncate and overwrite each
other's lines.  Rank 0 keeps the name, and only rank 0 saves checkpoints (to `<save-folder>/<name>`) and writes the
training loop's log lines; a rank > 0's own log holds what train.py itself logs before the loop.

--quiet-ranks (an option of the launcher, before the script) keeps ranks > 0 off the terminal: the stdout and stderr of
rank r > 0 go to DIR/launch.rank<r>.log (DIR defaults to the current directory), and the launcher names those files when
it ends.  test.py prints its progress bar and results on every rank; with the flag only rank 0's reach the terminal.

The launcher waits for every child.  When one fails, it terminates the others and exits with that child's code (128 + the
signal number for a child killed by a signal); on SIGINT / SIGTERM it terminates them all.  No child outlives it.
"""
from __future__ import annotations

import os
import signal
import socket
import subprocess
import sys
import threading
import time

_TERM_GRACE = 10.0          # seconds between SIGTERM and SIGKILL


REFERENCE_DEFAULT_NAME = "model"          # utils/constant.py: --name


def rank_name_args(args, rank: int):
    """args with --name suffixed by `.rank<r>` for rank r > 0 (added with the reference's default when absent)."""
    if rank == 0:
        return list(args)
    out, found, i = [], False, 0
    while i < len(args):
        a = args[i]
        if a == "--name" and i + 1 < len(args):
            out += [a, f"{args[i + 1]}.rank{rank}"]
            found = True
            i += 2
        elif a.startswith("--name="):
            out.append(f"{a}.rank{rank}")
            found = True
            i += 1
        else:
            out.append(a)
            i += 1
    if not found:
        out += ["--name", f"{REFERENCE_DEFAULT_NAME}.rank{rank}"]
    return out


def split_device_ids(argv):
    """(argv without --parallel / --device-ids, the --device-ids values as ints or None)."""
    out, ids, i = [], None, 0
    while i < len(argv):
        a = argv[i]
        if a == "--parallel":
            i += 1
        elif a == "--device-ids":
            i += 1
            ids = []
            while i < len(argv) and not argv[i].startswith("-"):
                ids.append(int(argv[i]))
                i += 1
            if not ids:
                raise ValueError("--device-ids expects at least one id")
        elif a.startswith("--device-ids="):
            ids = [int(a.split("=", 1)[1])]
            i += 1
        else:
            out.append(a)
            i += 1
    return out, ids


def visible_devices(env=None):
    """The GPUs this process sees, as the strings CUDA_VISIBLE_DEVICES takes."""
    env = os.environ if env is None else env
    vis = env.get("CUDA_VISIBLE_DEVICES")
    if vis is not None:
        return [d.strip() for d in vis.split(",") if d.strip()]
    import torch
    return [str(i) for i in range(torch.cuda.device_count())]


def backend_for(devices) -> str:
    """NCCL when every rank has its own GPU, gloo when two ranks share one."""
    return "nccl" if len(set(devices)) == len(devices) else "gloo"


def free_port(addr="127.0.0.1") -> int:
    with socket.socket() as s:
        s.bind((addr, 0))
        return s.getsockname()[1]


def plan(argv, env=None):
    """([per-rank argv tail], [per-rank environment]) for `launch argv`: argv[0] is the script."""
    env = dict(os.environ if env is None else env)
    if not argv:
        raise ValueError("usage: python -m b200asr.launch SCRIPT [ARGS...]")
    args, ids = split_device_ids(argv)
    visible = visible_devices(env)
    if ids is None:
        ids = list(range(len(visible)))
    if not ids:
        raise ValueError("no GPU visible and no --device-ids given")
    bad = [d for d in ids if not 0 <= d < len(visible)]
    if bad:
        raise ValueError(f"--device-ids {bad}: only {len(visible)} GPU(s) visible")
    devices = [visible[d] for d in ids]
    world = len(devices)
    addr = env.get("MASTER_ADDR", "127.0.0.1")
    port = str(free_port(addr))
    backend = backend_for(devices)
    envs = []
    for rank, dev in enumerate(devices):
        e = dict(env)
        e.update(CUDA_VISIBLE_DEVICES=dev, RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world),
                 LOCAL_WORLD_SIZE=str(world), MASTER_ADDR=addr, MASTER_PORT=port, B200ASR_DIST_BACKEND=backend)
        envs.append(e)
    return [[args[0]] + rank_name_args(args[1:], r) for r in range(world)], envs


def launcher_options(argv):
    """(directory for the output of ranks > 0, or None to leave it on the terminal; argv from the script on).  The
    launcher's own options come before the script: --quiet-ranks (the current directory) or --quiet-ranks=DIR."""
    quiet, i = None, 0
    while i < len(argv) and argv[i].startswith("-"):
        a = argv[i]
        if a == "--quiet-ranks":
            quiet = "."
        elif a.startswith("--quiet-ranks="):
            quiet = a.split("=", 1)[1] or "."
        else:
            raise ValueError(f"unknown launcher option {a!r}; usage: python -m b200asr.launch [--quiet-ranks[=DIR]] SCRIPT [ARGS...]")
        i += 1
    return quiet, argv[i:]


def rank_log_path(directory, rank: int) -> str:
    return os.path.join(directory, f"launch.rank{rank}.log")


def _exit_code(rc: int) -> int:
    return 128 - rc if rc < 0 else rc


def _stop(procs):
    """SIGTERM every child still running, SIGKILL what is left after the grace period, and reap them all."""
    for p in procs:
        if p.poll() is None:
            p.terminate()
    deadline = time.monotonic() + _TERM_GRACE
    for p in procs:
        try:
            p.wait(timeout=max(0.0, deadline - time.monotonic()))
        except subprocess.TimeoutExpired:
            p.kill()
            p.wait()


def run(argv, env=None, poll=0.1) -> int:
    """Start the children, wait for them; the exit code of the launcher.  argv: the launcher's options, the script and its
    arguments."""
    quiet, argv = launcher_options(argv)
    args, envs = plan(argv, env)
    procs, logs = [], []

    def on_signal(signum, frame):
        raise KeyboardInterrupt

    old = {}
    if threading.current_thread() is threading.main_thread():
        old[signal.SIGTERM] = signal.signal(signal.SIGTERM, on_signal)
    try:
        if quiet is not None and len(args) > 1:
            os.makedirs(quiet, exist_ok=True)
        for rank, (a, e) in enumerate(zip(args, envs)):
            out = None
            if quiet is not None and rank > 0:
                out = open(rank_log_path(quiet, rank), "w")
                logs.append(out)
            procs.append(subprocess.Popen([sys.executable] + a, env=e, stdout=out,
                                          stderr=subprocess.STDOUT if out is not None else None))
        while True:
            codes = [p.poll() for p in procs]
            failed = [c for c in codes if c not in (None, 0)]
            if failed:
                _stop(procs)
                return _exit_code(failed[0])
            if all(c == 0 for c in codes):
                return 0
            time.sleep(poll)
    except KeyboardInterrupt:
        _stop(procs)
        return 130
    finally:
        _stop(procs)
        for f in logs:
            f.close()
        if logs:
            print("b200asr.launch: the output of ranks > 0 is in " + ", ".join(f.name for f in logs), file=sys.stderr)
        for s, h in old.items():
            signal.signal(s, h)


if __name__ == "__main__":
    try:
        code = run(sys.argv[1:])
    except ValueError as e:
        print(f"b200asr.launch: {e}", file=sys.stderr)
        code = 2
    sys.exit(code)
