"""The data-parallel launcher (b200asr.launch) and the host arithmetic of the data-parallel Trainer.train, without a GPU:
  * per-rank environment and argv rewriting, backend choice for distinct and repeated device ids;
  * a failing child terminates the others, its exit code propagates, no child outlives the launcher;
  * shard sizes equal torch.chunk's (nn.DataParallel.scatter);
  * the reduced metric row gives the reference's batch loss (CE over the gathered tokens, CTC reduction="mean" over the
    gathered utterances) and its CER / WER sums.
"""
import importlib
import os
import subprocess
import sys
import textwrap
import time

import pytest
import torch

import b200asr
from oracle import asr_oracle as O

launch = importlib.import_module(b200asr.__name__ + ".launch")
parallel = importlib.import_module(b200asr.__name__ + ".parallel")
trainer = importlib.import_module(b200asr.__name__ + ".trainer")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_argv_rewriting_drops_parallel_and_device_ids():
    args, ids = launch.split_device_ids(["train.py", "--parallel", "--device-ids", "0", "1", "--batch-size", "8", "--cuda"])
    assert args == ["train.py", "--batch-size", "8", "--cuda"] and ids == [0, 1]
    args, ids = launch.split_device_ids(["train.py", "--cuda", "--device-ids", "3"])
    assert args == ["train.py", "--cuda"] and ids == [3]
    args, ids = launch.split_device_ids(["train.py", "--device-ids=2", "--epochs", "1"])
    assert args == ["train.py", "--epochs", "1"] and ids == [2]
    assert launch.split_device_ids(["train.py", "--lr", "1"]) == (["train.py", "--lr", "1"], None)
    with pytest.raises(ValueError):
        launch.split_device_ids(["train.py", "--device-ids", "--cuda"])


def test_per_rank_environment_and_backend():
    env = {"CUDA_VISIBLE_DEVICES": "4,5,6", "PATH": "/bin"}
    args, envs = launch.plan(["train.py", "--parallel", "--device-ids", "0", "2", "--cuda"], env)
    assert args == [["train.py", "--cuda"], ["train.py", "--cuda", "--name", "model.rank1"]]
    assert [e["CUDA_VISIBLE_DEVICES"] for e in envs] == ["4", "6"]
    assert [e["RANK"] for e in envs] == ["0", "1"] == [e["LOCAL_RANK"] for e in envs]
    assert all(e["WORLD_SIZE"] == "2" and e["LOCAL_WORLD_SIZE"] == "2" for e in envs)
    assert len({e["MASTER_PORT"] for e in envs}) == 1 and int(envs[0]["MASTER_PORT"]) > 0
    assert all(e["MASTER_ADDR"] == "127.0.0.1" and e["PATH"] == "/bin" for e in envs)
    assert all(e[parallel.BACKEND_ENV] == "nccl" for e in envs)
    args, envs = launch.plan(["train.py", "--name", "x", "--device-ids", "0", "0"], env)   # two ranks on one GPU: gloo
    assert args == [["train.py", "--name", "x"], ["train.py", "--name", "x.rank1"]]
    assert [e["CUDA_VISIBLE_DEVICES"] for e in envs] == ["4", "4"] and all(e[parallel.BACKEND_ENV] == "gloo" for e in envs)
    _, envs = launch.plan(["train.py"], env)                                   # no --device-ids: every visible GPU
    assert [e["CUDA_VISIBLE_DEVICES"] for e in envs] == ["4", "5", "6"] and envs[2]["RANK"] == "2"
    assert launch.backend_for(["0", "1"]) == "nccl" and launch.backend_for(["1", "0", "1"]) == "gloo"
    with pytest.raises(ValueError):
        launch.plan(["train.py", "--device-ids", "3"], env)
    with pytest.raises(ValueError):
        launch.plan(["train.py"], {"CUDA_VISIBLE_DEVICES": ""})


def test_ranks_after_the_first_get_their_own_name():
    """train.py opens log/<name> in truncating mode: ranks > 0 run with <name>.rank<r>, rank 0 with the name as given."""
    assert launch.rank_name_args(["--name", "asr", "--cuda"], 0) == ["--name", "asr", "--cuda"]
    assert launch.rank_name_args(["--name", "asr", "--cuda"], 2) == ["--name", "asr.rank2", "--cuda"]
    assert launch.rank_name_args(["--name=asr"], 1) == ["--name=asr.rank1"]
    assert launch.rank_name_args(["--cuda"], 3) == ["--cuda", "--name", "model.rank3"]


def _script(tmp_path, body):
    p = tmp_path / "child.py"
    p.write_text(textwrap.dedent(body))
    return str(p)


def _alive(pid):
    try:
        os.kill(pid, 0)
    except ProcessLookupError:
        return False
    try:                                       # a zombie of another parent counts as gone
        with open(f"/proc/{pid}/stat") as f:
            return f.read().split(")")[-1].split()[0] != "Z"
    except OSError:
        return False


def test_children_get_their_environment_and_argv(tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    script = _script(tmp_path, f"""
        import json, os, sys
        keys = ("RANK", "WORLD_SIZE", "CUDA_VISIBLE_DEVICES", "B200ASR_DIST_BACKEND", "MASTER_PORT")
        with open(os.path.join({str(out)!r}, os.environ["RANK"]), "w") as f:
            json.dump(dict(argv=sys.argv[1:], **{{k: os.environ[k] for k in keys}}), f)
        """)
    rc = launch.run([script, "--parallel", "--x", "1", "--device-ids", "1", "1"], dict(os.environ, CUDA_VISIBLE_DEVICES="0,7"))
    assert rc == 0
    import json
    got = [json.loads((out / str(r)).read_text()) for r in range(2)]
    assert got[0]["argv"] == ["--x", "1"] and got[1]["argv"] == ["--x", "1", "--name", "model.rank1"]
    for r, g in enumerate(got):
        assert g["RANK"] == str(r) and g["WORLD_SIZE"] == "2"
        assert g["CUDA_VISIBLE_DEVICES"] == "7" and g["B200ASR_DIST_BACKEND"] == "gloo"
    assert got[0]["MASTER_PORT"] == got[1]["MASTER_PORT"]


def test_failing_child_terminates_the_others_and_its_code_propagates(tmp_path):
    pids = tmp_path / "pids"
    pids.mkdir()
    script = _script(tmp_path, f"""
        import os, sys, time
        open(os.path.join({str(pids)!r}, str(os.getpid())), "w").close()
        if os.environ["RANK"] == "1":
            time.sleep(0.5)
            sys.exit(7)
        time.sleep(120)
        """)
    t0 = time.monotonic()
    rc = launch.run([script, "--device-ids", "0", "0", "0"], dict(os.environ, CUDA_VISIBLE_DEVICES="0"))
    assert rc == 7
    assert time.monotonic() - t0 < 60
    started = [int(p) for p in os.listdir(pids)]
    assert len(started) == 3
    assert not any(_alive(p) for p in started)


def test_launcher_module_runs_as_a_script(tmp_path):
    """python -m b200asr.launch from the repository tree: the exit code of a failing child, usage errors as code 2."""
    script = _script(tmp_path, "import os, sys; sys.exit(3 if os.environ['RANK'] == '0' else 0)\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0,1")
    r = subprocess.run([sys.executable, "-m", "b200asr.launch", script], cwd=ROOT, env=env, timeout=120)
    assert r.returncode == 3
    r = subprocess.run([sys.executable, "-m", "b200asr.launch"], cwd=ROOT, env=env, timeout=120, capture_output=True)
    assert r.returncode == 2 and b"usage" in r.stderr


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("B", [1, 2, 5, 32])
def test_shard_sizes_equal_torch_chunk(B, world):
    chunks = torch.arange(B).chunk(world)
    for rank in range(world):
        a, b = parallel.shard_range(B, rank, world)
        want = chunks[rank].tolist() if rank < len(chunks) else []
        assert list(range(a, b)) == want, (B, world, rank)


def _counts(hyp, gold):
    """trainer.py:96-104 for one utterance pair of strings."""
    from oracle.ref_shim import _edit_distance
    h, g = hyp, gold
    return (_edit_distance(h.replace(" ", ""), g.replace(" ", "")), _edit_distance_words(h, g),
            len(g.replace(" ", "")), len(g.split(" ")))


def _edit_distance_words(h, g):
    from oracle.ref_shim import _edit_distance
    words = {w: chr(0x4E00 + i) for i, w in enumerate(set(h.split() + g.split()))}
    return _edit_distance("".join(words[w] for w in h.split()), "".join(words[w] for w in g.split()))


@pytest.mark.parametrize("world", [2, 3])
def test_reduced_row_gives_the_reference_batch_loss_and_counts(world):
    g = torch.Generator().manual_seed(3)
    B, T, V = 5, 7, 11
    pred = torch.randn(B, T, V, generator=g, dtype=torch.float64)
    gold = torch.randint(1, V, (B, T), generator=g)
    gold[1, 4:] = 0; gold[3, 2:] = 0; gold[4, 1:] = 0
    hyps = ["ab c", "abc", "a bb", "", "x y z"]
    golds = ["ab c", "ab", "a b b", "c", "x z"]
    # CE, label-smoothed: the reference's loss is the sum over the non-PAD tokens / their number (utils/metrics.py:102-131)
    ref_loss, _ = O.cross_entropy_loss(pred, gold, 0.1)
    # CTC, reduction="mean": mean over the utterances of nll_b / target_length_b
    logp = torch.randn(9, B, V, generator=g, dtype=torch.float64).log_softmax(-1)
    tl = torch.tensor([3, 2, 3, 1, 2])
    il = torch.full((B,), 9)
    ref_ctc = torch.nn.functional.ctc_loss(logp, gold[:, :3].clamp_min(1), il, tl, reduction="mean")
    rows = []
    for rank in range(world):
        a, b = parallel.shard_range(B, rank, world)
        row = [0.0] * len(trainer.ROW)
        if b > a:
            l, n = O.cross_entropy_loss(pred[a:b], gold[a:b], 0.1)
            row[0], row[1] = float(l) * n, n
            for h, gg in zip(hyps[a:b], golds[a:b]):
                for k, c in enumerate(_counts(h, gg)):
                    row[2 + k] += c
        ctc = (torch.nn.functional.ctc_loss(logp[:, a:b], gold[a:b, :3].clamp_min(1), il[a:b], tl[a:b], reduction="mean") * (b - a)
               if b > a else torch.tensor(0.0))
        rows.append((row, float(ctc), b - a))
    total = [sum(r[0][k] for r in rows) for k in range(len(trainer.ROW))]
    assert trainer.loss_value(total) == pytest.approx(float(ref_loss), rel=1e-12)
    assert trainer.loss_value([sum(r[1] for r in rows), sum(r[2] for r in rows)]) == pytest.approx(float(ref_ctc), rel=1e-12)
    want = [sum(_counts(h, gg)[k] for h, gg in zip(hyps, golds)) for k in range(4)]
    assert total[2:6] == want and total[6] == 0
    assert trainer.loss_value([float("inf"), 3.0]) == float("inf")                  # an infinite shard skips the batch
