"""Data-parallel Transformer.evaluate without a GPU (modules.evaluate_sharded / decode_sharded, parallel.gather_rows):
gloo ranks on the CPU with the front end, the encoder and the two decodes stubbed, against the same stubs run by one
process on the whole batch:
  * rank r is handed utterances r, r + N, ... of the batch (inputs and lengths), at the batch's padded T, and a rank with
    no utterance decodes nothing;
  * every rank returns greedy_strings / the beam join of the whole batch, in batch order, for every B in 1..9 and N <= 4;
  * an utterance that ends no beam hypothesis on any one rank makes every rank print ">>>>>>> switch to greedy" once and
    return the greedy strings of the whole batch;
  * encoded_frames gives the length the vgg_cnn / emb_cnn front ends produce;
and the launcher's --quiet-ranks: ranks > 0 write nothing to the terminal, their output lands in the files the launcher
names, and without the flag every rank's output reaches the terminal as before.
"""
import contextlib
import importlib
import io
import os
import socket
import subprocess
import sys
import textwrap
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import b200asr

M = importlib.import_module(b200asr.__name__ + ".modules")
launch = importlib.import_module(b200asr.__name__ + ".launch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

V = 12
BATCHES = range(1, 10)
LABELS = {i: c for i, c in enumerate([M.PAD_CHAR, M.SOS_CHAR, M.EOS_CHAR] + [chr(0x61 + i) for i in range(V - 3)])}


# ------------------------------------------------------------------------------------------ stubs
def _utt(enc):
    """The utterance index each row of a stub encoder output carries."""
    return [int(x) for x in enc[:, 0, 0]]


def stub_greedy(dec, enc, steps=300, stop_at_eos=False, check_every=8):
    """Utterance u: 3 + (5u mod 7) tokens, then its EOS as -1 (greedy_decode_cached(stop_at_eos=True)'s rows)."""
    dec.calls.append(("greedy", _utt(enc)))
    ys = torch.full((enc.shape[0], steps), -1, dtype=torch.long)
    for r, u in enumerate(_utt(enc)):
        n = 3 + (5 * u) % 7
        ys[r, :n] = torch.tensor([3 + (u + 2 * j) % (V - 3) for j in range(n)])
    return ys


def stub_beam(dec, enc, beam_width, nbest=1, c_weight=1.0, steps=300, check_every=8, lm=None, lm_weight=0.1):
    """Utterance u: yseq SOS, 1 + (3u mod 5) tokens, EOS; no hypothesis for the utterances in dec.no_hyp."""
    dec.calls.append(("beam", _utt(enc)))
    S = min(steps, enc.shape[1])
    ids = torch.full((enc.shape[0], 1, S + 2), -1, dtype=torch.long)
    lengths = torch.zeros((enc.shape[0], 1), dtype=torch.long)
    for r, u in enumerate(_utt(enc)):
        if u in dec.no_hyp:
            continue
        y = [1] + [3 + (2 * u + j) % (V - 3) for j in range(1 + (3 * u) % 5)] + [2]
        ids[r, 0, :len(y)] = torch.tensor(y)
        lengths[r, 0] = len(y)
    nan = torch.full((enc.shape[0], 1), float("nan"))
    return ids, lengths, nan, nan


def _model(no_hyp=()):
    dec = types.SimpleNamespace(id2label=LABELS, trg_max_length=301, calls=[], no_hyp=set(no_hyp))
    return types.SimpleNamespace(decoder=dec, encoder=None, id2label=LABELS, feat_extractor="")


def _batch(B, T=40):
    """padded_input [B, 1, 4, T] whose every entry of utterance u is u; lengths 10 + u."""
    src = torch.arange(B, dtype=torch.float32).view(B, 1, 1, 1).expand(B, 1, 4, T).contiguous()
    return src, torch.arange(B, dtype=torch.int32) + 10


def stub_front_end(self, x):
    return x.view(x.shape[0], -1, x.shape[-1]).transpose(1, 2).contiguous(), None


def _install_stubs():
    M.greedy_decode_cached, M.beam_decode, M._front_end = stub_greedy, stub_beam, stub_front_end
    M._gold_strings = lambda self, tgt: [f"gold{i}" for i in range(tgt.shape[0])]
    seen = []

    def encoder(enc_self, feats, lengths, cf=None):
        seen.append((_utt(feats), lengths.tolist(), feats.shape[1]))
        return feats
    M._encoder_body = encoder
    return seen


def _one_process(B, beam, no_hyp=()):
    """What one process's evaluate computes for the whole batch, with the same stubs."""
    model = _model(no_hyp)
    src, _ = _batch(B)
    enc = stub_front_end(model, src)[0]
    if beam:
        ids, lengths, _, _ = stub_beam(model.decoder, enc, 4)
        _, strs = M.beam_strings(torch.cat([lengths.unsqueeze(-1), ids], dim=-1), LABELS)
        if len(strs) == B:
            return strs
    return M.greedy_strings(stub_greedy(model.decoder, enc).tolist(), LABELS)


CASES = [("greedy", False, ()), ("beam", True, ()), ("fallback", True, (1,)), ("fallback-last", True, ("last",))]


def _arm(rank, world, port, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    seen = _install_stubs()
    group = (dist.group.WORLD, rank, world)
    res = {}
    for B in BATCHES:
        for name, beam, no_hyp in CASES:
            no_hyp = tuple(B - 1 if u == "last" else u for u in no_hyp)
            if any(u >= B for u in no_hyp):
                continue
            model = _model(no_hyp)
            src, lens = _batch(B)
            seen.clear()
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                hyps, gold = M.evaluate_sharded(model, group, src, lens, torch.zeros(B, 3), beam, 4, None, 0.1, 1.0)
            res[(B, name)] = dict(hyps=hyps, gold=gold, out=out.getvalue(), calls=list(model.decoder.calls), seen=list(seen))
    torch.save(res, os.path.join(tmp, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_decode_assembles_the_whole_batch(world, tmp_path):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    mp.start_processes(_arm, args=(world, port, str(tmp_path)), nprocs=world, join=True, start_method="spawn")
    ranks = [torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in range(world)]
    assert set(ranks[0]) == set(ranks[-1]) and len(ranks[0]) > 3 * len(BATCHES)
    for (B, name), r0 in ranks[0].items():
        beam, no_hyp = {n: (b, h) for n, b, h in CASES}[name]
        no_hyp = tuple(B - 1 if u == "last" else u for u in no_hyp)
        want = _one_process(B, beam, no_hyp)
        fallback = beam and len(no_hyp) > 0
        for rank, res in enumerate(ranks):
            got = res[(B, name)]
            mine = list(range(rank, B, world))
            assert got["hyps"] == want and got["gold"] == [f"gold{i}" for i in range(B)], (B, name, rank)
            assert got["out"] == (">>>>>>> switch to greedy\n" if fallback else ""), (B, name, rank)
            if not mine:                                   # an empty share: nothing decoded, every collective joined
                assert got["calls"] == [] and got["seen"] == [], (B, name, rank)
                continue
            assert got["seen"] == [(mine, [10 + u for u in mine], 40)], (B, name, rank)
            kinds = (["beam", "greedy"] if fallback else ["beam"]) if beam else ["greedy"]
            assert got["calls"] == [(k, mine) for k in kinds], (B, name, rank)


@pytest.mark.parametrize("feat", ["vgg_cnn", "emb_cnn", ""])
def test_encoded_frames_is_the_front_end_output_length(feat):
    cfg = b200asr.ASRConfig(num_layers=1, num_heads=2, dim_model=64, dim_key=32, dim_value=32, dim_inner=128, vocab=V,
                            feat_extractor=feat, tgt_max_len=301, dropout=0.0)
    model = b200asr.build_model(cfg, id2label=LABELS).eval()
    for T in (40, 41, 42, 43, 57, 300):
        if feat:
            with torch.no_grad():
                want = model.conv(torch.zeros(1, 1, 161, T)).shape[-1]
        else:
            want = T
        assert M.encoded_frames(model, T) == want, (feat, T)


# ------------------------------------------------------------------------------------------ launcher --quiet-ranks
def _script(tmp_path):
    p = tmp_path / "child.py"
    p.write_text(textwrap.dedent("""
        import os, sys
        r = os.environ["RANK"]
        os.write(1, f"out of rank {r}\\n".encode())        # one write per line: lines of ranks sharing a pipe stay whole
        os.write(2, f"err of rank {r}\\n".encode())
        """))
    return str(p)


def _launch(tmp_path, *opts):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0", PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "b200asr.launch", *opts, _script(tmp_path), "--device-ids", "0", "0", "0"],
                          cwd=tmp_path, env=env, timeout=120, capture_output=True, text=True)


def test_quiet_ranks_keep_ranks_after_the_first_off_the_terminal(tmp_path):
    r = _launch(tmp_path, f"--quiet-ranks={tmp_path / 'logs'}")
    assert r.returncode == 0, r.stderr
    assert r.stdout == "out of rank 0\n"
    assert "err of rank 0" in r.stderr and "rank 1" not in r.stderr and "rank 2" not in r.stderr
    for rank in (1, 2):
        path = launch.rank_log_path(str(tmp_path / "logs"), rank)
        assert path in r.stderr                                    # the launcher names the files it wrote
        with open(path) as f:
            assert sorted(f.read().splitlines()) == [f"err of rank {rank}", f"out of rank {rank}"]
    assert not os.path.exists(launch.rank_log_path(str(tmp_path / "logs"), 0))
    r = _launch(tmp_path, "--quiet-ranks")                         # the current directory
    assert r.returncode == 0 and r.stdout == "out of rank 0\n"
    assert os.path.exists(tmp_path / "launch.rank1.log") and os.path.exists(tmp_path / "launch.rank2.log")


def test_without_the_flag_every_rank_reaches_the_terminal(tmp_path):
    r = _launch(tmp_path)
    assert r.returncode == 0, r.stderr
    assert sorted(r.stdout.splitlines()) == [f"out of rank {k}" for k in range(3)]
    assert sorted(x for x in r.stderr.splitlines() if x.startswith("err")) == [f"err of rank {k}" for k in range(3)]
    assert "b200asr.launch" not in r.stderr
    assert not any(n.startswith("launch.rank") for n in os.listdir(tmp_path))


def test_launcher_options_come_before_the_script():
    assert launch.launcher_options(["train.py", "--quiet-ranks"]) == (None, ["train.py", "--quiet-ranks"])
    assert launch.launcher_options(["--quiet-ranks", "test.py", "--x"]) == (".", ["test.py", "--x"])
    assert launch.launcher_options(["--quiet-ranks=out", "test.py"]) == ("out", ["test.py"])
    with pytest.raises(ValueError, match="unknown launcher option"):
        launch.launcher_options(["--quiet", "test.py"])
    r = subprocess.run([sys.executable, "-m", "b200asr.launch", "--bogus", "x.py"], cwd=ROOT, timeout=120, capture_output=True)
    assert r.returncode == 2 and b"usage" in r.stderr
