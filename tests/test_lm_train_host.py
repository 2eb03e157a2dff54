"""CPU tests of the LM training entry point's host side (end2end-asr-pytorch_b200/lm_train.py).

  * Corpus: the word stream of a synthetic manifest pair -- mixed Chinese and English transcripts, upper case, characters
    outside the label set, an empty transcript, trailing newlines -- equals what the UNMODIFIED reference makes of the
    same files: SpectrogramDataset.parse_transcript (utils/data_loader.py), then calculate_lm_score's string step
    (utils/lstm_utils.py:9-44, recorded at its LM.evaluate call) split, plus '<eos>'.  Modules the reference imports but
    this does not use are stubbed as tests/test_loader_host.py stubs them (librosa, torchaudio).
  * Vocabulary: '<eos>' 0, '<oov>' 1, then first appearance; validation words outside it are '<oov>'.
  * Batches: batchify / get_batch windows equal the reference LM's.
  * Checkpoint: keys and types, torch.load with its default arguments (weights_only), b200asr.LM and the reference's LM.
  * The learning-rate rule, and the CLI failing on a machine without a GPU."""
import importlib
import json
import os
import subprocess
import sys
import types

import pytest
import torch

import b200asr
from oracle import ref_shim

LT = b200asr.lm_train
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")

LABELS = list("abcdefghijklmnopqrstuvwxyz' ") + list("你好世界今天我们") + ["a"]       # "a" twice: kept once
TRAIN = [
    "Hello World\n",
    "你好 世界\n\n",
    "今天 we GO 你好home\n",
    "",                                       # empty transcript: no LM string
    "### !!!\n",                              # nothing inside the label set
    "  Hello   我们  ok  \n",
    "MIXED我们case 天 world\n",
]
VALID = ["hello 世界 unknown\n", "新 words 今天\n", "\n"]


def _write_corpus(tmp_path):
    paths = {}
    for tag, texts in (("train", TRAIN), ("valid", VALID)):
        lines = []
        for i, t in enumerate(texts):
            p = tmp_path / f"{tag}{i}.txt"
            p.write_text(t, encoding="utf8")
            lines.append(f"{tmp_path}/{tag}{i}.wav,{p}")
        m = tmp_path / f"{tag}.csv"
        m.write_text("\n".join(lines) + "\n\n")
        paths[tag] = str(m)
    labels = tmp_path / "labels.json"
    labels.write_text(json.dumps(LABELS, ensure_ascii=False))
    return paths["train"], paths["valid"], str(labels)


def test_labels_are_built_as_train_py_builds_them(tmp_path):
    _, _, labels = _write_corpus(tmp_path)
    l2i, i2l = LT.load_labels(labels)
    chars = ["¶", "§", "¤"] + LABELS[:-1]
    assert l2i == {c: i for i, c in enumerate(chars)} and i2l == dict(enumerate(chars))


def test_vocabulary_order_and_oov(tmp_path):
    train, valid, labels = _write_corpus(tmp_path)
    l2i, i2l = LT.load_labels(labels)
    c = LT.Corpus([train], [valid], l2i, i2l)
    assert c.idx2word[:2] == ["<eos>", "<oov>"] and c.word2idx["<eos>"] == 0 and c.word2idx["<oov>"] == 1
    assert c.idx2word[2:6] == ["hello", "world", "你", "好"]
    assert all(c.word2idx[w] == i for i, w in enumerate(c.idx2word)) and len(c.word2idx) == len(c.idx2word)
    seen = []
    for i in c.train.tolist():                              # ids after <eos> / <oov> appear in order of first appearance
        if i > 1 and i not in seen:
            seen.append(i)
    assert seen == list(range(2, len(c.idx2word)))
    valid_words = [c.idx2word[i] for i in c.valid.tolist()]
    assert valid_words == ["hello", "世", "界", "<oov>", "<eos>", "<oov>", "今", "天", "<eos>"]
    assert c.train.dtype == c.valid.dtype == torch.int64


def test_manifest_lines(tmp_path):
    m = tmp_path / "m.csv"
    m.write_text("a.wav,a.txt\n\nb.wav,b.txt,extra\n")
    assert LT.transcript_paths([str(m), str(m)]) == ["a.txt", "b.txt"] * 2
    m.write_text("a.wav,a.txt\nonly_one_field\n")
    with pytest.raises(ValueError, match="m.csv:2: expected 'audio,transcript'"):
        LT.transcript_paths([str(m)])


@pytest.fixture
def ref(monkeypatch):
    """The reference's data_loader and lstm_utils modules, imported with librosa / torchaudio stubbed."""
    import scipy.signal
    for name in ("hamming", "hann", "blackman", "bartlett"):
        if not hasattr(scipy.signal, name):
            monkeypatch.setattr(scipy.signal, name, getattr(scipy.signal.windows, name), raising=False)
    for name in ("librosa", "torchaudio"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except ImportError:
                monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
    if torch.utils.data.Sampler.__init__ is object.__init__:     # torch >= 2.2 dropped Sampler(data_source)
        monkeypatch.setattr(torch.utils.data.Sampler, "__init__", lambda self, data_source=None: None)
    ref_shim.load([])
    return importlib.import_module("utils.data_loader"), importlib.import_module("utils.lstm_utils")


def _reference_words(DL, lu, manifest, l2i, i2l):
    """The reference's word stream: parse_transcript, calculate_lm_score's string (the one it hands LM.evaluate) split,
    '<eos>'; transcripts whose string is empty never reach evaluate."""
    ds = types.SimpleNamespace(label2id=l2i)
    asked = []
    lm = types.SimpleNamespace(evaluate=lambda s: (asked.append(s), (0.0, 0))[1])
    words = []
    for line in open(manifest).readlines():
        fields = line.strip().split(",")
        if fields == [""]:
            continue
        ids = DL.SpectrogramDataset.parse_transcript(ds, fields[1])
        n = len(asked)
        if ids:
            lu.calculate_lm_score(torch.tensor([ids]), lm, i2l)
        if len(asked) > n:
            words += asked[-1].split() + ["<eos>"]
    return words


@needs_ref
def test_word_stream_matches_the_reference(tmp_path, ref):
    DL, lu = ref
    train, valid, labels = _write_corpus(tmp_path)
    l2i, i2l = LT.load_labels(labels)
    c = LT.Corpus([train], [valid], l2i, i2l)
    want = _reference_words(DL, lu, train, l2i, i2l)
    assert [c.idx2word[i] for i in c.train.tolist()] == want
    assert "hello" in want and "你" in want and "<eos>" in want          # the corpus exercises both kinds of run
    want_v = [w if w in c.word2idx else "<oov>" for w in _reference_words(DL, lu, valid, l2i, i2l)]
    assert [c.idx2word[i] for i in c.valid.tolist()] == want_v
    for p in [ln.strip().split(",")[1] for ln in open(train) if ln.strip()]:
        assert LT.parse_transcript(p, l2i) == DL.SpectrogramDataset.parse_transcript(types.SimpleNamespace(label2id=l2i), p)


@needs_ref
@pytest.mark.parametrize("n,bsz,bptt", [(25, 4, 3), (200, 20, 35), (1001, 10, 35), (40, 20, 35), (21, 10, 7)])
def test_batches_match_the_reference_lm(ref, n, bsz, bptt):
    _, lu = ref
    data = torch.randint(0, 50, (n,), generator=torch.Generator().manual_seed(n))
    mine, theirs = LT.batchify(data, bsz), lu.LM.batchify(None, data, bsz, False)
    assert torch.equal(mine, theirs)
    windows = 0
    for i in range(0, mine.size(0) - 1, bptt):
        (x, y), (rx, ry) = LT.get_batch(mine, i, bptt), lu.LM.get_batch(None, theirs, i, bptt)
        assert torch.equal(x, rx) and torch.equal(y, ry)
        windows += 1
    assert windows == (mine.size(0) - 1 + bptt - 1) // bptt


def _plain(v):
    """True iff v is built from CPU tensors and str / int / float / bool / list / dict only."""
    if torch.is_tensor(v):
        return v.device.type == "cpu"
    if isinstance(v, dict):
        return type(v) is dict and all(isinstance(k, str) and _plain(x) for k, x in v.items())
    if isinstance(v, list):
        return all(_plain(x) for x in v)
    return type(v) in (str, int, float, bool)


@pytest.mark.parametrize("tied", [False, True])
def test_checkpoint_round_trip(tmp_path, tied):
    train, valid, labels = _write_corpus(tmp_path)
    l2i, i2l = LT.load_labels(labels)
    corpus = LT.Corpus([train], [valid], l2i, i2l)
    args = LT.parser().parse_args(["--train-manifest-list", train, "--valid-manifest-list", valid, "--labels-path", labels,
                                   "--emsize", "16", "--nhid", "16" if tied else "12", "--nlayers", "2"] + (["--tied"] if tied else []))
    torch.manual_seed(0)
    model = b200asr.RNNModel("LSTM", len(corpus.idx2word), args.emsize, args.nhid, args.nlayers, args.dropout, args.tied)
    ck = LT.checkpoint(model, corpus, args)
    assert set(ck) == {"word2idx", "idx2word", "ntoken", "ninp", "nhid", "nlayers", "dropout", "tie_weights", "model_state_dict"}
    assert _plain(ck)
    assert (ck["ntoken"], ck["ninp"], ck["nhid"], ck["nlayers"], ck["dropout"], ck["tie_weights"]) == \
        (len(corpus.idx2word), 16, args.nhid, 2, 0.2, tied)
    path = tmp_path / "lm.pt"
    torch.save(ck, path)
    back = torch.load(path)                                  # default arguments: weights_only=True
    assert back["word2idx"] == corpus.word2idx and back["idx2word"] == corpus.idx2word
    lm = b200asr.LM(str(path))
    assert lm.word2idx == corpus.word2idx and lm.idx2word == corpus.idx2word
    for k, v in model.state_dict().items():
        assert torch.equal(lm.model.state_dict()[k], v), k
    assert (lm.model.decoder.weight is lm.model.encoder.weight) == tied


@needs_ref
def test_checkpoint_loads_into_the_reference_lm(tmp_path, ref):
    _, lu = ref
    train, valid, labels = _write_corpus(tmp_path)
    l2i, i2l = LT.load_labels(labels)
    corpus = LT.Corpus([train], [valid], l2i, i2l)
    args = LT.parser().parse_args(["--train-manifest-list", train, "--valid-manifest-list", valid, "--labels-path", labels,
                                   "--emsize", "10", "--nhid", "14"])
    model = b200asr.RNNModel("LSTM", len(corpus.idx2word), 10, 14, 2, 0.2, False)
    path = tmp_path / "lm.pt"
    torch.save(LT.checkpoint(model, corpus, args), path)
    lm = lu.LM(str(path))                                    # its torch.load(model_path): weights_only=True
    for k, v in model.state_dict().items():
        assert torch.equal(lm.model.state_dict()[k], v), k
    assert lm.seq_to_tensor("hello zzz 你")[1] == 1


def test_learning_rate_rule():
    lr, best, saved = 20.0, None, []
    for val in (5.0, 4.0, 4.5, 4.0, 3.9, float("nan"), 3.0):
        save, best, lr = LT.lr_after_epoch(val, best, lr)
        saved.append((save, best, lr))
    assert saved == [(True, 5.0, 20.0), (True, 4.0, 20.0), (False, 4.0, 5.0), (False, 4.0, 1.25), (True, 3.9, 1.25),
                     (False, 3.9, 0.3125), (True, 3.0, 0.3125)]


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_cli_fails_without_a_gpu(tmp_path):
    train, valid, labels = _write_corpus(tmp_path)
    save = tmp_path / "lm.pt"
    r = subprocess.run([sys.executable, "-m", "b200asr.lm_train", "--train-manifest-list", train, "--valid-manifest-list", valid,
                        "--labels-path", labels, "--save", str(save), "--epochs", "1"], cwd=ROOT, timeout=300, capture_output=True,
                       text=True, env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode != 0 and "b200asr.lm_train:" in r.stderr, (r.returncode, r.stderr[-2000:])
    assert not save.exists()
