"""The installed AudioDataLoader on the device (end2end-asr-pytorch_b200/loader.py) and b200asr_stft_features_packed.

* The packed entry point against b200asr_stft_features_ex on the same zero-padded batch: bit for bit.
* The installed loader against the unmodified one (stubbed as tests/test_loader_host.py stubs it, its stft
  tests/augment_oracle's float64 one), at num_workers 0 and 2, with and without noise; no host synchronisation.
* The reference's Trainer.train and test.py's evaluate over an installed loader against the same items collated by
  collate_waves with the noise draws the loader made."""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests.helpers import rel_err
from tests.test_gpu_linear_precisions import Banded, _waves

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_ARG, BAD_ALIGN = 0, -5, -2
GUARD = 1024
NO_CUT = 2 ** 31 - 1
BAR = 5e-5                                   # tests/test_gpu_feature_augment.py's 3xTF32 bar for collate_waves
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _call(L, waves, Tmax, packed, shift=0, window=0, noise=None, max_frames=NO_CUT, normalize=1, prec=3, order=None):
    """One raw call over NaN-poisoned buffers: padded ([B, Lmax], NaN past each length) or packed (back to back from
    `shift` floats into the buffer, in `order`, NaN between).  Returns (rc, out, frames, launches)."""
    lib = L.load()
    lens = [len(w) for w in waves]
    B, Lmax = len(waves), max(1, max(lens))
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ws = torch.full((lib.b200asr_stft_features_ex_ws_bytes(B, Lmax, 320, 160) // 4 + GUARD,), NAN, device="cuda")
    nws = ws.numel() - GUARD
    out = Banded((B, 1, 161, Tmax))
    frames = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    bank, bank_len, start, level = noise if noise is not None else (None, 0, None, None)
    st = torch.cuda.current_stream().cuda_stream
    if packed:
        order = list(range(B)) if order is None else order
        offs, pos = [0] * B, shift
        for b in order:
            offs[b] = pos
            pos += lens[b] + 3                                            # a NaN gap between utterances
        buf = torch.full((pos + 1,), NAN)
        for b in range(B):
            buf[offs[b]:offs[b] + lens[b]] = torch.from_numpy(waves[b])
        buf = buf.cuda()
        offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_stft_features_packed(L.ptr(buf), L.ptr(offsets), L.ptr(lt), L.ptr(out.t), L.ptr(frames), L.ptr(ws), B,
                                              Lmax, Tmax, 320, 160, 1, normalize, window, 0, L.ptr(bank), bank_len, L.ptr(start),
                                              L.ptr(level), max_frames, prec, st)
    else:
        buf = torch.full((B, Lmax), NAN)
        for b in range(B):
            buf[b, :lens[b]] = torch.from_numpy(waves[b])
        buf = buf.cuda()
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_stft_features_ex(L.ptr(buf), L.ptr(lt), L.ptr(out.t), L.ptr(frames), L.ptr(ws), B, Lmax, Tmax, 320, 160, 1,
                                          normalize, window, 0, L.ptr(bank), bank_len, L.ptr(start), L.ptr(level), max_frames, prec, st)
    n = lib.b200asr_launch_count() - n0
    torch.cuda.synchronize()
    assert bool(ws[nws:].isnan().all()) and out.bands_intact()
    return rc, out.t, frames, n


@pytest.mark.parametrize("B", [1, 33])
@pytest.mark.parametrize("window", [0, 1, 2, 3])
def test_packed_is_the_padded_call_bit_for_bit(L, B, window):
    """Lengths from 1 sample to 16 s, offsets at odd samples and in another order than the batch, with and without noise,
    with the cut binding and not, normalised and not: the bits and launches of b200asr_stft_features_ex."""
    g = np.random.default_rng(B * 10 + window)
    lens = ([256000] if B == 1 else [1, 159, 160, 161, 256000, 64000] + g.integers(2, 256000, B - 6).tolist())
    waves = _waves(lens, seed=B + window)
    bank_np = (0.3 * g.standard_normal(300000)).astype(np.float32)
    bank = torch.from_numpy(bank_np).cuda()
    starts = [int(g.integers(0, 300000 - n)) if b % 3 else -1 for b, n in enumerate(lens)]
    levels = g.uniform(0, 0.5, B).astype(np.float32)
    noise = (bank, bank.numel(), torch.tensor(starts, dtype=torch.int64, device="cuda"), torch.from_numpy(levels).cuda())
    order = g.permutation(B).tolist()
    T = 1 + max(lens) // 160
    for kw in (dict(), dict(noise=noise), dict(max_frames=700, noise=noise), dict(max_frames=T + 5), dict(normalize=0, noise=noise),
               dict(normalize=0, max_frames=3)):
        Tmax = min(T, kw.get("max_frames", T))
        a = _call(L, waves, Tmax, False, window=window, **kw)
        for shift in (1, 3):
            b = _call(L, waves, Tmax, True, shift=shift, window=window, order=order, **kw)
            assert a[0] == b[0] == OK and a[3] == b[3], kw
            assert torch.equal(a[2], b[2]) and torch.equal(a[1].nan_to_num(7.0), b[1].nan_to_num(7.0)), (kw, shift)
        assert bool(torch.isfinite(a[1]).all()), kw


def test_packed_rejections_launch_nothing(L):
    lib = L.load()
    waves = _waves([4000, 2500], seed=1)
    wave = torch.from_numpy(np.concatenate(waves + [np.zeros(8, np.float32)])).cuda()
    lens = torch.tensor([4000, 2500], dtype=torch.int32, device="cuda")
    offs = torch.tensor([0, 4000, 0], dtype=torch.int64, device="cuda")
    ws = torch.empty(lib.b200asr_stft_features_ex_ws_bytes(2, 4000, 320, 160) // 4, device="cuda")
    out = torch.full((2, 1, 161, 26), NAN, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(w=L.ptr(wave), o=L.ptr(offs), window=0):
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_stft_features_packed(w, o, L.ptr(lens), L.ptr(out), None, L.ptr(ws), 2, 4000, 26, 320, 160, 1, 1, window, 0,
                                              None, 0, None, None, NO_CUT, 3, st)
        return rc, lib.b200asr_launch_count() - n0

    assert call(o=None) == (BAD_ARG, 0) and call(w=None) == (BAD_ARG, 0)
    assert call(o=L.ptr(offs) + 4) == (BAD_ALIGN, 0) and call(w=L.ptr(wave) + 2) == (BAD_ALIGN, 0)
    assert call(window=5) == (BAD_ARG, 0) and "stft_features_packed" in L.last_error()
    torch.cuda.synchronize()
    assert bool(out.isnan().all())
    # the offsets are device data: a negative one makes its utterance NaN and reads nothing before wave
    neg = torch.tensor([-4000, 4000], dtype=torch.int64, device="cuda")
    assert call(o=L.ptr(neg))[0] == OK
    torch.cuda.synchronize()
    assert bool(out[0].isnan().all()) and bool(torch.isfinite(out[1]).all())
    assert call(o=L.ptr(offs + 1))[0] == OK                               # odd offsets are fine


# ----------------------------------------------------------------------------------------------- the installed loader

@pytest.fixture
def env(monkeypatch):
    from tests.test_loader_host import Env
    return Env(monkeypatch)


def _materialise(batches):
    return [tuple(t.clone() if t.is_cuda else t for t in b) for b in batches]


@needs_ref
@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("prob", [None, 0.5])
def test_installed_loader_matches_the_reference_loader(env, tmp_path, workers, prob):
    """The same batches as the unmodified loader on the same seeds: host tensors equal (values, dtypes), inputs on the
    current device within collate_waves' bar of the reference's (its stft is augment_oracle's float64 one)."""
    import b200asr
    DL = env.DL
    lengths = [4000, 4800, 3200, 32000, 1600, 2560, 5000, 3999, 4100, 16000, 161]
    ds = env.dataset(tmp_path, lengths, prob=prob, window="hann")
    _run = lambda: list(DL.AudioDataLoader(ds, num_workers=workers, batch_sampler=DL.BucketingSampler(ds, batch_size=4)))  # noqa: E731
    torch.manual_seed(3), np.random.seed(3), __import__("random").seed(3)
    want = _run()
    b200asr.install()
    try:
        torch.manual_seed(3), np.random.seed(3), __import__("random").seed(3)
        got = _materialise(_run())
    finally:
        b200asr.uninstall()
    assert len(got) == len(want) == 3
    for g, w in zip(got, want):
        assert g[0].is_cuda and g[0].dtype == torch.float32 and not any(t.is_cuda for t in g[1:])
        for a, b in zip(g[1:], w[1:]):
            assert a.dtype == b.dtype and torch.equal(a, b)
        assert g[0].shape == w[0].shape and rel_err(g[0].cpu(), w[0]) < BAR


@needs_ref
@pytest.mark.parametrize("workers", [0, 2])
def test_installed_loader_makes_no_host_sync(env, tmp_path, workers):
    import b200asr
    DL = env.DL
    ds = env.dataset(tmp_path, [16000, 8000, 12000, 4000] * 4, prob=0.5)
    b200asr.install()
    try:
        it = iter(DL.AudioDataLoader(ds, num_workers=workers, batch_size=4))
        next(it)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in range(3):
                next(it)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        b200asr.uninstall()


class _Replay:
    """An rng that gives NoiseClips.draw_one recorded draws back: one (add, clip, level, rand, start) row per utterance."""

    def __init__(self, rows):
        self.rows, self.k = list(rows), -1

    def binomial(self, n, p):
        self.k += 1
        return self.rows[self.k][0]

    def choice(self, n):
        return self.rows[self.k][1]

    def uniform(self, lo, hi):
        return self.rows[self.k][2]

    def rand(self):
        return self.rows[self.k][3]


class _Recorder:
    """Records every item the installed loader's workers make (num_workers=0: in this process) with its noise draws."""

    def __init__(self, monkeypatch):
        from b200asr import features, loader
        self.items, self.draws = [], []
        get, draw = loader.PackedItems.__getitem__, features.NoiseClips.draw_one

        def getitem(s, i):
            it = get(s, i)
            self.items.append(it)
            return it

        def draw_one(s, *a, **k):
            row = draw(s, *a, **k)
            self.draws.append(row)
            return row

        monkeypatch.setattr(loader.PackedItems, "__getitem__", getitem)
        monkeypatch.setattr(features.NoiseClips, "draw_one", draw_one)

    def collated(self, env, ds, sizes, window):
        """collate_waves over the recorded items, batch by batch, with the recorded draws."""
        import b200asr
        items, draws = list(self.items), list(self.draws)          # collate_waves' own draws are recorded too
        conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window=window, noise_dir="n", noise_prob=0.5,
                    noise_levels=(0.0, 0.5))
        bank = b200asr.NoiseBank([env.clips[p] for p in sorted(env.clips)], 16000)
        out, k = [], 0
        for n in sizes:
            batch = [(it.wave, it.ids) for it in items[k:k + n]]
            out.append(b200asr.collate_waves(batch, conf, env.ns.constant.args.src_max_len, bank, rng=_Replay(draws[k:k + n])))
            k += n
        assert k == len(items) == len(draws)
        return out


SMALL = ["--num-layers", "1", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
         "--dim-inner", "128", "--feat_extractor", "vgg_cnn", "--tgt-max-len", "16", "--dropout", "0.0", "--cuda", "--warmup", "4",
         "--k-lr", "0.02", "--min-lr", "1e-6", "--src-max-len", "90"]


def _model(env, extra=()):
    ns = ref_shim.load(SMALL + list(extra))
    i2l = {i: c for c, i in env.label2id.items()}
    torch.manual_seed(123456)
    return ns, ns.functions.init_transformer_model(ns.constant.args, env.label2id, i2l).cuda(), i2l


@needs_ref
def test_trainer_epoch_over_the_installed_loader(env, tmp_path, monkeypatch):
    """One epoch of the reference's Trainer.train over an installed loader (noise on, the cut binding) gives the losses
    and weights, bit for bit, of the bound loop fed the same items through collate_waves with the same noise draws."""
    import copy
    import b200asr
    ds = env.dataset(tmp_path, [16000, 8000, 12000, 4000, 9000, 15000, 3000, 11000], prob=0.5, src_max_len=90)
    valid = [b200asr.collate_waves([(w, [1, 4, 5, 2]) for w in _waves([7000, 5000], seed=3)],
                                   dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming"), 90)]
    rec = _Recorder(monkeypatch)
    results = []
    for arm in ("loader", "collate_waves"):
        ns, model, i2l = _model(env)
        ns.constant.args.src_max_len, ns.constant.args.save_folder, ns.constant.args.name = 90, str(tmp_path), arm
        opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
        losses = []
        b200asr.install()
        cur = ns.trainer.calculate_metrics
        ns.trainer.calculate_metrics = lambda *a, **k: (lambda out: (losses.append(float(out[0].item())), out)[1])(cur(*a, **k))
        try:
            if arm == "loader":
                np.random.seed(1), torch.manual_seed(1), __import__("random").seed(1)
                train = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))
            else:
                train = rec.collated(env, ds, [3, 3, 2], "hamming")
            ns.trainer.Trainer().train(model, train, None, [copy.deepcopy(valid)], opt, "ce", 0, 1, env.label2id, i2l)
        finally:
            ns.trainer.calculate_metrics = cur
            b200asr.uninstall()
        results.append((losses, {k: v.detach().clone() for k, v in model.state_dict().items()}))
    assert any(d[0] for d in rec.draws)                                    # some utterance took noise
    (la, wa), (lb, wb) = results
    assert len(la) == 4 and la == lb                                       # 3 training batches + 1 validation batch
    assert all(torch.equal(wa[k], wb[k]) for k in wa)


@needs_ref
def test_test_py_evaluate_over_the_installed_loader(env, tmp_path, monkeypatch, capsys):
    """test.py's evaluate(model, test_loader), loaded from its file, prints the same CER and WER over an installed loader
    as over the same items collated by collate_waves."""
    import b200asr
    ns, model, i2l = _model(env, ["--tgt-max-len", "300"])          # greedy decoding runs 300 positions
    path = os.path.join(ns.root, "test.py")
    if not os.path.exists(path):
        pytest.skip("the staged reference has no test.py")
    spec = importlib.util.spec_from_file_location("reference_test_script", path)
    script = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script)
    ds = env.dataset(tmp_path, [16000, 8000, 12000, 4000, 9000], prob=0.5, src_max_len=90, window="blackman")
    rec = _Recorder(monkeypatch)
    texts = []
    for arm in ("loader", "collate_waves"):
        ns.constant.args.src_max_len = 90
        b200asr.install()
        try:
            if arm == "loader":
                np.random.seed(2), torch.manual_seed(2), __import__("random").seed(2)
                test_loader = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=2))
            else:
                test_loader = rec.collated(env, ds, [2, 2, 1], "blackman")
            capsys.readouterr()
            script.evaluate(model, test_loader)
        finally:
            b200asr.uninstall()
        # the progress text without tqdm's rate and timing, which differ between runs
        texts.append(re.findall(r"TEST CER:[\d.]+% WER:[\d.]+% CER_EN:[\d.]+% CER_ZH:[\d.]+%", capsys.readouterr().err)[-1])
    assert texts[0] == texts[1], texts
