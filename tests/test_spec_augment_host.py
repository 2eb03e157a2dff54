"""CPU checks of SpecAugment (features.SpecAugment, b200asr_spec_augment): the host restatement of its counter-based
draws (tests/spec_augment_util.py) and their ranges, the warp's map, the policy's argument validation and pickling, and
the C entry point's rejections, which need no GPU, and the kernel's build (no spills, no local memory)."""
import pickle

import numpy as np
import pytest
import torch

import b200asr
from tests import spec_augment_util as SA

L = b200asr._lib


@pytest.fixture(scope="module")
def lib():
    import os
    import __graft_entry__
    if not os.path.exists(L.LIB_PATH):
        __graft_entry__.build()
    return L.load()


def test_splitmix64_is_the_published_generator():
    """SplitMix64 (Steele, Lea and Flood 2014; Vigna's reference code) from state 1234567: its first two outputs."""
    assert SA.splitmix64(1234567) == 6457827717110365317
    assert SA.splitmix64((1234567 + SA.GOLDEN) & SA.M64) == 3203168211198807973


def _all_draws(sizes, F, T, W, Fp, nf, Tp, p, nt, counters=range(200), seed=7):
    return np.stack([SA.draws(sizes, F, T, W, Fp, nf, Tp, p, nt, seed, k) for k in counters])


def test_draw_ranges_and_coverage():
    """Over 600 counters: every draw within its range and every value of a small range met."""
    W, Fp, Tp, p, nf, nt, F, T = 3, 5, 6, 0.5, 2, 2, 11, 40
    sizes = [40, 9, 8, 7, 1, 0, 12]                     # 9 = 2W + 3, 8 = 2W + 2 (warps), 7 = 2W + 1 (does not)
    D = _all_draws(sizes, F, T, W, Fp, nf, Tp, p, nt, counters=range(600))
    for b, Tb in enumerate(sizes):
        c, w = D[:, b, 0], D[:, b, 1]
        if Tb > 2 * W + 1:
            assert set(c) == set(range(W, Tb - W)) and set(w) == set(range(-W, W + 1)), b
        else:
            assert not c.any() and not w.any(), b
        for m in range(nf):
            f, f0 = D[:, b, 2 + 2 * m], D[:, b, 3 + 2 * m]
            assert set(f) == set(range(Fp + 1)) and (f0 >= 0).all() and (f0 <= F - f).all()
            assert set(f0[f == 0]) == set(range(F + 1))
        cap = min(Tp, int(np.floor(p * Tb)))
        for m in range(nt):
            t, t0 = D[:, b, 2 + 2 * nf + 2 * m], D[:, b, 3 + 2 * nf + 2 * m]
            assert set(t) == set(range(cap + 1)) and (t0 >= 0).all() and (t0 <= Tb - t).all(), b
    # slots are independent: the two masks of a kind are not the same draw
    assert (D[:, :, 2] != D[:, :, 4]).any() and (D[:, :, 6] != D[:, :, 8]).any()


def test_draw_edge_policies():
    """p = 0 and Tp = 0 give empty time masks (t0 still drawn in [0, T_b]); Fp = 0 empty frequency masks; T_b = 1 and
    T_b <= 2W + 1 no warp; W = 0 draws c but w = 0."""
    D = _all_draws([1, 5, 30], 9, 30, 2, 0, 1, 10, 0.0, 1)
    assert not D[:, :, 0:2][:, :2].any() and not D[:, :, 2].any() and not D[:, :, 4].any()
    assert set(D[:, 2, 5]) == set(range(31)) and set(D[:, 0, 5]) == {0, 1}
    D = _all_draws([1, 30], 9, 30, 0, 9, 0, 0, 1.0, 1)
    assert not D[:, 0, :2].any() and set(D[:, 1, 0]) == set(range(30)) and not D[:, 1, 1].any()
    assert not D[:, :, 2].any()
    D = _all_draws([1], 9, 30, 0, 9, 0, 5, 1.0, 1)                 # T_b = 1, p = 1: t in [0, 1]
    assert set(D[:, 0, 2]) == {0, 1} and set(D[:, 0, 3][D[:, 0, 2] == 1]) == {0}
    # the cap is floor(float32(p) * T_b) in double: float32(0.3) * 10 = 3.0000001...
    assert max(SA.draws([10], 3, 10, 0, 0, 0, 99, 0.3, 1, 1, k)[0, 2] for k in range(300)) == 3


def test_draws_depend_on_seed_counter_and_utterance():
    a = SA.draws([50] * 4, 161, 50, 5, 27, 2, 20, 1.0, 2, 1, 0)
    assert not np.array_equal(a, SA.draws([50] * 4, 161, 50, 5, 27, 2, 20, 1.0, 2, 1, 1))
    assert not np.array_equal(a, SA.draws([50] * 4, 161, 50, 5, 27, 2, 20, 1.0, 2, 2, 0))
    assert len({tuple(r) for r in a}) == 4


def test_warp_map():
    """s(0) = 0, s(c + w) = c, s(T_b - 1) = T_b - 1, increasing, and the identity without a shift; the degenerate ends."""
    for Tb, c, w in [(20, 8, 3), (20, 8, -3), (8, 3, -3), (8, 4, 3), (8, 4, 0), (2000, 80, 80)]:
        s = [SA.source_position(t, Tb, c, w) for t in range(Tb)]
        assert s[0] == 0 and s[-1] == Tb - 1 and (s[c + w] == c or c + w in (0, Tb - 1))
        assert all(x < y for x, y in zip(s, s[1:])), (Tb, c, w)
        if c + w == 0:                                   # frame 1 starts the second piece, just past c
            assert s[1] == c + (Tb - 1 - c) / (Tb - 1)
        if c + w == Tb - 1:
            assert s[Tb - 2] == (Tb - 2) * c / (Tb - 1)
        if w == 0:
            assert s == list(range(Tb))
    x = np.arange(2 * 3 * 9, dtype=np.float64).reshape(2, 1, 3, 9)
    out, zero, bound = SA.reference(x, np.array([[0, 0], [4, 0]], np.int32), [9, 6], 0, 0)
    assert np.array_equal(out[0], x[0]) and np.array_equal(out[1, ..., :6], x[1, ..., :6]) and zero[1, ..., 6:].all()
    assert not bound.any()


@pytest.mark.parametrize("kw", [dict(W=-1), dict(Fp=-1), dict(Tp=-2), dict(n_freq_masks=-1), dict(n_time_masks=65),
                                dict(n_freq_masks=65), dict(p=-0.1), dict(p=1.5), dict(p=float("nan")), dict(W=2.0),
                                dict(Fp=True), dict(p="0.5"), dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.5),
                                dict(W=2 ** 31)])
def test_policy_rejects_bad_arguments(kw):
    args = dict(W=5, Fp=27, n_freq_masks=2, Tp=40, p=1.0, n_time_masks=2, seed=1)
    args.update(kw)
    with pytest.raises(ValueError):
        b200asr.SpecAugment(**args)


def test_policy_has_no_defaults_and_pickles():
    with pytest.raises(TypeError):
        b200asr.SpecAugment(80, 27, 1, 100, 1.0, 1)                      # no default seed
    a = b200asr.SpecAugment(80, 27, 2, 100, 1.0, 2, seed=2 ** 64 - 1)
    a.counter = 17
    b = pickle.loads(pickle.dumps(a))
    assert vars(b) == vars(a) and b.counter == 17 and b.draws_per_utterance == 10
    assert "W=80" in repr(b)


def test_apply_needs_cuda_tensors():
    a = b200asr.SpecAugment(2, 3, 1, 4, 1.0, 1, seed=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        a.apply(torch.zeros(1, 1, 5, 8), torch.tensor([8], dtype=torch.int32))
    assert a.counter == 0


def test_draws_ints(lib):
    assert lib.b200asr_spec_augment_draws_ints(0, 0) == 2
    assert lib.b200asr_spec_augment_draws_ints(1, 2) == 8
    assert lib.b200asr_spec_augment_draws_ints(64, 64) == 258
    assert lib.b200asr_spec_augment_draws_ints(65, 0) == lib.b200asr_spec_augment_draws_ints(0, -1) == 0


def test_entry_point_rejections_need_no_device(lib):
    """Argument checks run on the host before any launch: pointers that are never dereferenced."""
    base = dict(i=1 << 20, o=1 << 24, d=1 << 28, f=1 << 29, B=2, F=7, T=9, W=1, Fp=3, nf=1, Tp=4, p=1.0, nt=1)

    def call(**kw):
        a = dict(base, **kw)
        return lib.b200asr_spec_augment(a["i"], a["o"], a["d"], a["f"], a["B"], a["F"], a["T"], a["W"], a["Fp"], a["nf"],
                                        a["Tp"], a["p"], a["nt"], 1, 0, None)
    BAD_SHAPE, BAD_ALIGN, BAD_ARG = -1, -2, -5
    for k in ("i", "o", "d", "f"):
        assert call(**{k: None}) == BAD_ARG, k
        assert call(**{k: base[k] + 2}) == BAD_ALIGN, k
    for k in ("B", "F", "T"):
        assert call(**{k: 0}) == BAD_SHAPE, k
    assert call(B=65536) == BAD_SHAPE and call(F=1 << 16, T=1 << 15) == BAD_SHAPE and call(F=1 << 21, T=1, Fp=0) == BAD_SHAPE
    assert call(W=-1) == BAD_ARG and call(Fp=-1) == BAD_ARG and call(Fp=8) == BAD_ARG and call(Tp=-1) == BAD_ARG
    assert call(p=-0.5) == BAD_ARG and call(p=1.01) == BAD_ARG and call(p=float("nan")) == BAD_ARG
    assert call(nf=-1) == BAD_ARG and call(nt=65) == BAD_ARG
    assert call(o=base["i"]) == BAD_ARG and call(o=base["i"] + 4 * 2 * 7 * 9 - 4) == BAD_ARG
    assert "spec_augment" in L.last_error()


def test_kernel_compiles_without_spills_or_local_memory(tmp_path):
    """spec_augment.cu recompiled with build.sh's flags and -Xptxas -v: no stack frame and no spill stores; and in the
    built library, STACK:0 LOCAL:0 (cuobjdump -res-usage)."""
    import os
    import re
    import subprocess
    from tests.test_engine_build import CSRC, CUOBJDUMP, LIB, NVCC, ROOT, _build_flags, _need
    _need(NVCC)
    log = subprocess.run([NVCC, *_build_flags(), "-Xptxas", "-v,-warn-spills", "-c", os.path.join(CSRC, "spec_augment.cu"),
                          "-o", str(tmp_path / "spec_augment.o")], capture_output=True, text=True, cwd=ROOT, check=True).stderr
    props = re.findall(r"Function properties for (\S*spec_augment_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores",
                       log)
    assert len(props) == 1 and props[0][1:] == ("0", "0"), log[-2000:]
    _need(CUOBJDUMP, LIB)
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = [u for n, u in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out) if "spec_augment_kernel" in n]
    assert len(usage) == 1 and re.search(r"\bSTACK:0\b", usage[0]) and re.search(r"\bLOCAL:0\b", usage[0]), usage


@pytest.mark.skipif(not __import__("oracle.ref_shim", fromlist=["available"]).available(),
                    reason="reference checkout not staged (oracle/make_ref.py)")
def test_loader_on_the_reference_iterator_refuses_a_policy(monkeypatch, tmp_path):
    """An installed AudioDataLoader that runs the reference's own iterator (here: a caller's collate_fn) raises for a
    dataset carrying spec_augment instead of yielding unaugmented batches; it runs as before without the attribute."""
    from tests.test_loader_host import Env
    env = Env(monkeypatch)
    ds = env.dataset(tmp_path, [4000, 3000], prob=None)
    ds.spec_augment = b200asr.SpecAugment(2, 3, 1, 4, 1.0, 1, seed=0)
    b200asr.install()
    try:
        loader = env.DL.AudioDataLoader(ds, batch_size=2, collate_fn=lambda items: items)
        with pytest.raises(RuntimeError, match="spec_augment"):
            iter(loader)
        del ds.spec_augment
        assert len(next(iter(loader))) == 5                       # the reference's own _collate_fn 5-tuple
    finally:
        b200asr.uninstall()
