"""Greedy decoding and Transformer.evaluate on the device (csrc/decode.cu, modules.greedy_search / transformer_evaluate).

  * b200asr_decode_attn against float64: every (dk, dv) in {16, 32, 64, 128}^2; Tk in {1, 2, 31, 32, 33, 1000, 8192} and
    both sides of the first and last chunk boundaries; R in {1, 3, 32, 129} and H in {1, 8}; K/V read from a slab-major cache,
    a token-major projection and column slices of a wider buffer; large-magnitude scores.  Output and workspace are
    NaN-poisoned first; two calls give identical bits; rejected calls write and launch nothing.
  * Decoder.greedy_search on tests/golden/greedy.npz's model returns the strings of the reference's own ids (up to the first
    near-tie), "" for an utterance that emits EOS at step 0 and all 300 labels for one that never does.
  * The unmodified reference: Transformer.evaluate gives identical hypotheses and gold strings installed and uninstalled,
    greedy and beam, for feat_extractor '', vgg_cnn and emb_cnn (eval mode, non-trivial running statistics), including a batch
    that falls back to greedy; greedy_search with lm_rescoring=True or in training mode is the reference's own method; a
    positional table shorter than 300 positions raises before anything is launched.
  * An installed evaluate synchronises with the host at most ceil(300 / check_every) + 2 times.
"""
import math
import warnings

import pytest
import torch

import b200asr
import b200asr.modules as M
from oracle import asr_oracle as O
from oracle import ref_shim
from tests.gpu_util import cuda_model
from tests.helpers import load_greedy_golden

pytestmark = pytest.mark.gpu

L = b200asr._lib
DEV = "cuda"
U32 = 2.0 ** -24          # fp32 unit roundoff
HEAD_DIMS = (16, 32, 64, 128)


def _lib():
    return L.load()


# ------------------------------------------------------------------------------------------ decode_attn vs float64
def make_kv(layout, R, Tk, H, d, g, mag=1.0):
    """(tensor passed as the base pointer, (row stride, key stride), [R, Tk, H, d] view of the same values)."""
    if layout == "cache":               # [Tk][R][H*d]
        buf = torch.randn(Tk, R, H * d, generator=g, device=DEV) * mag
        return buf, (H * d, R * H * d), buf.view(Tk, R, H, d).permute(1, 0, 2, 3)
    if layout == "proj":                # [R][Tk][H*d]
        buf = torch.randn(R, Tk, H * d, generator=g, device=DEV) * mag
        return buf, (Tk * H * d, H * d), buf.view(R, Tk, H, d)
    w = H * d + 12                      # columns 8 .. 8 + H*d of a wider [R][Tk][w] buffer (a fused K|V projection, say)
    buf = torch.full((R, Tk, w), float("nan"), device=DEV)
    buf[:, :, 8:8 + H * d] = torch.randn(R, Tk, H * d, generator=g, device=DEV) * mag
    view = buf[:, :, 8:8 + H * d]
    return view, (Tk * w, w), view.reshape(R, Tk, H, d)


def run_decode_attn(q, k, ks, v, vs, R, H, dk, dv, Tk, scale):
    out = torch.full((R, H * dv), float("nan"), device=DEV)
    nws = _lib().b200asr_decode_attn_ws_bytes(R, H, Tk, dv) // 4
    ws = torch.full((max(nws, 1),), float("nan"), device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    L.check(_lib().b200asr_decode_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), ws.data_ptr() if nws else None,
                                       R, H, dk, dv, Tk, ks[0], ks[1], vs[0], vs[1], scale, st), "decode_attn")
    return out


def check_decode_attn(R, H, dk, dv, Tk, layout, seed, mag=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    scale = 1.0 / math.sqrt(dk)
    q = torch.randn(R, H * dk, generator=g, device=DEV) * mag
    k, ks, k4 = make_kv(layout, R, Tk, H, dk, g, mag)
    v, vs, v4 = make_kv(layout, R, Tk, H, dv, g)
    out = run_decode_attn(q, k, ks, v, vs, R, H, dk, dv, Tk, scale)
    q64, k64, v64 = q.double().view(R, H, dk), k4.double(), v4.double()
    s = torch.einsum("rhd,rjhd->rhj", q64, k64) * scale
    ref = torch.einsum("rhj,rjhd->rhd", torch.softmax(s, dim=-1), v64)
    # Bound: score error <= (dk + 1) u S with S = max_j sum_i |scale q_i k_ji|, so each weight e^(s - m) is off by a relative
    # 2 (dk + 2) u S (the max's error and expf included); the sums of at most Tk weights and weighted V rows add 2 (Tk + 8) u,
    # relative to max |v| (the output is a convex combination of V rows).  Twice that, per (row, head).
    S = torch.einsum("rhd,rjhd->rhj", q64.abs(), k64.abs()).amax(-1) * scale
    vmax = v64.abs().amax(dim=(1, 3))
    bound = 2 * U32 * vmax * (2 * (dk + 2) * S + 2 * (Tk + 8))
    err = (out.double().view(R, H, dv) - ref).abs().amax(-1)
    assert torch.isfinite(out).all(), (R, H, dk, dv, Tk, layout)
    assert (err <= bound).all(), (R, H, dk, dv, Tk, layout, float((err / bound).max()))
    return float((err / (vmax * U32)).max())


def chunk_boundaries(R, H, dv=16, top=8192):
    """Tk at which the number of key chunks changes (from the workspace query), first two and last two up to `top`."""
    n = [_lib().b200asr_decode_attn_ws_bytes(R, H, t, dv) // (R * H * (dv + 2) * 4) for t in range(1, top + 1)]
    n = [max(c, 1) for c in n]
    b = [t + 1 for t in range(1, top) if n[t] != n[t - 1]]
    return sorted(set(b[:2] + b[-2:]))


@pytest.mark.parametrize("dk", HEAD_DIMS)
@pytest.mark.parametrize("dv", HEAD_DIMS)
def test_decode_attn_matches_float64(dk, dv):
    R, H = 3, 8
    tks = {1, 2, 31, 32, 33, 1000, 8192}
    for b in chunk_boundaries(R, H):
        tks |= {b - 1, b, b + 1}
    worst = 0.0
    for i, Tk in enumerate(sorted(tks)):
        for layout in ("cache", "proj", "slice"):
            worst = max(worst, check_decode_attn(R, H, dk, dv, Tk, layout, seed=100 * i + dk + dv))
    print(f"decode_attn dk={dk} dv={dv}: max |err| = {worst:.1f} u max|v|")


@pytest.mark.parametrize("R", (1, 3, 32, 129))
@pytest.mark.parametrize("H", (1, 8))
def test_decode_attn_rows_and_heads(R, H):
    tks = {1, 33, 200, 1000}
    for b in chunk_boundaries(R, H, top=2100):
        tks |= {b - 1, b, b + 1}
    for i, Tk in enumerate(sorted(tks)):
        for dk, dv in ((64, 64), (16, 128), (128, 32)):
            for layout in ("cache", "proj", "slice"):
                check_decode_attn(R, H, dk, dv, Tk, layout, seed=7 * i + R + H)


def test_decode_attn_large_scores():
    """Scores of magnitude ~100s: exp without the max subtraction would overflow."""
    for Tk in (5, 200, 3000):
        for dk, dv in ((64, 64), (128, 16), (16, 128)):
            check_decode_attn(3, 8, dk, dv, Tk, "proj", seed=Tk + dk, mag=6.0)
            check_decode_attn(2, 2, dk, dv, Tk, "cache", seed=Tk + dv, mag=6.0)


def test_decode_attn_is_reproducible():
    g = torch.Generator(device=DEV).manual_seed(5)
    for R, H, Tk in ((32, 8, 200), (3, 8, 5000), (32, 8, 16)):
        q = torch.randn(R, H * 64, generator=g, device=DEV)
        k, ks, _ = make_kv("proj", R, Tk, H, 64, g)
        v, vs, _ = make_kv("proj", R, Tk, H, 64, g)
        a = run_decode_attn(q, k, ks, v, vs, R, H, 64, 64, Tk, 0.125)
        b = run_decode_attn(q, k, ks, v, vs, R, H, 64, 64, Tk, 0.125)
        assert torch.equal(a, b)


def test_decode_attn_rejections_write_and_launch_nothing():
    lib = _lib()
    R, H, d, Tk = 4, 2, 64, 300
    q = torch.randn(R, H * d, device=DEV)
    kv = torch.randn(R, Tk, H * d + 4, device=DEV)
    out = torch.full((R, H * d), float("nan"), device=DEV)
    ws = torch.full((lib.b200asr_decode_attn_ws_bytes(R, H, Tk, d) // 4,), float("nan"), device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    ok = dict(k=kv.data_ptr(), ws=ws.data_ptr(), dk=d, Tk=Tk, krs=Tk * (H * d + 4), kks=H * d + 4)
    bad = [dict(ws=None), dict(dk=48), dict(Tk=0), dict(Tk=70000), dict(k=kv.data_ptr() + 4), dict(kks=H * d + 2),
           dict(krs=-4)]
    torch.cuda.synchronize()
    n0 = lib.b200asr_launch_count()
    for change in bad:
        a = dict(ok, **change)
        rc = lib.b200asr_decode_attn(q.data_ptr(), a["k"], kv.data_ptr(), out.data_ptr(), a["ws"], R, H, a["dk"], d, a["Tk"],
                                     a["krs"], a["kks"], Tk * (H * d + 4), H * d + 4, 0.125, st)
        assert rc in (-1, -2, -5), change
    torch.cuda.synchronize()
    assert lib.b200asr_launch_count() == n0
    assert out.isnan().all() and ws.isnan().all()
    a = ok
    assert lib.b200asr_decode_attn(q.data_ptr(), a["k"], kv.data_ptr(), out.data_ptr(), a["ws"], R, H, d, d, Tk, a["krs"],
                                   a["kks"], a["krs"], a["kks"], 0.125, st) == 0
    assert torch.isfinite(out).all() and lib.b200asr_launch_count() == n0 + 2      # split keys: partials + merge


# ------------------------------------------------------------------------------------------ greedy strings vs the reference
def golden_labels(V):
    """ref_shim.labels without the reference: PAD/SOS/EOS characters, then one CJK character per id."""
    return {i: c for i, c in enumerate([M.PAD_CHAR, M.SOS_CHAR, M.EOS_CHAR] + [chr(0x4E00 + i) for i in range(V - 3)])}


@pytest.fixture(scope="module")
def greedy_golden():
    cfg, P, enc, ref_ids, ref_len = load_greedy_golden()
    full = dict(O.init_params(cfg, seed=1))              # encoder / front-end entries are unused by the decode
    full.update(P)
    return cfg, full, enc, ref_ids, ref_len


def _decoder(cfg, P):
    dec = cuda_model(cfg, P, train=False).decoder
    dec.id2label = golden_labels(cfg.vocab)
    return dec


def test_greedy_search_returns_the_reference_strings(greedy_golden):
    cfg, P, enc, ref_ids, ref_len = greedy_golden
    _, margins = O.greedy_decode(P, cfg, enc, steps=300)
    dec = _decoder(cfg, P)
    strs = dec.greedy_search(enc.cuda())
    band = 1e-4 * float(margins.abs().max())             # the band of the greedy fixture test (test_gpu_parity.py)
    lab = dec.id2label
    for b in range(enc.shape[0]):
        n = int(ref_len[b])
        want = "".join(lab[int(i)] for i in ref_ids[b, :n])
        safe = int((margins[b] > band).long().cumprod(0).sum())
        m = min(n, safe)
        assert m >= 32, "fixture degenerate: near-tie too early"
        assert strs[b][:m] == want[:m], b                 # one character per label
        if safe >= n:
            assert strs[b] == want, b


def test_greedy_search_without_any_eos_gives_300_labels(greedy_golden):
    cfg, P, enc, _, _ = greedy_golden
    P = dict(P)
    P["decoder.output_linear.weight"] = P["decoder.output_linear.weight"].clone()
    P["decoder.output_linear.weight"][2] = 0.0          # the EOS logit is 0; with logits spread, another one always wins
    ids_o, margins = O.greedy_decode(P, cfg, enc, steps=300)
    dec = _decoder(cfg, P)
    ids = dec.greedy_decode_cached(enc.cuda(), steps=300).cpu()
    assert not (ids == 2).any(), "test input degenerate: EOS emitted"
    strs = dec.greedy_search(enc.cuda())
    band = 1e-4 * float(margins.abs().max())
    for b in range(enc.shape[0]):
        assert len(strs[b]) == 300 and strs[b] == "".join(dec.id2label[int(i)] for i in ids[b]), b
        safe = int((margins[b] > band).long().cumprod(0).sum())
        assert strs[b][:safe] == "".join(dec.id2label[int(i)] for i in ids_o[b, :safe]), b


def test_greedy_search_with_eos_at_step_zero_gives_empty_strings(greedy_golden):
    cfg, P, enc, _, _ = greedy_golden
    P = dict(P)
    last = f"decoder.layers.{cfg.num_layers - 1}.pos_ffn.layer_norm"
    g = torch.Generator().manual_seed(4)
    beta = torch.randn(cfg.dim_model, generator=g)
    P[last + ".weight"] = torch.zeros(cfg.dim_model)    # every decoder output is beta ...
    P[last + ".bias"] = beta
    P["decoder.output_linear.weight"] = P["decoder.output_linear.weight"].clone()
    P["decoder.output_linear.weight"][2] = 10.0 * beta  # ... and EOS its best match
    dec = _decoder(cfg, P)
    assert dec.greedy_search(enc.cuda()) == [""] * enc.shape[0]
    assert (dec.greedy_decode_cached(enc.cuda(), steps=8).cpu() == 2).all()
    ids = dec.greedy_decode_cached(enc.cuda(), steps=300, stop_at_eos=True, check_every=8).cpu()
    assert (ids == -1).all()                            # -1 from the first EOS on, that EOS included


# ------------------------------------------------------------------------------------------ the unmodified reference
FLAGS = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
         "--dim-inner", "128", "--tgt-max-len", "301", "--dropout", "0.0", "--cuda"]
FRAMES = {"": (24, 310), "vgg_cnn": (96, None), "emb_cnn": (48, None)}      # (short batch, batch ending no beam hypothesis)


def _reference_model(feat, V=40, eos_scale=2.2):
    ns = ref_shim.load(FLAGS + ["--feat_extractor", feat], q12_shim=True)
    l2i, i2l = ref_shim.labels(V)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.decoder.output_linear.weight.mul_(4.0)                 # spread the logits
        model.decoder.output_linear.weight[2].mul_(eos_scale)        # utterances end at different steps
        if feat == "emb_cnn":
            for bn in (model.conv[1], model.conv[4]):
                bn.running_mean.copy_(0.2 * torch.randn(bn.running_mean.shape, generator=g))
                bn.running_var.copy_(0.5 + torch.rand(bn.running_var.shape, generator=g))
                bn.num_batches_tracked.fill_(10)
    return ns, model.cuda().eval(), g


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
@pytest.mark.parametrize("feat", ["", "vgg_cnn", "emb_cnn"])
def test_reference_evaluate_installed_matches_uninstalled(feat):
    ns, model, g = _reference_model(feat, eos_scale=1.0 if feat == "emb_cnn" else 2.2)     # emb_cnn: EOS would win at once
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    V = 40
    eos_row = model.decoder.output_linear.weight[2].detach().clone()
    short, long_ = FRAMES[feat]
    batches = [(short, 1.0)] + ([(long_, 0.0)] if long_ else [])
    data = []
    for T, s in batches:
        src = torch.randn(2, 1, 161, T, generator=g).cuda()
        lens = torch.full((2,), T, dtype=torch.int32).cuda()
        tgt = torch.randint(3, V, (2, 6), generator=g).cuda()
        data.append((src, lens, tgt, s))
    results = {}
    try:
        for installed in (False, True):
            if installed:
                b200asr.install()
            out = []
            for src, lens, tgt, s in data:
                with torch.no_grad():
                    model.decoder.output_linear.weight[2] = eos_row * s
                    for beam in (False, True):
                        rest, hyps, gold = model.evaluate(src, lens, tgt, beam_search=beam, beam_width=4, beam_nbest=1,
                                                          c_weight=0.1)
                        out.append((beam, list(hyps), list(gold)))
                        if installed:
                            assert rest == [[None, None], [None, None]]
            results[installed] = out
    finally:
        b200asr.uninstall()
        with torch.no_grad():
            model.decoder.output_linear.weight[2] = eos_row
    assert results[True] == results[False], (results[True], results[False])
    for _, hyps, gold in results[True]:
        assert len(hyps) == 2 and all(len(x) == 301 for x in gold)
    print(feat, [[len(h) for h in r[1]] for r in results[True]])


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_greedy_search_special_cases(monkeypatch):
    ns, model, g = _reference_model("")
    dec = model.decoder
    enc = torch.randn(2, 24, 64, generator=g).cuda()
    with torch.no_grad():
        try:                                             # lm_rescoring=True: the reference's method fails by itself
            dec.greedy_search(enc, lm_rescoring=True)
            ref_err = None
        except Exception as e:                           # noqa: BLE001 - whatever the reference raises
            ref_err = (type(e), str(e))
        dec.train()
        ref_train = dec.greedy_search(enc)
        dec.eval()
        try:
            b200asr.install()
            monkeypatch.setattr(M, "greedy_decode_cached", None)        # the device path must not be taken
            try:
                dec.greedy_search(enc, lm_rescoring=True)
                got_err = None
            except Exception as e:                       # noqa: BLE001
                got_err = (type(e), str(e))
            dec.train()
            got_train = dec.greedy_search(enc)
            dec.eval()
            monkeypatch.undo()
            dec.trg_max_length = 299
            torch.cuda.synchronize()
            n0 = _lib().b200asr_launch_count()
            with pytest.raises(ValueError, match="trg_max_length"):
                dec.greedy_search(enc)
            assert _lib().b200asr_launch_count() == n0
        finally:
            dec.trg_max_length = 301
            b200asr.uninstall()
    assert ref_err is not None and got_err == ref_err
    assert got_train == ref_train


# ------------------------------------------------------------------------------------------ host synchronisations
def test_installed_evaluate_syncs_a_bounded_number_of_times():
    cfg = b200asr.ASRConfig(num_layers=2, num_heads=2, dim_model=64, dim_key=32, dim_value=32, dim_inner=128, vocab=40,
                            feat_extractor="", tgt_max_len=301, dropout=0.0)
    torch.manual_seed(0)
    model = b200asr.build_model(cfg, id2label=golden_labels(40)).cuda().eval()        # one character per label
    with torch.no_grad():
        model.decoder.output_linear.weight[2] = 0.0       # no utterance ends: all 300 steps run
    g = torch.Generator().manual_seed(1)
    src = torch.randn(4, 1, 161, 30, generator=g).cuda()
    lens = torch.full((4,), 30, dtype=torch.int32).cuda()
    tgt = torch.randint(3, 40, (4, 6), generator=g).cuda()
    model.evaluate(src, lens, tgt)                         # warm-up: weight splits, workspaces
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            _, hyps, gold = model.evaluate(src, lens, tgt)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    limit = math.ceil(300 / 8) + 2
    print(f"installed evaluate: {len(syncs)} host syncs (limit {limit}); uninstalled it is about B * (300 + tgt_max_len)")
    assert 0 < len(syncs) <= limit, [str(w.message)[:120] for w in syncs]
    assert len(hyps) == 4 and all(len(h) == 300 for h in hyps) and all(len(s) == 301 for s in gold)
