"""Training the LSTM language model on the device: RNNModel("LSTM").forward and its backward through time (csrc/lstm.cu:
LstmCellPolicyT<true>, LstmCellBwdPolicy, lstm_dropout, lstm_grad_unprepare; ops.LstmStackFn; modules.rnn_model_forward).

  * The stack (embedding, nn.LSTM, h_n / c_n) and every gradient against float64 nn.LSTM with CPU autograd over nhid
    {8, 13, 650}, 1-3 layers, T {1, 2, 35, 200}, B {1, 20, 129}, no / zero / random initial state, with and without
    gradients on h_n / c_n.
  * RNNModel end to end through nn.CrossEntropyLoss against float64, untied and tied.
  * Dropout masks equal a host restatement of the counter-based generator; eval mode applies none; backward regenerates
    them; successive calls draw new ones.  Two calls give identical bits.
  * Eval-mode NLL equals the rescoring path (ops.lstm_lm_nll_sums).
  * The reference's word-language-model loop and LM.evaluate installed vs on cuDNN.
  * Rejections, the GRU fallback and no host synchronisation.
Outputs and workspaces come from an allocator whose cached blocks were filled with NaN first.  Errors are max-norm,
relative to the largest reference entry; bars state the error measured on one H100 80GB HBM3 (700 W power limit).
"""
import importlib
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import b200asr
from oracle import ref_shim
from tests.test_gpu_flash_attention import _dropout_key, _splitmix64

pytestmark = pytest.mark.gpu

M = importlib.import_module(b200asr.__name__ + ".modules")      # the package's own modules (its rng is the one forward uses)
ops = importlib.import_module(b200asr.__name__ + ".ops")

L = b200asr._lib
DEV = "cuda"
H_TOL = 2e-5        # layer outputs, h_n, c_n, logits (as the forward test of test_gpu_engine_schedule.py; measured 8.9e-6 max)
GRAD_TOL = 1e-4     # every gradient (measured 1.8e-5 max)


def _poison():
    """Fill the caching allocator's free blocks with NaN, so that buffers the path forgets to write show up as NaN."""
    big = torch.full((96 << 20,), float("nan"), device=DEV)
    small = [torch.full((1 << 16,), float("nan"), device=DEV) for _ in range(64)]
    del big, small


def _err(got, ref):
    ref = ref.detach().double().cpu()
    return float((got.detach().double().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _model(ntoken, ninp, nhid, nlayers, tie=False, seed=0, dropout=0.0):
    torch.manual_seed(seed)
    m = M.RNNModel("LSTM", ntoken, ninp, nhid, nlayers, dropout=dropout, tie_weights=tie)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(1.0 / math.sqrt(nhid) * torch.randn(p.shape))
    return m.to(DEV)


def _thresh16(p):
    return int(min(max(p * 65536.0 + 0.5, 0.0), 65535.0))


def _mask(rows, cols, width, p, seed, offset):
    """common.cuh dropout_keep at element index row * width + col (the padded layout) as the float64 factor
    keep / (1 - p16) of the fp32 kernels, [rows, cols]."""
    with np.errstate(over="ignore"):
        idx = np.arange(rows * width, dtype=np.uint64)
        r = _splitmix64(np.uint64(_dropout_key(seed, offset)) + (idx >> np.uint64(2)) * np.uint64(0x9E3779B97F4A7C15))
        bits = (r >> (np.uint64(16) * (idx & np.uint64(3)))) & np.uint64(0xFFFF)
    t = _thresh16(p)
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(t) / np.float32(65536.0)))
    keep = (bits >= np.uint64(t)).reshape(rows, width)[:, :cols]
    return torch.from_numpy(keep.astype(np.float64) * inv)


def _ref_stack(model, inp, hidden, masks=None):
    """float64 CPU restatement: embedding, per-layer nn.LSTM, masks (emb, layer outputs) multiplied in.  Returns the leaf
    tensors and (out, h_n, c_n)."""
    rnn = model.rnn
    nl, nhid = rnn.num_layers, rnn.hidden_size
    emb = model.encoder.weight.detach().double().cpu().requires_grad_(True)
    T, B = inp.shape
    x = emb[inp.cpu()]
    if masks is not None:
        x = x * masks[0].view(T, B, -1)
    layers = []
    for l in range(nl):
        lstm = nn.LSTM(x.shape[-1] if l == 0 else nhid, nhid, 1).double()
        with torch.no_grad():
            for nm in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                getattr(lstm, nm + "_l0").copy_(getattr(rnn, f"{nm}_l{l}").detach().double().cpu())
        layers.append(lstm)
    h0 = c0 = None
    if hidden is not None:
        h0 = hidden[0].detach().double().cpu().requires_grad_(True)
        c0 = hidden[1].detach().double().cpu().requires_grad_(True)
    hn, cn = [], []
    for l, lstm in enumerate(layers):
        st = None if h0 is None else (h0[l:l + 1], c0[l:l + 1])
        x, (h, c) = lstm(x, st)
        hn.append(h[0])
        cn.append(c[0])
        if masks is not None:
            x = x * masks[1 + l].view(T, B, -1)
    return dict(emb=emb, layers=layers, h0=h0, c0=c0), (x, torch.stack(hn), torch.stack(cn))


def _compare_grads(model, leaves, hidden, errs):
    rnn = model.rnn
    errs["d_emb"] = _err(model.encoder.weight.grad, leaves["emb"].grad)
    for l, lstm in enumerate(leaves["layers"]):
        for nm in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            errs[f"d_{nm}_l{l}"] = _err(getattr(rnn, f"{nm}_l{l}").grad, getattr(lstm, nm + "_l0").grad)
    if hidden is not None:
        errs["dh0"] = _err(hidden[0].grad, leaves["h0"].grad)
        errs["dc0"] = _err(hidden[1].grad, leaves["c0"].grad)


# (nhid, ninp, nlayers, T, B, initial state, gradients on h_n / c_n)
STACK_CASES = [
    (8, 12, 1, 1, 1, "none", False), (8, 12, 2, 2, 20, "rand", True), (8, 12, 3, 35, 129, "rand", True),
    (8, 12, 1, 200, 20, "zero", True), (13, 20, 1, 2, 1, "rand", False), (13, 20, 2, 35, 20, "none", True),
    (13, 20, 3, 200, 129, "rand", True), (13, 20, 1, 1, 129, "zero", True), (650, 400, 1, 35, 20, "rand", True),
    (650, 400, 2, 2, 129, "none", False), (650, 400, 3, 1, 1, "rand", True), (650, 400, 1, 200, 20, "zero", False),
]


@pytest.mark.parametrize("nhid,ninp,nl,T,B,state,out_grads", STACK_CASES)
def test_stack_matches_float64(nhid, ninp, nl, T, B, state, out_grads):
    g = torch.Generator().manual_seed(nhid * 7 + T * 3 + B)
    model = _model(T * B, ninp, nhid, nl, seed=T + B)
    inp = torch.randperm(T * B, generator=g).view(T, B)           # every token once: the embedding gradient is dx
    hidden = None
    if state != "none":
        scale = 0.0 if state == "zero" else 0.5
        hidden = tuple((scale * torch.randn(nl, B, nhid, generator=g)).to(DEV).requires_grad_(True) for _ in range(2))
    R = torch.randn(T, B, nhid, generator=g, dtype=torch.float64)
    Rh, Rc = torch.randn(nl, B, nhid, generator=g, dtype=torch.float64), torch.randn(nl, B, nhid, generator=g, dtype=torch.float64)
    _poison()
    out, (hn, cn) = ops.lstm_stack(model, inp.to(DEV), hidden)
    loss = (out * R.float().to(DEV)).sum()
    if out_grads:
        loss = loss + (hn * Rh.float().to(DEV)).sum() + (cn * Rc.float().to(DEV)).sum()
    loss.backward()
    leaves, (o64, h64, c64) = _ref_stack(model, inp, hidden)
    l64 = (o64 * R).sum() + ((h64 * Rh).sum() + (c64 * Rc).sum() if out_grads else 0.0)
    l64.backward()
    errs = dict(out=_err(out, o64), h_n=_err(hn, h64), c_n=_err(cn, c64))
    _compare_grads(model, leaves, hidden, errs)
    print(f"stack nhid={nhid} L={nl} T={T} B={B} {state} out_grads={out_grads}: " +
          " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < (H_TOL if k in ("out", "h_n", "c_n") else GRAD_TOL), (k, v)


def test_grad_unprepare_inverts_prepare():
    """b200asr_lstm_prepare then b200asr_lstm_grad_unprepare is the identity on W_ih and W_hh; the bias comes back as
    b_ih + b_hh in both outputs."""
    lib = L.load()
    ninp, nhid = 13, 21
    I, H = 16, 24
    g = torch.Generator().manual_seed(0)
    w_ih, w_hh = torch.randn(4 * nhid, ninp, generator=g).to(DEV), torch.randn(4 * nhid, nhid, generator=g).to(DEV)
    b_ih, b_hh = torch.randn(4 * nhid, generator=g).to(DEV), torch.randn(4 * nhid, generator=g).to(DEV)
    wp, hp, bp = torch.empty(4 * H, I, device=DEV), torch.empty(4 * H, H, device=DEV), torch.empty(4 * H, device=DEV)
    P = L.ptr
    assert lib.b200asr_lstm_prepare(P(w_ih), P(w_hh), P(b_ih), P(b_hh), ninp, nhid, P(wp), P(hp), P(bp), None) == 0
    outs = [torch.full(s, float("nan"), device=DEV) for s in ((4 * nhid, ninp), (4 * nhid, nhid), (4 * nhid,), (4 * nhid,))]
    assert lib.b200asr_lstm_grad_unprepare(P(wp), P(hp), P(bp), ninp, nhid, *[P(t) for t in outs], None) == 0
    assert torch.equal(outs[0], w_ih) and torch.equal(outs[1], w_hh)
    want = (b_ih + b_hh).view(4, nhid)
    assert torch.equal(outs[2].view(4, nhid), want) and torch.equal(outs[3].view(4, nhid), want)
    assert lib.b200asr_lstm_grad_unprepare(None, P(hp), P(bp), ninp, nhid, P(outs[0]), None, None, None, None) == -5
    assert L.last_error().startswith("lstm_grad_unprepare:")


# ------------------------------------------------------------------------------------------ RNNModel end to end
@pytest.mark.parametrize("tie", [False, True])
def test_rnn_model_end_to_end_matches_float64(tie):
    ntoken, nhid, nl, T, B = 300, 48, 2, 35, 20
    ninp = nhid if tie else 40
    model = _model(ntoken, ninp, nhid, nl, tie=tie, seed=3)
    model.train()
    g = torch.Generator().manual_seed(1)
    inp = torch.randint(0, ntoken, (T, B), generator=g)
    tgt = torch.randint(0, ntoken, (T * B,), generator=g)
    hidden = tuple((0.3 * torch.randn(nl, B, nhid, generator=g)).to(DEV) for _ in range(2))
    _poison()
    decoded, (hn, cn) = model(inp.to(DEV), hidden)
    assert decoded.shape == (T, B, ntoken) and hn.shape == (nl, B, nhid)
    loss = nn.CrossEntropyLoss()(decoded.view(-1, ntoken), tgt.to(DEV))
    loss.backward()
    leaves, (o64, _, _) = _ref_stack(model, inp, hidden)
    # tied: the decoder weight is the embedding leaf itself, so its gradient is the sum of both uses
    w = leaves["emb"] if tie else model.decoder.weight.detach().double().cpu().requires_grad_(True)
    b = model.decoder.bias.detach().double().cpu().requires_grad_(True)
    logits = o64 @ w.t() + b
    l64 = nn.CrossEntropyLoss()(logits.view(-1, ntoken), tgt)
    l64.backward()
    errs = dict(logits=_err(decoded, logits), loss=abs(float(loss) - float(l64)) / abs(float(l64)))
    _compare_grads(model, leaves, None, errs)
    errs["d_dec_b"] = _err(model.decoder.bias.grad, b.grad)
    if not tie:
        errs["d_dec_w"] = _err(model.decoder.weight.grad, w.grad)
    print(f"RNNModel tie={tie}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < (H_TOL if k in ("logits", "loss") else GRAD_TOL), (k, v)


# ------------------------------------------------------------------------------------------ dropout
def _dropout_case(seed, offset0, model, inp, hidden, p):
    """float64 reference of a train-mode call whose masks are at offsets offset0 + 1 (embedding), + 2, + 3 (layer outputs)."""
    T, B = inp.shape
    I, H = (model.encoder.weight.shape[1] + 7) // 8 * 8, (model.rnn.hidden_size + 7) // 8 * 8
    ninp, nhid = model.encoder.weight.shape[1], model.rnn.hidden_size
    masks = [_mask(T * B, ninp, I, p, seed, offset0 + 1)] + [_mask(T * B, nhid, H, p, seed, offset0 + 2 + l)
                                                           for l in range(model.rnn.num_layers)]
    return masks, _ref_stack(model, inp, hidden, masks)


def test_dropout_masks_match_the_generator_and_backward_regenerates_them():
    ntoken, ninp, nhid, nl, T, B, p = 60, 12, 13, 2, 7, 5, 0.3
    model = _model(ntoken, ninp, nhid, nl, seed=9, dropout=p)
    g = torch.Generator().manual_seed(2)
    inp = torch.randint(0, ntoken, (T, B), generator=g)
    hidden = tuple((0.3 * torch.randn(nl, B, nhid, generator=g)).to(DEV).requires_grad_(True) for _ in range(2))
    R = torch.randn(T, B, nhid, generator=g, dtype=torch.float64)
    ops.manual_seed(1234)
    firsts = []
    for call in range(2):                  # successive calls: offsets 1-3, then 4-6
        model.zero_grad(set_to_none=True)
        for t in hidden:
            t.grad = None
        out, _ = ops.lstm_stack(model, inp.to(DEV), hidden, p_emb=p, p_mid=p, p_out=p)
        (out * R.float().to(DEV)).sum().backward()
        masks, (leaves, (o64, _, _)) = _dropout_case(1234, 3 * call, model, inp, hidden, p)
        (o64 * R).sum().backward()
        assert torch.equal(out.cpu() == 0, masks[-1].view(T, B, nhid) == 0)     # the output mask, element for element
        errs = dict(out=_err(out, o64))
        _compare_grads(model, leaves, hidden, errs)
        print(f"dropout call {call}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
        for k, v in errs.items():
            assert v < (H_TOL if k == "out" else GRAD_TOL), (k, v)
        firsts.append(masks)
    assert not torch.equal(firsts[0][0], firsts[1][0])
    # the module's forward draws the same three masks (embedding, between layers, output) in train mode ...
    ops.manual_seed(77)
    decoded, _ = model(inp.to(DEV), tuple(t.detach() for t in hidden))
    masks, (_, (o64, _, _)) = _dropout_case(77, 0, model, inp, hidden, p)
    ref = o64 @ model.decoder.weight.detach().double().cpu().t() + model.decoder.bias.detach().double().cpu()
    assert _err(decoded, ref) < H_TOL
    # ... and none in eval mode
    model.eval()
    decoded, _ = model(inp.to(DEV), tuple(t.detach() for t in hidden))
    _, (o64, _, _) = _ref_stack(model, inp, hidden)
    ref = o64 @ model.decoder.weight.detach().double().cpu().t() + model.decoder.bias.detach().double().cpu()
    assert _err(decoded, ref) < H_TOL


def test_forward_backward_is_reproducible():
    model = _model(500, 64, 96, 2, seed=4, dropout=0.2)
    model.train()
    g = torch.Generator().manual_seed(3)
    inp = torch.randint(0, 500, (35, 20), generator=g).to(DEV)
    tgt = torch.randint(0, 500, (700,), generator=g).to(DEV)
    runs = []
    for _ in range(2):
        ops.manual_seed(99)
        model.zero_grad(set_to_none=True)
        hidden = tuple(t.requires_grad_(True) for t in model.init_hidden(20))
        decoded, (hn, cn) = model(inp, hidden)
        (nn.CrossEntropyLoss()(decoded.view(-1, 500), tgt) + hn.sum() + cn.sum()).backward()
        runs.append([decoded.detach().clone(), hn.detach().clone(), cn.detach().clone(), hidden[0].grad, hidden[1].grad] +
                    [p.grad.clone() for p in model.parameters()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_eval_nll_matches_rescoring_path():
    ntoken, nhid, nl, T, B = 200, 40, 2, 12, 6
    model = _model(ntoken, 24, nhid, nl, seed=6)
    model.eval()
    g = torch.Generator().manual_seed(8)
    ids = torch.randint(0, ntoken, (T + 1, B), generator=g)
    with torch.no_grad():
        decoded, _ = model(ids[:-1].to(DEV), model.init_hidden(B))
        nll = -torch.log_softmax(decoded.double(), -1).gather(2, ids[1:].to(DEV).unsqueeze(-1)).squeeze(-1)
    mine = nll.sum(0).cpu()
    resc = torch.from_numpy(ops.lstm_lm_nll_sums(model, [ids[:, b].numpy() for b in range(B)], DEV)).double()
    e = float(((mine - resc).abs() / resc.abs()).max())
    print(f"eval NLL vs rescoring: max rel err {e:.1e}")
    assert e < 1e-5, e


# ------------------------------------------------------------------------------------------ rejections and fallback
def test_rejections_fallback_and_no_host_sync():
    model = _model(50, 16, 24, 2, seed=1)
    B = 3
    inp = torch.randint(0, 50, (5, B)).to(DEV)
    h = model.init_hidden(B)
    for bad_inp in (inp.int(), inp.cpu(), inp[:, :0], inp.view(-1)):
        with pytest.raises(ValueError):
            model(bad_inp, h)
    for bad in ((h[0][:1], h[1]), (h[0], h[1].double()), (h[0].cpu(), h[1]), (h[0], h[1][:, :2]), (h[0],)):
        with pytest.raises(ValueError):
            model(inp, bad)
    model(inp, h)                                          # warm: operands built, kernels attributed
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        hidden = tuple(t.requires_grad_(True) for t in model.init_hidden(B))
        decoded, (hn, cn) = model(inp, hidden)
        (decoded.square().mean() + hn.sum() + cn.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())


def _reference(flags):
    ns = ref_shim.load(flags, q12_shim=True)
    return ns, importlib.import_module("utils.lstm_utils")


FLAGS = ["--num-layers", "1", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
         "--dim-inner", "64", "--feat_extractor", "", "--tgt-max-len", "8", "--dropout", "0.0", "--cuda"]


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_gru_model_runs_its_own_forward_after_install():
    _, lu = _reference(FLAGS)
    torch.manual_seed(0)
    gru = lu.RNNModel("GRU", 30, 16, 16, 2, dropout=0.0).cuda().eval()
    inp = torch.randint(0, 30, (6, 2)).cuda()
    with torch.no_grad():
        want, _ = gru(inp, gru.init_hidden(2))
        try:
            b200asr.install()
            got, _ = gru(inp, gru.init_hidden(2))
        finally:
            b200asr.uninstall()
    assert torch.equal(got, want)


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_word_lm_loop_installed_matches_cudnn(tmp_path):
    """Five windows of the word-language-model loop (B = 20, bptt = 35, clip 0.25, SGD lr 20, dropout 0) on the reference's
    RNNModel with batches from its own LM.batchify / get_batch, installed vs on cuDNN (fp32, no TF32); then LM.evaluate."""
    _, lu = _reference(FLAGS)
    ntoken, emsize, nhid, nl, B, bptt = 100, 48, 64, 2, 20, 35
    words = ["<eos>", "<oov>"] + [f"w{i}" for i in range(ntoken - 2)]
    w2i = {w: i for i, w in enumerate(words)}
    torch.manual_seed(11)
    rnn = lu.RNNModel("LSTM", ntoken, emsize, nhid, nl, dropout=0.0)
    path = tmp_path / "lm.pt"
    torch.save(dict(word2idx=w2i, idx2word=words, ntoken=ntoken, ninp=emsize, nhid=nhid, nlayers=nl, dropout=0.0, tie_weights=False,
                    model_state_dict=rnn.state_dict()), path)
    corpus = torch.randint(0, ntoken, (B * bptt * 5 + B,), generator=torch.Generator().manual_seed(5))
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    def loop(lm, model, cuda):
        model.train()
        data = lm.batchify(corpus, B, cuda)
        hidden = model.init_hidden(B)
        crit = nn.CrossEntropyLoss()
        losses = []
        for i in range(0, 5 * bptt, bptt):
            x, y = lm.get_batch(data, i, bptt)
            hidden = lm.repackage_hidden(hidden)
            model.zero_grad()
            output, hidden = model(x, hidden)
            loss = crit(output.view(-1, ntoken), y)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), 0.25)
            for p in model.parameters():
                p.data.add_(p.grad, alpha=-20.0)
            losses.append(loss.item())
        return losses, {k: v.detach().cpu().double() for k, v in model.state_dict().items()}

    runs = {}
    try:
        for installed in (False, True):
            if installed:
                b200asr.install()
            lm = lu.LM(str(path))
            runs[installed] = loop(lm, lm.model, True) + (float(lm.evaluate("w1 w2 w3 w7 zz w9")[0]),)
    finally:
        b200asr.uninstall()
    lm = lu.LM(str(path))
    f64 = loop(lm, lm.model.cpu().double(), False)            # the same loop in float64 (CPU), the yardstick of both
    dist = lambda r: (max(abs(a - b) / abs(b) for a, b in zip(r[0], f64[0])), max(_err(r[1][k], f64[1][k]) for k in f64[1]))
    (le0, pe0), (le1, pe1) = dist(runs[False]), dist(runs[True])
    ee = abs(runs[True][2] - runs[False][2]) / abs(runs[False][2])
    print(f"word LM loop vs float64: losses max rel {le1:.1e} installed, {le0:.1e} cuDNN; final parameters max rel {pe1:.1e} "
          f"installed, {pe0:.1e} cuDNN; evaluate installed vs cuDNN rel {ee:.1e}")
    # SGD at lr 20 moves the parameters by 5 (the clip norm times lr) per window, so rounding differences grow along the
    # trajectory; each path is held to the float64 loop, the installed one within 50x cuDNN's own distance from it.
    assert le1 <= 50 * le0 + 1e-5 and pe1 <= 50 * pe0 + 1e-4, (le1, le0, pe1, pe0)
    assert ee < 50 * max(le0, 1e-6), ee
