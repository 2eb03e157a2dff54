"""Beam search with LSTM-LM rescoring on the device (csrc/lstm.cu, csrc/beam.cu's end log, Decoder.beam_decode(lm=...)).

  * The LSTM stack (b200asr_lstm_prepare, the input-projection GEMM, b200asr_lstm_layer_fwd) against float64 nn.LSTM for
    nhid in {8, 48, 50, 200, 650, 1024}, ninp != nhid, 1-3 layers, 1 / 127 / 128 / 129 / 300 sequences with lengths all 1,
    ragged and all equal; padded units must read back as exactly 0.
  * b200asr_lm_nll against float64 for ntoken 2 .. 50001 (logits also shifted by +200); lm_seq_sum bit-identical across calls.
  * b200asr_beam_step_log: the end log equals a host restatement (forced endings included); the packed backtrack walks it.
  * Every rejection returns its status and message and leaves the outputs untouched.
  * Decoder.beam_decode(lm=...) reproduces tests/golden/beam_lm.npz; lm_weight = c_weight = 0 equals beam_decode(c_weight=0);
    two calls agree bit for bit; the reference's evaluate(beam_search=True, lm_rescoring=True) gives the same strings
    installed and uninstalled.
Outputs and workspaces are NaN-poisoned first.  Bars state the error measured on one H100 80GB HBM3 (700 W power limit) and sit about 3x above it.
"""
import math

import numpy as np
import pytest
import torch

import b200asr
import b200asr.modules as M
import b200asr.ops as ops
from oracle import beam_oracle as BO
from oracle import lm_oracle as LO
from oracle import ref_shim
from tests.beam_lm_util import load_beam_lm_golden
from tests.test_gpu_beam_search import MARGIN_BAR, ref_beam_step, _recs

pytestmark = pytest.mark.gpu

L = b200asr._lib
DEV = "cuda"
LSTM_TOL = 1.2e-4      # LSTM layer outputs vs float64, max |err| (|h| < 1; measured 3.9e-5 max, nhid = 8, 127 sequences)
NLL_RTOL = 2.5e-5      # lm_nll vs float64, relative to max(1, |nll|) (measured 7.6e-6 max with logits near +200, where the
                       # fp32 logits' own spacing is 1.5e-5; 3.3e-7 without the shift)
SCORE_RTOL = 5e-4      # beam_decode(lm) scores and final scores vs the reference's fp32 CPU ones (measured 1.6e-4 max)


def _lib():
    return L.load()


def _lm_model(ntoken, ninp, nhid, nlayers, tie=False, seed=0, scale=0.5):
    torch.manual_seed(seed)
    m = M.RNNModel("LSTM", ntoken, ninp, nhid, nlayers, dropout=0.0, tie_weights=tie)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(scale * torch.randn(p.shape))
    return m.to(DEV)


def _pack(lens):
    lens = np.asarray(lens)
    order = np.argsort(-lens, kind="stable")
    T = int(lens.max())
    Mt = np.array([(lens > t).sum() for t in range(T)])
    off = np.concatenate([[0], np.cumsum(Mt)[:-1]])
    return order, Mt, off


# ------------------------------------------------------------------------------------------ LSTM stack vs float64
@pytest.mark.parametrize("nhid,ninp,nlayers", [(8, 12, 1), (48, 32, 2), (50, 40, 3), (200, 96, 2), (650, 400, 2), (1024, 512, 1)])
@pytest.mark.parametrize("nseq", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("shape", ["ones", "ragged", "equal"])
def test_lstm_layers_match_float64(nhid, ninp, nlayers, nseq, shape):
    g = np.random.default_rng(nhid * 1000 + nseq)
    ntoken = 97
    lens = {"ones": np.ones(nseq, int), "ragged": g.integers(1, 24, nseq), "equal": np.full(nseq, 9)}[shape]
    model = _lm_model(ntoken, ninp, nhid, nlayers, seed=nseq, scale=1.0 / math.sqrt(nhid) * 2)
    op = ops.lstm_lm_operands(model, DEV)
    order, Mt, off = _pack(lens)
    P = int(Mt.sum())
    seqs = [g.integers(0, ntoken, int(n)) for n in lens]
    inp = np.empty(P, dtype=np.int64)
    for j, s in enumerate(order):
        inp[off[:lens[s]] + j] = seqs[s]
    outs = ops.lstm_lm_layers(op, torch.from_numpy(inp).to(DEV), Mt)
    torch.cuda.synchronize()
    ref = torch.nn.LSTM(ninp, nhid, nlayers).double()
    ref.load_state_dict({k[4:]: v.double().cpu() for k, v in model.state_dict().items() if k.startswith("rnn.")})
    emb = model.encoder.weight.detach().double().cpu()
    worst = 0.0
    last = outs[-1].cpu()
    H = op.H
    assert last.shape == (P, H)
    assert (last[:, nhid:] == 0).all()                       # padded units stay exactly 0
    for o in outs:
        assert not o.isnan().any()
    with torch.no_grad():
        for j, s in enumerate(order):
            y, _ = ref(emb[torch.from_numpy(seqs[s])].unsqueeze(1))
            mine = last[off[:lens[s]] + j, :nhid].double()
            e = float((mine - y[:, 0]).abs().max())
            worst = max(worst, e)
    print(f"lstm nhid={nhid} ninp={ninp} L={nlayers} nseq={nseq} {shape}: max abs err {worst:.2e}")
    assert worst < LSTM_TOL, worst


def test_lstm_operands_refresh_when_a_parameter_changes():
    model = _lm_model(50, 16, 24, 1)
    a = ops.lstm_lm_operands(model, DEV)
    assert ops.lstm_lm_operands(model, DEV) is a
    with torch.no_grad():
        model.rnn.weight_hh_l0.mul_(0.5)
    b = ops.lstm_lm_operands(model, DEV)
    assert b is not a and not torch.equal(a.layers[0][2], b.layers[0][2])


# ------------------------------------------------------------------------------------------ NLL
@pytest.mark.parametrize("V", [2, 3, 255, 256, 257, 10000, 50001])
@pytest.mark.parametrize("shift", [0.0, 200.0])
def test_lm_nll_matches_float64_and_sums_are_reproducible(V, shift):
    g = torch.Generator().manual_seed(V)
    rows = 67
    x = torch.randn(rows, V, generator=g) * 4 + shift
    ld = V + 3
    xd = torch.full((rows, ld), float("nan"), device=DEV)
    xd[:, :V] = x.to(DEV)
    tg = torch.randint(0, V, (rows,), generator=g)
    tgd = tg.to(DEV)
    nll = torch.full((rows,), float("nan"), device=DEV)
    rc = _lib().b200asr_lm_nll(L.ptr(xd), ld, L.ptr(tgd), L.ptr(nll), rows, V, None)
    assert rc == 0, L.last_error()
    ref = torch.logsumexp(x.double(), 1) - x.double()[torch.arange(rows), tg]
    e = float(((nll.cpu().double() - ref).abs() / ref.abs().clamp_min(1.0)).max())
    print(f"lm_nll V={V} shift={shift}: max rel err {e:.2e}")
    assert e < NLL_RTOL, e
    lens = torch.tensor([5, 4, 4, 2, 1], dtype=torch.int64)          # M_t = 5, 4, 3, 3, 1
    off = torch.tensor([0, 5, 9, 12, 15], dtype=torch.int64)
    offd, lensd = off.to(DEV), lens.to(DEV)
    outs = []
    for _ in range(2):
        sums = torch.full((5,), float("nan"), device=DEV)
        rc = _lib().b200asr_lm_seq_sum(L.ptr(nll), L.ptr(offd), L.ptr(lensd), 5, L.ptr(sums), None)
        assert rc == 0, L.last_error()
        outs.append(sums.cpu())
    assert torch.equal(outs[0], outs[1])
    n = nll.cpu().double()
    for s in range(5):
        want = sum(float(n[int(off[t]) + s]) for t in range(int(lens[s])))
        assert abs(float(outs[0][s]) - want) <= 1e-5 * max(1.0, abs(want))


# ------------------------------------------------------------------------------------------ end log
@pytest.mark.parametrize("W", [2, 4, 8])
def test_beam_step_log_matches_host_restatement(W):
    V, B, steps, t_eos = 33, 3, 6, 4
    recs = _recs(V)
    cap = W * steps
    g = torch.Generator().manual_seed(W)
    R = B * W
    state = torch.zeros(R, 4, dtype=torch.int32)
    state[::W, 0] = 1
    state[:, 3] = -1
    score = torch.full((R,), float("-inf"))
    score[::W] = 0.0
    idx = (torch.arange(R, dtype=torch.int32) % W).view(R, 1)
    d = {k: v.to(DEV) for k, v in dict(state=state, score=score).items()}
    args = dict(tab=torch.tensor(recs, dtype=torch.int32, device=DEV), tok=torch.full((R,), -1, device=DEV, dtype=torch.long),
                hist_tok=torch.full((steps, R), -1, device=DEV, dtype=torch.int32),
                hist_par=torch.full((steps, R), -1, device=DEV, dtype=torch.int32),
                ps=torch.full((B, 32), float("nan"), device=DEV), pf=torch.full((B, 32), float("nan"), device=DEV),
                pr=torch.full((B, 32), -1, device=DEV, dtype=torch.int32), pn=torch.zeros(B, device=DEV, dtype=torch.int32),
                live=torch.full((1,), B, device=DEV, dtype=torch.int32))
    idxs = [torch.full((R, steps + 1), -1, device=DEV, dtype=torch.int32) for _ in range(2)]
    idxs[0][:, :1] = idx.to(DEV)
    end_ref = torch.full((B, cap), -1, device=DEV, dtype=torch.int32)
    end_sc = torch.full((B, cap), float("nan"), device=DEV)
    end_n = torch.zeros(B, device=DEV, dtype=torch.int32)
    host_pool = [[] for _ in range(B)]
    P = L.ptr
    for t in range(t_eos + 1):
        logits = torch.randn(R, V, generator=g) * 2
        logits[:, 2] += torch.randn(R, generator=g) * 2 + 1      # EOS chosen by some rows
        exp = ref_beam_step(logits, recs, W, t, t_eos, 32, 0.1, d["score"].cpu(), d["state"].cpu(), idxs[t % 2].cpu()[:, :t + 1],
                            host_pool)
        host_pool = exp["pool"]
        rc = _lib().b200asr_beam_step_log(P(logits.to(DEV)), P(args["tab"]), B, W, V, t, t_eos, steps, 32, 0.1, P(d["score"]),
                                          P(d["state"]), P(args["tok"]), P(idxs[t % 2]), P(idxs[(t + 1) % 2]), steps + 1,
                                          P(args["hist_tok"]), P(args["hist_par"]), P(args["ps"]), P(args["pf"]), P(args["pr"]),
                                          P(args["pn"]), P(args["live"]), P(end_ref), P(end_sc), P(end_n), cap, None)
        assert rc == 0, L.last_error()
        if int(args["live"].item()) == 0:
            break
    torch.cuda.synchronize()
    n, refs, sc = end_n.cpu(), end_ref.cpu(), end_sc.cpu()
    total = 0
    for b in range(B):
        want = sorted(host_pool[b], key=lambda e: e[2])            # every ended entry (< 32 here), in insertion order
        assert int(n[b]) == len(want)
        assert refs[b, :len(want)].tolist() == [e[2] for e in want]
        for i, (_, s, _) in enumerate(want):
            assert abs(float(sc[b, i]) - s) <= 2e-6 * max(1.0, abs(s))
        assert (refs[b, len(want):] == -1).all() and sc[b, len(want):].isnan().all()
        assert any(e[2] & 1 for e in want) or int(args["live"].item()) == 0 or t < t_eos
        total += len(want)
    assert total > 0 and any(int(r) & 1 for r in refs.flatten() if r >= 0)         # forced endings present
    # packed backtrack: the walk of every entry, laid out back to back
    ents = np.concatenate([b * cap + np.arange(int(n[b])) for b in range(B)]).astype(np.int64)
    r = refs.flatten().numpy().astype(np.int64)[ents]
    lens = (r >> 1) // W + 2 + (r & 1)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    up = torch.from_numpy(np.concatenate([ents, offs])).to(DEV)
    ids = torch.full((int(lens.sum()) + 5,), -7, device=DEV, dtype=torch.long)
    rc = _lib().b200asr_beam_backtrack_packed(P(args["hist_tok"]), P(args["hist_par"]), P(end_ref), P(end_n), cap, P(up),
                                              up.data_ptr() + 8 * len(ents), len(ents), P(ids), B, W, steps, None)
    assert rc == 0, L.last_error()
    ids = ids.cpu()
    ht, hp = args["hist_tok"].cpu(), args["hist_par"].cpu()
    for j, e in enumerate(ents):
        b, ref = int(e) // cap, int(r[j])
        tt, k = (ref >> 1) // W, (ref >> 1) % W
        y = []
        for s in range(tt, -1, -1):
            y.append(int(ht[s, b * W + k]))
            k = int(hp[s, b * W + k])
        want = [1] + y[::-1] + ([2] if ref & 1 else [])
        assert ids[offs[j]:offs[j] + lens[j]].tolist() == want
    assert (ids[int(lens.sum()):] == -7).all()


# ------------------------------------------------------------------------------------------ rejections
def test_rejections_leave_outputs_untouched():
    P = L.ptr
    x = torch.zeros(4096, device=DEV)
    h = torch.full((4096,), float("nan"), device=DEV)
    c = torch.full((4096,), float("nan"), device=DEV)
    w16 = torch.zeros(8192, device=DEV, dtype=torch.bfloat16)
    cases = [(np.array([3, 2], np.int32), 12, "multiple of 8"), (np.array([2, 3], np.int32), 8, "non-increasing"),
             (np.array([0], np.int32), 8, "non-increasing")]
    for bs, H, msg in cases:
        rc = _lib().b200asr_lstm_layer_fwd(P(x), P(w16), bs.ctypes.data, len(bs), H, P(c), P(h), None)
        assert rc == -1 and L.last_error().startswith("lstm_layer_fwd:") and msg in L.last_error(), L.last_error()
    bs = np.array([1], np.int32)
    assert _lib().b200asr_lstm_layer_fwd(None, P(w16), bs.ctypes.data, 1, 8, P(c), P(h), None) == -5
    assert _lib().b200asr_lstm_layer_fwd(P(x), P(w16), bs.ctypes.data, 0, 8, P(c), P(h), None) == -1
    assert _lib().b200asr_lstm_prepare(P(x), P(x), None, None, 0, 8, P(h), P(h), P(h), None) == -1
    assert L.last_error().startswith("lstm_prepare:")
    tg = torch.zeros(4, device=DEV, dtype=torch.long)
    assert _lib().b200asr_lm_nll(P(x), 4, P(tg), P(h), 4, 5, None) == -1 and L.last_error().startswith("lm_nll:")
    assert _lib().b200asr_lm_nll(P(x), 4, P(tg), P(h), 4, 0, None) == -1
    assert _lib().b200asr_lm_seq_sum(P(x), None, P(tg), 1, P(h), None) == -5 and L.last_error().startswith("lm_seq_sum:")
    i32 = torch.zeros(64, device=DEV, dtype=torch.int32)
    rc = _lib().b200asr_beam_step_log(P(x), P(i32), 1, 2, 8, 0, 5, 4, 1, 0.1, P(h), P(i32), P(tg), P(i32), P(i32[32:]), 5,
                                      P(i32), P(i32), P(h), P(h), P(i32), P(i32), P(i32), P(i32), P(h), P(i32), 7, None)
    assert rc == -1 and L.last_error().startswith("beam_step_log:") and "end_cap" in L.last_error()
    rc = _lib().b200asr_beam_backtrack_packed(P(i32), P(i32), P(i32), P(i32), 4, None, P(tg), 1, P(tg), 1, 2, 4, None)
    assert rc == -5 and L.last_error().startswith("beam_backtrack_packed:")
    torch.cuda.synchronize()
    assert h.isnan().all() and c.isnan().all()


# ------------------------------------------------------------------------------------------ decoder level
@pytest.fixture(scope="module")
def golden():
    cfg, id2label, w2i, lms, cases = load_beam_lm_golden()
    for c in cases:
        P = {k: v.double() for k, v in c["P"].items()}
        c["oracle"] = BO.beam_search(P, cfg, c["enc"].double(), c["W"], c["nbest"], c["c_weight"], id2label)
        lm = lms[c["lm"]]
        PL = {k: v.double() for k, v in lm["P"].items()}
        c["ofinal"] = []
        for h in c["ended"]:
            s, nw, _, _ = LO.lm_score(h["yseq"], id2label, w2i, PL, lm["nlayers"])
            c["ofinal"].append(LO.final_score(h["score"], s, nw, c["lm_weight"], c["c_weight"]))
    return cfg, id2label, w2i, lms, cases


def _decoder(cfg, P, id2label):
    from oracle import asr_oracle as O
    from tests.gpu_util import cuda_model
    full = dict(O.init_params(cfg, seed=1))
    full.update(P)
    model = cuda_model(cfg, full, train=True)
    model.decoder.id2label = id2label
    return model.decoder


class _LM:
    def __init__(self, spec, w2i):
        self.word2idx = w2i
        self.model = M.RNNModel("LSTM", spec["ntoken"], spec["ninp"], spec["nhid"], spec["nlayers"], dropout=0.0,
                                tie_weights=spec["tie"])
        self.model.load_state_dict(spec["P"])
        self.model.to(DEV).eval()


def test_beam_decode_with_lm_matches_reference_fixture(golden):
    cfg, id2label, w2i, lms, cases = golden
    n_ok = n_all = 0
    worst = 0.0
    for ci, c in enumerate(cases):
        dec = _decoder(cfg, c["P"], id2label)
        lm = _LM(lms[c["lm"]], w2i)
        enc = c["enc"].to(DEV)
        ids, lengths, score, final = [x.cpu() for x in dec.beam_decode(enc, c["W"], nbest=c["nbest"], c_weight=c["c_weight"], lm=lm,
                                                                       lm_weight=c["lm_weight"])]
        assert dec.training
        ys, strs = dec.beam_search(enc, beam_width=c["W"], nbest=c["nbest"], lm_rescoring=True, lm=lm, lm_weight=c["lm_weight"],
                                   c_weight=c["c_weight"])
        k = 0
        for b in range(enc.shape[0]):
            n_all += 1
            mine = [ids[b, i, :int(n)].tolist() for i, n in enumerate(lengths[b]) if int(n) > 0]
            for y in mine:
                assert ys[k] == y and strs[k] == "".join(id2label[t] for t in y[1:])
                k += 1
            js = [j for j, h in enumerate(c["ended"]) if h["utt"] == b]
            fin = sorted((c["ofinal"][j] for j in js), reverse=True)[:c["nbest"] + 1]
            pool_margin = min([fin[i] - fin[i + 1] for i in range(len(fin) - 1)] or [math.inf])
            margin = min(c["oracle"][b]["step_margins"] + [pool_margin])
            want = [c["ended"][int(j)]["yseq"] for j in c["nbest_idx"][b] if j >= 0]
            print(f"case {ci} utterance {b}: margin {margin:.2e}, same n-best as the reference: {mine == want}")
            if margin <= MARGIN_BAR:
                continue
            assert mine == want, (ci, b)
            m = len(want)
            ref_f = torch.tensor([c["ended"][int(j)]["final"] for j in c["nbest_idx"][b][:m]], dtype=torch.float64)
            ref_s = torch.tensor([c["ended"][int(j)]["score"] for j in c["nbest_idx"][b][:m]], dtype=torch.float64)
            e = float(((final[b, :m].double() - ref_f).abs() / ref_f.abs().clamp_min(1.0)).max())
            e = max(e, float(((score[b, :m].double() - ref_s).abs() / ref_s.abs().clamp_min(1.0)).max()))
            worst = max(worst, e)
            assert e < SCORE_RTOL, (ci, b, e)
            assert torch.isnan(score[b, m:]).all() and (lengths[b, m:] == 0).all()
            n_ok += 1
        assert k == len(ys)
    print(f"beam_decode(lm): {n_ok}/{n_all} utterances compared, max rel score err {worst:.2e}")
    assert n_ok * 4 >= n_all * 3, (n_ok, n_all)


def test_lm_weight_zero_equals_beam_decode_without_lm(golden):
    cfg, id2label, w2i, lms, cases = golden
    c = cases[3]
    dec = _decoder(cfg, c["P"], id2label)
    enc = c["enc"].to(DEV)
    a = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=8, c_weight=0.0, lm=_LM(lms[0], w2i), lm_weight=0.0)]
    b = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=8, c_weight=0.0)]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(a[2].isnan(), b[2].isnan()) and torch.equal(a[2].nan_to_num(), b[2].nan_to_num())


def test_beam_decode_with_lm_is_reproducible(golden):
    cfg, id2label, w2i, lms, cases = golden
    c = cases[4]
    dec = _decoder(cfg, c["P"], id2label)
    lm = _LM(lms[1], w2i)
    enc = c["enc"].to(DEV)
    a = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=4, c_weight=1.0, lm=lm, lm_weight=5.0)]
    b = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=4, c_weight=1.0, lm=lm, lm_weight=5.0)]
    for x, y in zip(a, b):
        assert torch.equal(x.isnan(), y.isnan()) and torch.equal(x.nan_to_num(), y.nan_to_num())


def test_mirror_lm_loads_the_reference_checkpoint_format(tmp_path, golden):
    _, _, w2i, lms, _ = golden
    spec = lms[1]
    path = tmp_path / "lm.pt"
    torch.save(dict(word2idx=w2i, idx2word=list(w2i), ntoken=spec["ntoken"], ninp=spec["ninp"], nhid=spec["nhid"],
                    nlayers=spec["nlayers"], dropout=0.2, tie_weights=spec["tie"], model_state_dict=spec["P"]), path)
    lm = b200asr.LM(str(path))
    assert lm.model.decoder.weight is lm.model.encoder.weight
    assert M.lstm_lm_parts(lm) is not None and M.lstm_lm_parts(object()) is None


# ------------------------------------------------------------------------------------------ the reference's evaluate
@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_evaluate_with_lm_rescoring_installed_matches_uninstalled(tmp_path):
    import importlib
    flags = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
             "--dim-inner", "128", "--feat_extractor", "", "--tgt-max-len", "301", "--dropout", "0.0", "--cuda"]
    ns = ref_shim.load(flags, q12_shim=True)
    lstm_utils = importlib.import_module("utils.lstm_utils")
    V = 40
    l2i, i2l = ref_shim.labels(V)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.decoder.output_linear.weight.mul_(4.0)
        model.decoder.output_linear.weight[2] *= -1.0
    model = model.cuda().eval()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    words = ["<eos>", "<oov>"] + sorted({w for s in i2l.values() for w in s.split()})[:20]
    w2i = {w: i for i, w in enumerate(words)}
    torch.manual_seed(3)
    rnn = lstm_utils.RNNModel("LSTM", len(words), 24, 40, 2, dropout=0.0)
    with torch.no_grad():
        for p in rnn.parameters():
            p.copy_(0.5 * torch.randn(p.shape))
    path = tmp_path / "lm.pt"
    torch.save(dict(word2idx=w2i, idx2word=words, ntoken=len(words), ninp=24, nhid=40, nlayers=2, dropout=0.0, tie_weights=False,
                    model_state_dict=rnn.state_dict()), path)
    lm = lstm_utils.LM(str(path))
    src = torch.randn(2, 1, 161, 24, generator=g).cuda()
    lens = torch.full((2,), 24, dtype=torch.int32).cuda()
    tgt = torch.randint(3, V, (2, 6), generator=g).cuda()
    results = {}
    try:
        for installed in (False, True):
            if installed:
                b200asr.install()
            with torch.no_grad():
                _, strs, _ = model.evaluate(src, lens, tgt, beam_search=True, beam_width=4, beam_nbest=1, lm_rescoring=True, lm=lm,
                                            lm_weight=2.0, c_weight=0.1)
            results[installed] = list(strs)
    finally:
        b200asr.uninstall()
    assert results[True] == results[False], results
