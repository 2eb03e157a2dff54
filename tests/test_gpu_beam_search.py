"""Beam search on the device (csrc/beam.cu, Decoder.beam_decode / beam_search) against float64 and against the reference.

  * b200asr_beam_step through the C ABI against a host float64 restatement: W in {1, 2, 3, 8, 16, 32}, V in {W, 33, 4364};
    utterances with 1..W live rows; the forced-EOS step; EOS chosen by some rows and not others; exact ties within a row and
    across parents; pool insertion with equal final scores; the index table after reordering; the live counter; every
    rejection (status, message, outputs untouched).
  * b200asr_beam_self_attn against float64 for every (dk, dv) in {16, 32, 64, 128}^2 and histories of 2 to 301 positions,
    with random index tables and with every row pointing at one slot.
  * Decoder.beam_decode / beam_search on tests/golden/beam.npz's model return the reference's yseqs and strings for every
    utterance whose float64 decision margins all exceed the bar; W = 1 is greedy decoding; two calls agree bit for bit.
  * The reference's own Transformer.evaluate(..., beam_search=True) gives the same strings uninstalled and installed,
    including a batch that falls back to greedy_search.
Every output and workspace is poisoned first (NaN, or -1 for integers).  Bars state the error measured on one H100 80GB HBM3
(400 W power limit) and sit about 3x above it.
"""
import math

import numpy as np
import pytest
import torch

import b200asr
import b200asr.modules as M
from oracle import asr_oracle as O
from oracle import beam_oracle as BO
from oracle import ref_shim
from tests.beam_util import golden_yseqs, load_beam_golden

pytestmark = pytest.mark.gpu

L = b200asr._lib
DEV = "cuda"
SCORE_RTOL = 2e-6         # beam_step scores and pooled final scores vs float64 (measured 6.2e-7 max, V = 4364)
ATTN_TOL = 6e-6           # beam_self_attn vs float64, max |err| / max |ref| (measured 1.9e-6 max, dk = 128, dv = 64)
DECODE_RTOL = 2.5e-4      # beam_decode scores vs the reference's fp32 CPU scores, up to 40 steps (measured 8.5e-5 max)
MARGIN_BAR = 1.2e-3       # a hypothesis's score differs from the reference's by up to 4.2e-4 (measured): decisions whose
                          # float64 margin is below ~3x that may legitimately go either way


def _lib():
    return L.load()


def _i32(*shape, fill=-1):
    return torch.full(shape, fill, device=DEV, dtype=torch.int32)


# ------------------------------------------------------------------------------------------ beam_step: host restatement
def ref_beam_step(logits, recs, W, t, t_eos, nbest, c_weight, score, state, idx_cur, pool):
    """float64 restatement of one step.  Returns (kept per utterance, new score/state/next_tok/idx rows, pools, dead count)."""
    B = logits.shape[0] // W
    lg = logits.double().cpu()
    exp = dict(score=score.clone(), state=state.clone(), tok={}, idx={}, hist={}, pool=[list(p) for p in pool], died=0)
    for b in range(B):
        live = [j for j in range(W) if state[b * W + j, 0]]
        cands = []
        for j in live:
            x = lg[b * W + j]
            lp = (x - torch.logsumexp(x, 0)).tolist()
            order = sorted(range(len(lp)), key=lambda v: (-lp[v], v))[:W]
            cands += [(float(score[b * W + j]) + lp[v], j * W + r, v, j) for r, v in enumerate(order)]
        kept = sorted(cands, key=lambda c: (-c[0], c[1]))[:W]
        n = 0
        for k, (s, _, v, j) in enumerate(kept):
            words, tail = int(state[b * W + j, 1]), int(state[b * W + j, 2])
            r = recs[v]
            words += (r >> 3) - (tail & ((r >> 2) & 1))
            if not r & 1:
                tail = (r >> 1) & 1
            exp["hist"][(b, k)] = (v, int(state[b * W + j, 3]))
            if t == t_eos or v == 2:
                fs = s + math.sqrt(words) * c_weight
                p = exp["pool"][b]
                pos = 0
                while pos < len(p) and not fs > p[pos][0]:
                    pos += 1
                p.insert(pos, (fs, s, ((t * W + k) << 1) | (t == t_eos)))
                del p[nbest:]
            else:
                exp["score"][b * W + n] = s
                exp["state"][b * W + n] = torch.tensor([1, words, tail, k])
                exp["tok"][b * W + n] = v
                exp["idx"][b * W + n] = idx_cur[b * W + j, :t + 1].tolist() + [n]
                n += 1
        for s_ in range(n, W):
            exp["score"][b * W + s_] = float("-inf")
            exp["state"][b * W + s_] = torch.tensor([0, 0, 0, -1])
            exp["tok"][b * W + s_] = 0
            exp["idx"][b * W + s_] = [s_] * (t + 2)
        exp["died"] += int(len(kept) > 0 and n == 0)
    return exp


def run_beam_step(logits, recs, W, t, t_eos, nbest, c_weight, score, state, idx_cur, pool, steps=40, stride=None):
    """Poisons every output, calls the C ABI and returns (rc, device buffers)."""
    R, V = logits.shape
    B = R // W
    stride = stride or steps + 1
    d = dict(logits=logits.to(DEV).contiguous(), tab=torch.tensor(recs, dtype=torch.int32, device=DEV),
             score=score.to(DEV).clone(), state=state.to(DEV).clone(), tok=torch.full((R,), -1, device=DEV, dtype=torch.long),
             idx_cur=torch.full((R, stride), -1, device=DEV, dtype=torch.int32), idx_nxt=_i32(R, stride),
             hist_tok=_i32(steps, R), hist_par=_i32(steps, R),
             pool_score=torch.full((B, nbest), float("nan"), device=DEV), pool_final=torch.full((B, nbest), float("nan"), device=DEV),
             pool_ref=_i32(B, nbest), pool_n=torch.zeros(B, device=DEV, dtype=torch.int32),
             n_live=torch.full((1,), B, device=DEV, dtype=torch.int32))
    d["idx_cur"][:, :idx_cur.shape[1]] = idx_cur.to(DEV)
    for b, p in enumerate(pool):
        for i, (fs, s, ref) in enumerate(p):
            d["pool_final"][b, i], d["pool_score"][b, i], d["pool_ref"][b, i] = fs, s, ref
        d["pool_n"][b] = len(p)
    P = L.ptr
    rc = _lib().b200asr_beam_step(P(d["logits"]), P(d["tab"]), B, W, V, t, t_eos, steps, nbest, float(c_weight), P(d["score"]),
                                  P(d["state"]), P(d["tok"]), P(d["idx_cur"]), P(d["idx_nxt"]), stride, P(d["hist_tok"]),
                                  P(d["hist_par"]), P(d["pool_score"]), P(d["pool_final"]), P(d["pool_ref"]), P(d["pool_n"]),
                                  P(d["n_live"]), None)
    torch.cuda.synchronize()
    return rc, d


def check_beam_step(exp, d, W, t, nbest):
    R = d["score"].shape[0]
    B = R // W
    state, score = d["state"].cpu(), d["score"].cpu()
    assert torch.equal(state, exp["state"])
    live = exp["state"][:, 0] == 1
    err = ((score[live].double() - exp["score"][live].double()).abs() / exp["score"][live].double().abs().clamp_min(1.0)).max() \
        if live.any() else torch.tensor(0.0)
    assert float(err) < SCORE_RTOL, float(err)
    print(f"beam_step W={W} t={t}: max rel score err {float(err):.2e}")
    assert torch.isinf(score[~live]).all() and (score[~live] < 0).all()
    tok, idx = d["tok"].cpu(), d["idx_nxt"].cpu()
    for r in range(R):
        assert int(tok[r]) == exp["tok"][r], r
        assert idx[r, :t + 2].tolist() == exp["idx"][r], (r, idx[r, :t + 2].tolist(), exp["idx"][r])
        assert (idx[r, t + 2:] == -1).all()
    ht, hp = d["hist_tok"].cpu(), d["hist_par"].cpu()
    for (b, k), (v, par) in exp["hist"].items():
        assert int(ht[t, b * W + k]) == v and int(hp[t, b * W + k]) == par, (b, k)
    written = torch.zeros_like(ht, dtype=torch.bool)
    for (b, k) in exp["hist"]:
        written[t, b * W + k] = True
    assert (ht[~written] == -1).all() and (hp[~written] == -1).all()
    pn, pf, ps, pr = d["pool_n"].cpu(), d["pool_final"].cpu(), d["pool_score"].cpu(), d["pool_ref"].cpu()
    for b in range(B):
        p = exp["pool"][b]
        assert int(pn[b]) == len(p)
        assert pr[b, :len(p)].tolist() == [e[2] for e in p], (b, pr[b].tolist(), p)
        for i, (fs, s, _) in enumerate(p):
            assert abs(float(pf[b, i]) - fs) <= SCORE_RTOL * max(1.0, abs(fs)) and abs(float(ps[b, i]) - s) <= SCORE_RTOL * max(1.0, abs(s))
        assert torch.isnan(pf[b, len(p):]).all() and (pr[b, len(p):] == -1).all()
    assert int(d["n_live"].item()) == B - exp["died"]


def _recs(V):
    labels = {0: "¶", 1: "§", 2: "¤"}
    pieces = [" ", "a", "b c", " d", "e ", "", "¤"]
    g = np.random.default_rng(V)
    for v in range(3, V):
        labels[v] = "".join(pieces[i] for i in g.integers(0, len(pieces), 2))
    return M.word_records(labels, V)


def _setup(W, V, seed, eos_rows=()):
    """Three utterances with W, 1 and about W/2 live rows (compacted), random scores / word states / histories."""
    g = torch.Generator().manual_seed(seed)
    B, t = 3, 5
    R = B * W
    logits = torch.randn(R, V, generator=g) * 3.0
    for r in eos_rows:
        if r < R:
            logits[r, 2] = logits[r].max() + 2.0
    nlive = [W, 1, max(1, (W + 1) // 2)]
    state = torch.zeros(R, 4, dtype=torch.int32)
    state[:, 3] = -1
    score = torch.full((R,), float("-inf"))
    for b, n in enumerate(nlive):
        for j in range(n):
            r = b * W + j
            state[r] = torch.tensor([1, int(torch.randint(0, 5, (1,), generator=g)), int(torch.randint(0, 2, (1,), generator=g)), j])
            score[r] = -float(torch.rand(1, generator=g)) * 10
    idx = torch.randint(0, W, (R, t + 1), generator=g, dtype=torch.int32)
    return logits, state, score, idx, t


@pytest.mark.parametrize("W", [1, 2, 3, 8, 16, 32])
@pytest.mark.parametrize("V", ["W", 33, 4364])
@pytest.mark.parametrize("forced", [False, True])
def test_beam_step_matches_float64(W, V, forced):
    V = W if V == "W" else V
    if V < 3:
        V = 3 if W <= 3 else W                  # EOS must exist
    if W > V:
        pytest.skip("W > V is a rejection (test_beam_step_rejections)")
    logits, state, score, idx, t = _setup(W, V, seed=W * 1000 + V, eos_rows=(0, 2, W + 0))
    recs = _recs(V)
    nbest = min(W, 5)
    t_eos = t if forced else t + 4
    pool = [[(-30.0, -30.0, 77)], [], []]
    exp = ref_beam_step(logits, recs, W, t, t_eos, nbest, 0.1, score, state, idx, pool)
    rc, d = run_beam_step(logits, recs, W, t, t_eos, nbest, 0.1, score, state, idx, pool)
    assert rc == 0, L.last_error()
    check_beam_step(exp, d, W, t, nbest)
    if forced:
        assert int(d["n_live"].item()) == 0 and (d["state"][:, 0] == 0).all()


@pytest.mark.parametrize("W", [2, 3, 8])
def test_beam_step_exact_ties_and_stable_pool(W):
    """Equal logits within a row (the lower token id first), identical parents (the earlier parent first) and ended
    hypotheses whose final scores equal each other and a pooled entry (the earlier entry stays first)."""
    V = 33
    B, R, t = 2, 2 * W, 3
    logits = torch.full((R, V), -5.0)
    logits[:, 7] = logits[:, 9] = logits[:, 4] = 1.0          # a three-way tie in every row
    logits[:, 2] = 1.0                                        # ... with EOS among it: EOS (id 2) ranks first
    state = torch.zeros(R, 4, dtype=torch.int32)
    state[:, 3] = -1
    score = torch.full((R,), float("-inf"))
    for b in range(B):
        for j in range(min(W, 2)):                            # two identical live parents per utterance
            state[b * W + j] = torch.tensor([1, 2, 1, j])
            score[b * W + j] = -1.5
    idx = torch.arange(R, dtype=torch.int32).remainder(W).view(R, 1).repeat(1, t + 1)
    recs = _recs(V)
    nbest = 2
    # the kernel's own fp32 final score of the EOS hypothesis, so that the pooled entry below ties with it exactly
    rc, d = run_beam_step(logits, recs, W, t, t + 7, nbest, 0.0, score, state, idx, [[], []])
    assert rc == 0, L.last_error()
    fs = float(d["pool_final"][0, 0])
    rc, d = run_beam_step(logits, recs, W, t, t + 7, nbest, 0.0, score, state, idx, [[(fs, fs, 99)], []])
    assert rc == 0, L.last_error()
    ht, hp = d["hist_tok"].cpu()[t], d["hist_par"].cpu()[t]
    want_tok = {2: [2, 4], 3: [2, 4, 7], 8: [2, 4, 7, 9, 2, 4, 7, 9]}[W]     # (score desc, parent, rank)
    want_par = {2: [0, 0], 3: [0, 0, 0], 8: [0, 0, 0, 0, 1, 1, 1, 1]}[W]
    for b in range(B):
        assert ht[b * W:(b + 1) * W].tolist() == want_tok and hp[b * W:(b + 1) * W].tolist() == want_par, (b, ht.tolist())
    pr, pn = d["pool_ref"].cpu(), d["pool_n"].cpu()
    assert pn.tolist() == [2, 2 if W == 8 else 1]
    assert pr[0].tolist() == [99, (t * W) << 1]               # equal final score: the pooled entry stays first
    if W == 8:
        assert pr[1].tolist() == [(t * W) << 1, (t * W + 4) << 1]   # equal: parent 0's EOS before parent 1's
    assert torch.equal(d["pool_final"].cpu()[0], torch.tensor([fs, fs]))


@pytest.mark.parametrize("case", ["W0", "W33", "Wgt V", "nbest0", "nbest33", "t>=steps", "stride", "null", "alias"])
def test_beam_step_rejections(case):
    W, V, nbest, t, steps, stride = 4, 33, 2, 3, 10, 11
    if case == "W0": W = 0
    if case == "W33": W = 33
    if case == "Wgt V": V = 3
    if case == "nbest0": nbest = 0
    if case == "nbest33": nbest = 33
    if case == "t>=steps": t = 10
    if case == "stride": stride = t + 1
    Wa = max(W, 1)
    R = 2 * Wa
    bufs = [torch.full((R, max(V, 1)), float("nan"), device=DEV), torch.zeros(max(V, 1), device=DEV, dtype=torch.int32),
            torch.full((R,), float("nan"), device=DEV), _i32(R, 4), torch.full((R,), -1, device=DEV, dtype=torch.long),
            _i32(R, 12), _i32(R, 12), _i32(10, R), _i32(10, R), torch.full((2, 33), float("nan"), device=DEV),
            torch.full((2, 33), float("nan"), device=DEV), _i32(2, 33), _i32(2), _i32(1)]
    before = [b.clone() for b in bufs]
    P = [L.ptr(b) for b in bufs]
    if case == "null":
        P[0] = None
    nxt = P[5] if case == "alias" else P[6]
    rc = _lib().b200asr_beam_step(P[0], P[1], 2, W, V, t, 20, steps, nbest, 0.1, P[2], P[3], P[4], P[5], nxt, stride, P[7], P[8],
                                  P[9], P[10], P[11], P[12], P[13], None)
    torch.cuda.synchronize()
    assert rc == (-5 if case in ("null", "alias") else -1), (case, rc)
    msg = L.last_error()
    assert msg.startswith("beam_step:"), msg
    if case.startswith("W"):
        assert "beam width" in msg
    if case.startswith("nbest"):
        assert "nbest" in msg
    for a, b in zip(bufs, before):
        assert torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def test_beam_step_index_table_follows_reordering():
    """Three steps of a W = 3 beam with scripted logits: after each step every survivor's index row is its parent's row
    plus its own slot, so a history reordered twice still names the slots that hold its positions."""
    W, V, B = 3, 33, 1
    recs = _recs(V)
    steps = 6
    d = None
    idx = torch.zeros(W, 1, dtype=torch.int32)
    idx[:, 0] = torch.arange(W, dtype=torch.int32)
    state = torch.tensor([[1, 0, 0, -1], [0, 0, 0, -1], [0, 0, 0, -1]], dtype=torch.int32)
    score = torch.tensor([0.0, float("-inf"), float("-inf")])
    g = torch.Generator().manual_seed(5)
    for t in range(3):
        logits = torch.randn(W, V, generator=g) * 2
        logits[:, 2] = -20.0
        exp = ref_beam_step(logits, recs, W, t, 50, 1, 0.1, score, state, idx, [[]])
        rc, d = run_beam_step(logits, recs, W, t, 50, 1, 0.1, score, state, idx, [[]], steps=steps)
        assert rc == 0, L.last_error()
        check_beam_step(exp, d, W, t, 1)
        state, score = d["state"].cpu(), d["score"].cpu()
        idx = d["idx_nxt"].cpu()[:, :t + 2]


# ------------------------------------------------------------------------------------------ beam_self_attn
@pytest.mark.parametrize("dk", [16, 32, 64, 128])
@pytest.mark.parametrize("dv", [16, 32, 64, 128])
def test_beam_self_attn_matches_float64(dk, dv):
    B, W, H = 2, 3, 2
    R = B * W
    g = torch.Generator().manual_seed(dk * 7 + dv)
    worst = 0.0
    for t in (1, 2, 31, 32, 33, 199, 300):
        S = t + 1
        kc = torch.randn(S, R, H * dk, generator=g)
        vc = torch.randn(S, R, H * dv, generator=g)
        q = torch.randn(R, H * dk, generator=g)
        for mode in ("random", "one-slot"):
            idx = torch.randint(0, W, (R, S + 3), generator=g, dtype=torch.int32) if mode == "random" \
                else torch.full((R, S + 3), 1, dtype=torch.int32)
            out = torch.full((R, H * dv), float("nan"), device=DEV)
            qd, kd, vd, idd = q.to(DEV), kc.to(DEV), vc.to(DEV), idx.to(DEV)
            rc = _lib().b200asr_beam_self_attn(L.ptr(qd), L.ptr(kd), L.ptr(vd), L.ptr(idd), L.ptr(out), R, H, W, dk, dv, t, S + 3,
                                               0.3, None)
            assert rc == 0, L.last_error()
            ref = torch.empty(R, H * dv, dtype=torch.float64)
            for r in range(R):
                rows = (r - r % W) + idx[r, :S].long()
                K = kc.double()[torch.arange(S), rows].view(S, H, dk)
                Vv = vc.double()[torch.arange(S), rows].view(S, H, dv)
                qq = q.double()[r].view(H, dk)
                p = torch.softmax(torch.einsum("hd,shd->hs", qq, K) * 0.3, dim=1)
                ref[r] = torch.einsum("hs,shd->hd", p, Vv).reshape(-1)
            e = float((out.cpu().double() - ref).abs().max() / ref.abs().max())
            worst = max(worst, e)
            assert e < ATTN_TOL, (t, mode, e)
    print(f"beam_self_attn dk={dk} dv={dv}: max rel err {worst:.2e}")


def test_beam_self_attn_rejections():
    x = torch.zeros(64, device=DEV)
    i = torch.zeros(64, device=DEV, dtype=torch.int32)
    for dk, dv, t, stride in [(8, 32, 3, 8), (32, 48, 3, 8), (32, 32, 8, 8), (32, 32, 8192, 9000)]:
        out = torch.full((64,), float("nan"), device=DEV)
        rc = _lib().b200asr_beam_self_attn(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(i), L.ptr(out), 2, 1, 1, dk, dv, t, stride, 1.0, None)
        assert rc == -1 and L.last_error().startswith("beam_self_attn:") and out.isnan().all()


# ------------------------------------------------------------------------------------------ decoder level
@pytest.fixture(scope="module")
def golden():
    cfg, id2label, cases = load_beam_golden()
    for c in cases:       # the float64 oracle's decision margins
        P = {k: v.double() for k, v in c["P"].items()}
        c["oracle"] = BO.beam_search(P, cfg, c["enc"].double(), c["W"], c["nbest"], c["c_weight"], id2label)
    return cfg, id2label, cases


def _decoder(cfg, P, id2label):
    from tests.gpu_util import cuda_model
    full = dict(O.init_params(cfg, seed=1))
    full.update(P)
    model = cuda_model(cfg, full, train=True)           # beam_decode must switch dropout off and restore the mode
    model.decoder.id2label = id2label
    return model.decoder


def test_beam_decode_and_beam_search_match_reference_fixture(golden):
    cfg, id2label, cases = golden
    n_ok = n_all = 0
    worst = worst_abs = 0.0
    for ci, c in enumerate(cases):
        dec = _decoder(cfg, c["P"], id2label)
        enc = c["enc"].to(DEV)
        ids, lengths, score, final = dec.beam_decode(enc, c["W"], nbest=c["nbest"], c_weight=c["c_weight"])
        assert dec.training
        ys, strs = dec.beam_search(enc, beam_width=c["W"], nbest=c["nbest"], c_weight=c["c_weight"])
        ids, lengths, score, final = ids.cpu(), lengths.cpu(), score.cpu(), final.cpu()
        k = 0
        for b in range(enc.shape[0]):
            n_all += 1
            o = c["oracle"][b]
            mine = [ids[b, i, :int(n)].tolist() for i, n in enumerate(lengths[b]) if int(n) > 0]
            assert all((ids[b, i, int(n):] == -1).all() for i, n in enumerate(lengths[b]))
            ref = golden_yseqs(c, b)
            for y in mine:      # the flat beam_search lists hold the same hypotheses in the same order
                assert ys[k] == y and strs[k] == "".join(id2label[t] for t in y[1:])
                k += 1
            margin = min(o["step_margins"] + [o["pool_margin"]])
            print(f"case {ci} utterance {b}: margin {margin:.2e}, same yseqs as the reference: {mine == ref}")
            if margin <= MARGIN_BAR:
                continue
            assert mine == ref, (ci, b)
            m = len(ref)
            if m:
                e = float(((score[b, :m].double() - c["score"][b, :m].double()).abs() / c["score"][b, :m].double().abs()).max())
                e = max(e, float(((final[b, :m].double() - c["final"][b, :m].double()).abs() / c["final"][b, :m].double().abs()).max()))
                worst = max(worst, e)
                worst_abs = max(worst_abs, float((score[b, :m].double() - c["score"][b, :m].double()).abs().max()))
                assert e < DECODE_RTOL, (ci, b, e)
            assert torch.isnan(score[b, m:]).all() and (lengths[b, m:] == 0).all()
            n_ok += 1
        assert k == len(ys)
    print(f"beam_decode: {n_ok}/{n_all} utterances compared, max rel score err {worst:.2e}, max abs {worst_abs:.2e}")
    assert n_ok * 4 >= n_all * 3, (n_ok, n_all)


def test_beam_width_one_is_greedy_decoding(golden):
    cfg, id2label, cases = golden
    c = next(c for c in cases if c["W"] == 1)
    dec = _decoder(cfg, c["P"], id2label)
    enc = c["enc"].to(DEV)
    Te = enc.shape[1]
    ids, lengths, _, _ = dec.beam_decode(enc, 1, nbest=1, c_weight=0.1)
    greedy = dec.greedy_decode_cached(enc, steps=Te).cpu()
    for b in range(enc.shape[0]):
        if min(c["oracle"][b]["step_margins"]) <= MARGIN_BAR:
            continue
        g = greedy[b].tolist()
        want = [1] + (g[:g.index(2) + 1] if 2 in g[:Te - 1] else g[:Te] + [2])
        assert ids[b, 0, :int(lengths[b, 0])].tolist() == want, b


def test_beam_decode_is_reproducible(golden):
    cfg, id2label, cases = golden
    c = next(c for c in cases if c["W"] == 8)
    dec = _decoder(cfg, c["P"], id2label)
    enc = c["enc"].to(DEV)
    a = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=4, c_weight=0.1)]
    b = [x.cpu() for x in dec.beam_decode(enc, 8, nbest=4, c_weight=0.1)]
    for x, y in zip(a, b):
        assert torch.equal(x.isnan(), y.isnan()) and torch.equal(x.nan_to_num(), y.nan_to_num())


def test_beam_decode_rejects_a_short_positional_table(golden):
    cfg, id2label, cases = golden
    dec = _decoder(cfg, cases[0]["P"], id2label)
    dec.trg_max_length = 20
    with pytest.raises(ValueError, match="trg_max_length"):
        dec.beam_decode(cases[0]["enc"].to(DEV), 2)
    with pytest.raises(ValueError):
        dec.beam_search(cases[0]["enc"].to(DEV), beam_width=2)


# ------------------------------------------------------------------------------------------ the reference's evaluate
@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_evaluate_with_beam_search_installed_matches_uninstalled():
    flags = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
             "--dim-inner", "128", "--feat_extractor", "", "--tgt-max-len", "301", "--dropout", "0.0", "--cuda"]
    ns = ref_shim.load(flags, q12_shim=True)
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
    model = model.cuda().eval()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    eos_row = model.decoder.output_linear.weight[2].detach().clone()
    batches = []
    for T, eos_scale in ((24, -1.0), (310, 0.0)):        # the second batch ends no hypothesis: evaluate falls back to greedy
        src = torch.randn(2, 1, 161, T, generator=g)
        lens = torch.full((2,), T, dtype=torch.int32)
        tgt = torch.randint(3, V, (2, 6), generator=g)
        batches.append((src.cuda(), lens.cuda(), tgt.cuda(), eos_scale))
    results = {}
    try:
        for installed in (False, True):
            if installed:
                b200asr.install()
            out = []
            for src, lens, tgt, s in batches:
                with torch.no_grad():
                    model.decoder.output_linear.weight[2] = eos_row * s
                    _, strs, _ = model.evaluate(src, lens, tgt, beam_search=True, beam_width=4, beam_nbest=1, c_weight=0.1)
                    enc, _ = model.encoder(src.view(2, 161, -1).transpose(1, 2).contiguous(), lens)
                    hyps = model.decoder.beam_search(enc, beam_width=4, nbest=1, c_weight=0.1)[1]
                out.append((list(strs), len(hyps)))
            results[installed] = out
    finally:
        b200asr.uninstall()
    assert results[True] == results[False], results
    assert results[True][0][1] == 2 and results[True][1][1] < 2        # the second batch took the fallback to greedy
