"""CPU checks of beam search with LM rescoring: the float64 oracle (oracle/lm_oracle.py) reproduces the live reference's
lm_score / num_words / OOV count of every ended hypothesis and its n-best (tests/golden/beam_lm.npz), and the host
segmentation of b200asr (modules.lm_string / lm_word_ids) gives the strings the reference's calculate_lm_score scores."""
import random

import pytest
import torch

import b200asr.modules as M
from oracle import lm_oracle as LO
from oracle import ref_shim
from tests.beam_lm_util import load_beam_lm_golden


@pytest.fixture(scope="module")
def golden():
    return load_beam_lm_golden()


def test_fixture_covers_the_cases(golden):
    _, id2label, w2i, lms, cases = golden
    assert sorted({c["W"] for c in cases}) == [1, 4, 8]
    assert {c["lm_weight"] for c in cases} == {0.0, 0.1, 5.0} and {c["c_weight"] for c in cases} == {0.0, 1.0}
    assert [(m["nlayers"], m["nhid"], m["tie"]) for m in lms] == [(2, 50, False), (1, 40, True)]
    ended = [h for c in cases for h in c["ended"]]
    assert any(h["lm"] == -999 for h in ended) and any(h["oov"] > 0 for h in ended)
    assert any(len(h["yseq"]) == c["enc"].shape[1] + 2 for c in cases for h in c["ended"])        # forced endings
    assert {" ", "ab", "c d"} <= set(id2label.values()) and any(M._has_letter_lo(s) for s in id2label.values())


@pytest.mark.parametrize("ci", range(6))
def test_oracle_reproduces_reference_lm_scores_and_nbest(golden, ci):
    _, id2label, w2i, lms, cases = golden
    c = cases[ci]
    lm = lms[c["lm"]]
    P = {k: v.double() for k, v in lm["P"].items()}
    finals = {}
    for j, h in enumerate(c["ended"]):
        lm_s, nw, oov, s = LO.lm_score(h["yseq"], id2label, w2i, P, lm["nlayers"])
        assert s == h["string"] and nw == h["nw"] and oov == h["oov"], (ci, j)
        want = h["lm"] if h["lm"] == -999 else h["lm"] - 2 * h["oov"]
        assert abs(lm_s - want) <= 1e-5 * max(1.0, abs(want)), (ci, j, lm_s, want)
        finals.setdefault(h["utt"], []).append((j, LO.final_score(h["score"], lm_s, nw, c["lm_weight"], c["c_weight"])))
    for b, row in enumerate(c["nbest_idx"]):
        js = [j for j, _ in finals.get(b, [])]
        got = [js[k] for k in LO.rank([f for _, f in finals.get(b, [])], c["nbest"])]
        assert got == [int(j) for j in row if j >= 0], (ci, b)


def test_host_segmentation_matches_fixture_strings(golden):
    _, id2label, w2i, _, cases = golden
    for c in cases:
        for h in c["ended"]:
            s = M.lm_string(h["yseq"], id2label)
            assert s == h["string"]
            if s:
                ids, oov = M.lm_word_ids(s, w2i)
                assert oov == h["oov"] and len(ids) == h["nw"]


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_host_segmentation_matches_reference_on_random_label_sequences():
    import importlib
    ref_shim.load([])
    lstm_utils = importlib.import_module("utils.lstm_utils")
    rnd = random.Random(7)
    specials = [M.PAD_CHAR, M.SOS_CHAR, M.EOS_CHAR]
    pieces = [" ", "  ", "a", "bc", "d e", " f", "g ", "中", "文 ", " 字", "中a", "a中", "b 中", "ア", "한", "é", "　"]
    seen = set()

    class Recorder:
        def evaluate(self, s):
            seen.add(s)
            self.last = s
            return torch.tensor(1.0), 0

    rec = Recorder()
    for trial in range(4000):
        V = rnd.randint(4, 16)
        id2label = dict(enumerate(specials))
        for v in range(3, V):
            id2label[v] = "".join(rnd.choice(pieces) for _ in range(rnd.randint(1, 2)))
        yseq = [1] + [rnd.randrange(V) for _ in range(rnd.randint(0, 10))] + [2]
        rec.last = ""
        score = lstm_utils.calculate_lm_score(torch.tensor([yseq]), rec, id2label)
        want = rec.last if score[0] != -999 else ""
        assert M.lm_string(yseq, id2label) == want, (yseq, id2label)
        assert LO.lm_string(yseq, id2label) == want, (yseq, id2label)
    assert len(seen) > 1000


def test_rescoring_ranks_ties_in_insertion_order():
    import numpy as np
    f = [np.float32(x) for x in (1.0, 2.0, 1.0, 2.0, -999.0, 2.0)]
    assert M.rank_nbest(f, 4) == [1, 3, 5, 0] and M.rank_nbest(f, 10) == [1, 3, 5, 0, 2, 4]
    assert LO.rank([float(x) for x in f], 4) == [1, 3, 5, 0]


def test_lm_final_score_follows_the_reference_fp32_order():
    import numpy as np
    lm, nw, fin = M.lm_final_score(np.float32(-3.25), np.float32(7.5), 3, 1, 0.1, 1.0)
    total = np.float32(3) * (np.float32(7.5) / np.float32(3))
    want_lm = (np.float32(-total) / np.float32(3) + np.float32(1)) - np.float32(2)
    assert nw == 4 and lm == float(want_lm)
    assert fin == np.float32(np.float32(-3.25) + np.float32(0.1) * want_lm) + np.float32(2.0)
    assert M.lm_final_score(np.float32(-1.5), 0.0, None, 0, 0.1, 1.0)[:2] == (-999.0, 0)
