"""CPU checks of beam search: the float64 oracle (oracle/beam_oracle.py) reproduces the live reference's
Decoder.beam_search (tests/golden/beam.npz), and the per-token word-state rule the device search uses to count words
equals the reference's len(s.split()) of the joined labels."""
import math
import random

import pytest
import torch

from oracle import beam_oracle as BO
from tests.beam_util import golden_yseqs, load_beam_golden

import b200asr.modules as M


@pytest.fixture(scope="module")
def golden():
    return load_beam_golden()


def test_golden_fixture_covers_the_cases(golden):
    _, id2label, cases = golden
    assert sorted({c["W"] for c in cases}) == [1, 2, 4, 8] and {c["c_weight"] for c in cases} == {0.0, 0.1, 1.0}
    Te = [c["enc"].shape[1] for c in cases]
    ended_early = forced = none = 0
    for c, te in zip(cases, Te):
        for b in range(c["enc"].shape[0]):
            n = c["lengths"][b]
            none += int(n[0]) == 0
            forced += any(int(x) == te + 2 for x in n)
            ended_early += any(0 < int(x) < te + 1 for x in n)
    assert ended_early and forced and none
    assert any(c["enc"].shape[1] > 300 for c in cases)
    assert {" ", "ab", "c d"} <= set(id2label.values())


@pytest.mark.parametrize("ci", range(6))
def test_oracle_beam_search_matches_reference_fixture(golden, ci):
    cfg, id2label, cases = golden
    c = cases[ci]
    P = {k: v.double() for k, v in c["P"].items()}
    res = BO.beam_search(P, cfg, c["enc"].double(), c["W"], c["nbest"], c["c_weight"], id2label)
    for b, r in enumerate(res):
        assert r["yseqs"] == golden_yseqs(c, b), (ci, b)
        k = len(r["yseqs"])
        if k:
            assert torch.allclose(torch.tensor(r["scores"], dtype=torch.float64), c["score"][b, :k].double(), rtol=1e-5, atol=0), (ci, b)
            assert torch.allclose(torch.tensor(r["finals"], dtype=torch.float64), c["final"][b, :k].double(), rtol=1e-5, atol=0), (ci, b)
        assert torch.isnan(c["score"][b, k:]).all() and (c["lengths"][b, k:] == 0).all()


def _words_by_rule(recs, seq):
    words, tail = 0, 0
    for v in seq:
        r = recs[v]
        w, head, t, empty = r >> 3, (r >> 2) & 1, (r >> 1) & 1, r & 1
        words += w - (tail & head)
        if not empty:
            tail = t
    return words


@pytest.mark.parametrize("seed", range(4))
def test_word_state_rule_equals_split_of_joined_labels(seed):
    rnd = random.Random(seed)
    specials = [BO.PAD_CHAR, BO.SOS_CHAR, BO.EOS_CHAR]
    pieces = [" ", "  ", "\t", "a", "bc", "d e", " f", "g ", " h i ", "", "x" + BO.EOS_CHAR, BO.PAD_CHAR + " ", "　", "中"]
    for _ in range(50):
        V = rnd.randint(4, 24)
        id2label = {i: s for i, s in enumerate(specials)}
        for v in range(3, V):
            id2label[v] = "".join(rnd.choice(pieces + specials) for _ in range(rnd.randint(1, 3)))
        recs = M.word_records(id2label, V)
        for _ in range(40):
            seq = [1] + [rnd.randrange(V) for _ in range(rnd.randint(0, 12))]
            assert _words_by_rule(recs, seq) == BO.num_words(seq, id2label), (id2label, seq)


def test_word_records_of_special_and_spaced_labels():
    recs = M.word_records({0: BO.PAD_CHAR, 1: BO.SOS_CHAR, 2: BO.EOS_CHAR, 3: " ", 4: "ab", 5: "c d", 6: " e"}, 8)
    assert recs[:3] == [1, 1, 1]                 # empty after the specials are removed
    assert recs[3] == 0                          # no word, spaces at both ends
    assert recs[4] == 8 + 4 + 2 and recs[5] == 16 + 4 + 2 and recs[6] == 8 + 2
    assert recs[7] == 1                          # a token the label map does not cover counts as empty
    assert math.isclose(BO.num_words([1, 4, 3, 5, 6, 2], {0: "", 1: "§", 2: "¤", 3: " ", 4: "ab", 5: "c d", 6: " e"}), 4)
