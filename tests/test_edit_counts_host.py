"""CPU checks of the training loop's CER / WER counts: the LabelTable built for b200asr_edit_counts, and the kernel's definition
(tests/edit_util.kernel_counts) against the reference's string path (reference_counts) over random id sequences.  The test's
Levenshtein is pinned against exhaustive enumeration of edit scripts on tiny strings."""
import itertools

import numpy as np
import pytest

import b200asr
from tests.edit_util import EOS, PAD, SOS, kernel_counts, label_set, levenshtein, reference_counts


def _table(id2label):
    return b200asr.LabelTable(id2label, 0, (SOS, EOS))


def _label(t, i):
    o, n = int(t.off[i]), int(t.length[i])
    return t.code_points[o:o + n].tolist(), t.flags[o:o + n].tolist()


def test_label_table_contents():
    t = _table({0: PAD, 1: SOS, 2: EOS, 3: "a", 4: "xyz", 5: "a" + SOS + "b" + EOS, 7: "\U0001f600 ", 8: ""})
    assert t.V == 9 and t.pad_id == 0 and t.max_label_len == 3
    assert t.valid.tolist() == [1, 1, 1, 1, 1, 1, 0, 1, 1]            # id 6 is missing
    assert _label(t, 0) == ([ord(PAD)], [0])
    assert _label(t, 1) == ([], []) and _label(t, 2) == ([], [])       # SOS / EOS dropped
    assert _label(t, 3) == ([ord("a")], [0])
    assert _label(t, 4) == ([ord(c) for c in "xyz"], [0, 0, 0])
    assert _label(t, 5) == ([ord("a"), ord("b")], [0, 0])              # § / ¤ inside a longer label
    assert _label(t, 6) == ([], [])
    assert _label(t, 7) == ([0x1F600, 32], [0, 3])
    assert _label(t, 8) == ([], [])
    assert t.off.tolist() == sorted(t.off.tolist())


@pytest.mark.parametrize("ch,flag", [(" ", 3), ("\t", 2), ("　", 2), ("\xa0", 2), ("\x1c", 2), ("\n", 2), ("_", 0),
                                     ("​", 0)])
def test_label_table_whitespace_flags(ch, flag):
    t = _table({0: PAD, 1: "x" + ch})
    assert _label(t, 1) == ([ord("x"), ord(ch)], [0, flag])
    assert bool(flag & 2) == ch.isspace() == (len(("a" + ch + "b").split()) == 2)


@pytest.mark.parametrize("bad,exc", [({0: PAD, 1: b"a"}, TypeError), ({0: PAD, 1: None}, TypeError), ({0: PAD, 1: 5}, TypeError),
                                     ([PAD, "a"], TypeError), ({}, TypeError), ({-1: "a"}, ValueError),
                                     ({"1": "a"}, ValueError), ({True: "a"}, ValueError)])
def test_label_table_rejects_bad_id2label(bad, exc):
    with pytest.raises(exc):
        b200asr.LabelTable(bad, 0, (SOS, EOS))


@pytest.mark.parametrize("drop", [("<s>",), ("",), (SOS, "ab"), (1,)])
def test_label_table_rejects_multi_code_point_drop_chars(drop):
    with pytest.raises(ValueError):
        b200asr.LabelTable({0: PAD, 1: "a"}, 0, drop)


def _exhaustive(a, b, alphabet):
    """Breadth-first search over single insertions, deletions and substitutions from a until b is reached."""
    seen, frontier, d = {a}, {a}, 0
    while b not in frontier:
        nxt = set()
        for s in frontier:
            for i in range(len(s) + 1):
                for c in alphabet:
                    nxt.add(s[:i] + c + s[i:])
                if i < len(s):
                    nxt.add(s[:i] + s[i + 1:])
                    for c in alphabet:
                        nxt.add(s[:i] + c + s[i + 1:])
        frontier = nxt - seen
        seen |= nxt
        d += 1
    return d


def test_levenshtein_matches_exhaustive_enumeration():
    strings = ["".join(p) for n in range(4) for p in itertools.product("ab", repeat=n)]
    for a in strings:
        for b in strings:
            assert levenshtein(a, b) == _exhaustive(a, b, "ab"), (a, b)
    rng = np.random.default_rng(0)
    for _ in range(40):
        a = "".join(rng.choice(list("abc"), rng.integers(0, 5)))
        b = "".join(rng.choice(list("abc"), rng.integers(0, 5)))
        assert levenshtein(a, b) == _exhaustive(a, b, "abc"), (a, b)
    assert levenshtein([5, 6, 7], [7, 6, 5]) == 2 and levenshtein([], [1, 2]) == 2


def _random_ids(rng, B, T, V, pad_frac=0.5, low=0):
    ids = rng.integers(low, V, size=(B, T))
    for b in range(B):
        if rng.random() < pad_frac:
            ids[b, rng.integers(0, T + 1):] = 0
    return ids


@pytest.mark.parametrize("seed", range(6))
def test_kernel_definition_matches_reference_string_path(seed):
    rng = np.random.default_rng(seed)
    id2label = label_set(40)
    table = _table(id2label)
    for B, T_h, T_g in [(1, 1, 3), (3, 17, 9), (8, 40, 33), (2, 0, 5)]:
        hyp = _random_ids(rng, B, T_h, 40, low=1)
        gold = _random_ids(rng, B, T_g, 40, low=1)
        per, totals = kernel_counts(hyp, gold, table)
        ref, first = reference_counts(hyp, gold, id2label, 0)
        assert first == -1
        np.testing.assert_array_equal(per, ref)
        assert totals[:4].tolist() == ref.sum(0).tolist() and totals[4] == -1


def test_kernel_definition_edge_strings():
    id2label = label_set(40)
    table = _table(id2label)
    sp, tab, word_a, word_b, join_sos = 3, 8, 4, 5, 15          # " ", "\t", "a", "b", SOS + " " + EOS
    cases = [
        ([[0]], [[0]]),                                          # both empty
        ([[sp, sp, sp]], [[sp, 0, word_a]]),                     # all spaces / PAD first... then a
        ([[sp, word_a, sp, sp, word_b, sp]], [[word_a, word_b]]),  # leading, repeated and trailing whitespace
        ([[word_a, 13, word_b]], [[word_a, 14, word_b]]),        # a + "a§" + b: § joins words
        ([[word_a, tab, word_b]], [[word_a, sp, word_b]]),       # tab splits words but is kept for the CER
        ([[word_a, join_sos, word_b]], [[word_a, word_b]]),
        ([[6, 6, 6]], [[6, 6, 6]]),                              # identical
    ]
    for hyp, gold in cases:
        per, _ = kernel_counts(np.array(hyp), np.array(gold), table)
        ref, _ = reference_counts(np.array(hyp), np.array(gold), id2label, 0)
        np.testing.assert_array_equal(per, ref)


def test_kernel_definition_first_missing_id():
    rng = np.random.default_rng(7)
    id2label = label_set(40, missing=(9, 21, 33))
    table = _table(id2label)
    ok = np.array(sorted(set(id2label) - {0}))
    hits = 0
    for _ in range(60):
        hyp, gold = ok[rng.integers(0, len(ok), (4, 12))], ok[rng.integers(0, len(ok), (4, 10))]
        for ids in (hyp, gold):
            ids[rng.integers(0, 4), rng.integers(0, ids.shape[1]):] = 0
            if rng.random() < 0.4:                               # 40, 41 are beyond V; PAD may hide them
                ids[rng.integers(0, 4), rng.integers(0, ids.shape[1])] = rng.choice([9, 21, 33, 40, 41])
        per, totals = kernel_counts(hyp, gold, table)
        ref, first = reference_counts(hyp, gold, id2label, 0)
        assert totals[4] == first
        hits += first != -1
        if first == -1:
            np.testing.assert_array_equal(per, ref)
    assert 10 < hits < 60
