"""Restatements of the training loop's CER / WER counts (b200asr_edit_counts) for the tests.

  * kernel_counts: the kernel's definition (include/b200asr.h) over a LabelTable's arrays, in numpy;
  * reference_counts: the reference's string path (trainer/asr/trainer.py:60-79, 96-104 with utils/metrics.py's
    calculate_cer / calculate_wer) restated over an id2label dict;
  * levenshtein: the edit distance both use, a row-vectorised DP.
"""
import numpy as np

PAD, SOS, EOS = "¶", "§", "¤"      # utils/constant.py's PAD_CHAR, SOS_CHAR, EOS_CHAR


def levenshtein(a, b):
    """Edit distance of two sequences (str, list or 1-D array) by rows: t_j = min(up + 1, diag + cost), then the left
    neighbour's chain D[i][j] = min_k (t_k + j - k) as a running minimum."""
    a = np.asarray([ord(c) for c in a] if isinstance(a, str) else a, dtype=np.int64)
    b = np.asarray([ord(c) for c in b] if isinstance(b, str) else b, dtype=np.int64)
    m = len(b)
    j = np.arange(m + 1, dtype=np.int64)
    row = j.copy()
    for i in range(1, len(a) + 1):
        t = np.empty(m + 1, dtype=np.int64)
        t[0] = i
        t[1:] = np.minimum(row[1:] + 1, row[:-1] + (b != a[i - 1]))
        row = np.minimum.accumulate(t - j) + j
    return int(row[m])


def _row_ids(row, pad):
    out = []
    for x in row:
        if int(x) == pad:
            break
        out.append(int(x))
    return out


def kernel_counts(hyp, gold, table):
    """(per_utt [B, 4], totals [5]) as int64 arrays, from the table's off / length / code_points / flags / valid."""
    off, length = table.off.numpy(), table.length.numpy()
    cps, flags, valid = table.code_points.numpy(), table.flags.numpy(), table.valid.numpy()
    hyp, gold = np.asarray(hyp), np.asarray(gold)

    def expand(row):
        c, f, bad = [], [], -1
        for t, i in enumerate(_row_ids(row, table.pad_id)):
            if 0 <= i < table.V and valid[i]:
                c.extend(cps[off[i]:off[i] + length[i]])
                f.extend(flags[off[i]:off[i] + length[i]])
            elif bad < 0:
                bad = i
        return np.asarray(c, dtype=np.int64), np.asarray(f, dtype=np.int64), bad

    def words(c, f):
        out, cur = [], []
        for cp, fl in zip(c, f):
            if fl & 2:
                if cur:
                    out.append(tuple(cur))
                cur = []
            else:
                cur.append(int(cp))
        if cur:
            out.append(tuple(cur))
        return out

    B = gold.shape[0]
    per = np.zeros((B, 4), dtype=np.int64)
    bad_gold, bad_hyp = [], []
    for b in range(B):
        ch, fh, bh = expand(hyp[b])
        cg, fg, bg = expand(gold[b])
        bad_gold.append(bg)
        bad_hyp.append(bh)
        wh, wg = words(ch, fh), words(cg, fg)
        ids = {}
        per[b, 0] = levenshtein(ch[(fh & 1) == 0], cg[(fg & 1) == 0])
        per[b, 1] = levenshtein([ids.setdefault(w, len(ids)) for w in wh], [ids.setdefault(w, len(ids)) for w in wg])
        per[b, 2] = int(((fg & 1) == 0).sum())
        per[b, 3] = int((fg & 1).sum()) + 1
    first = next((x for x in bad_gold + bad_hyp if x >= 0), -1)
    return per, np.concatenate([per.sum(0), [first]]).astype(np.int64)


def reference_counts(hyp, gold, id2label, pad, sos=SOS, eos=EOS):
    """The reference's string path: (per_utt [B, 4], first missing id or -1).  Strings are joined up to the first PAD with
    id2label (a missing id raises KeyError there, gold rows first), SOS / EOS removed from the joined strings, then
    calculate_cer(h.replace(' ', ''), g.replace(' ', '')), calculate_wer(h, g) (split(), words mapped to chr), len(g without
    ' ') and len(g.split(" "))."""
    def join(row):
        s = ""
        for x in row:
            if int(x) == pad:
                break
            s = s + id2label[int(x)]
        return s
    try:
        strs_gold = [join(r) for r in np.asarray(gold)]
        strs_hyps = [join(r) for r in np.asarray(hyp)]
    except KeyError as e:
        return None, e.args[0]
    per = []
    for h, g in zip(strs_hyps, strs_gold):
        h = h.replace(sos, "").replace(eos, "")
        g = g.replace(sos, "").replace(eos, "")
        vocab = set(h.split() + g.split())
        w2c = dict(zip(vocab, range(len(vocab))))
        w1 = "".join(chr(w2c[w]) for w in h.split())
        w2 = "".join(chr(w2c[w]) for w in g.split())
        per.append([levenshtein(h.replace(" ", ""), g.replace(" ", "")), levenshtein(w1, w2), len(g.replace(" ", "")),
                    len(g.split(" "))])
    return np.asarray(per, dtype=np.int64).reshape(-1, 4), -1


def label_set(vocab=40, missing=()):
    """An id2label with the reference's specials (0 PAD, 1 SOS, 2 EOS) and labels that exercise every rule: single and
    multi-code-point labels, ' ' and other whitespace (tab, ideographic space, no-break space, \\x1c), SOS / EOS inside
    longer labels, CJK and astral code points, repeated labels."""
    base = [PAD, SOS, EOS, " ", "a", "b", "ab", "  ", "\t", "　", "\xa0", "\x1c", "x y", "a" + SOS, EOS + "b",
            SOS + " " + EOS, "一", "\U0001f600", "ba", "a", "b ", " a", "c", "d", "e　f", "cd", "\n", "dc"]
    labels = (base + [chr(0x4E00 + i) for i in range(vocab)])[:vocab]
    return {i: s for i, s in enumerate(labels) if i not in set(missing)}
