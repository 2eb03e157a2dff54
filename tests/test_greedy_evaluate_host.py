"""Host side of the installed greedy decode and Transformer.evaluate (no GPU needed):

  * modules.greedy_strings against an independent restatement of Decoder.greedy_search's string building
    (models/asr/transformer.py:376, :385-393): per-step label lists, np.transpose, cut at the first entry equal to EOS_CHAR.
    Multi-character labels, a non-EOS label equal to EOS_CHAR, an utterance that emits EOS at step 0 and one that never does.
  * b200asr_decode_attn_ws_bytes: the key split depends on (R, H, Tk) only and sizes the partials; invalid calls are rejected
    before anything reaches the device.
  * install() binds Decoder.greedy_search and Transformer.evaluate on the reference's classes and uninstall() restores them.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import b200asr
import b200asr.modules as M
from oracle import ref_shim

L = b200asr._lib
STEPS = 300


def restated_strings(ids_full, id2label):
    """What the reference returns for token ids [B][300] (every step decoded, no device cut)."""
    B = len(ids_full)
    per_step = [[M.EOS_CHAR if ids_full[b][t] == M.EOS_TOKEN else id2label[ids_full[b][t]] for b in range(B)]
                for t in range(len(ids_full[0]))]
    out = []
    for row in np.transpose(per_step):
        s = ""
        for e in row:
            if e == M.EOS_CHAR:
                break
            s += e
        out.append(s)
    return out


def device_cut(ids_full):
    """greedy_decode_cached(stop_at_eos=True)'s ids: -1 from an utterance's first EOS on."""
    out = []
    for row in ids_full:
        r = list(row)
        if M.EOS_TOKEN in r:
            k = r.index(M.EOS_TOKEN)
            r[k + 1:] = [-1] * (len(r) - k - 1)
        out.append(r)
    return out


def test_greedy_strings_match_the_reference_string_building():
    V = 50
    id2label = {0: M.PAD_CHAR, 1: M.SOS_CHAR, 2: "<eos-label-unused>"}
    for i in range(3, V):
        id2label[i] = ["ab", " ", "x y", "中文", "q", "it's", "a\x00"][i % 7] + str(i)
    id2label[7] = M.EOS_CHAR          # a non-EOS token whose label is EOS_CHAR: the reference's cut is on the string
    id2label[8] = "multi char label"
    g = np.random.default_rng(0)
    ids = g.integers(3, V, size=(7, STEPS))
    ids[ids == 7] = 9
    ids[0, 0] = M.EOS_TOKEN           # EOS at step 0: ""
    ids[2, 40] = M.EOS_TOKEN          # EOS later, more tokens after it
    ids[2, 60] = M.EOS_TOKEN
    ids[3, 17] = 7                    # label == EOS_CHAR before any EOS
    ids[3, 90] = M.EOS_TOKEN
    ids[4, 5] = 7                     # label == EOS_CHAR and no EOS at all
    ids[5, 299] = M.EOS_TOKEN         # EOS at the last step
    # rows 1 and 6: no EOS, all 300 labels
    ids = ids.tolist()
    want = restated_strings(ids, id2label)
    got = M.greedy_strings(device_cut(ids), id2label)
    assert got == want
    assert want[0] == "" and want[4] == "".join(id2label[i] for i in ids[4][:5])
    assert want[1] == "".join(id2label[i] for i in ids[1]) and len(want[1]) > STEPS
    assert M.greedy_strings(ids, id2label) == want          # the full ids give the same strings


def test_greedy_strings_convert_labels_as_numpy_does():
    """The reference joins numpy string scalars: non-string labels become their str, trailing NULs are dropped."""
    id2label = {i: i * 10 for i in range(3, 12)}
    id2label[2] = "unused"
    ids = [[3, 4, 11, 2, 5], [5, 6, 7, 8, 9]]
    assert M.greedy_strings(device_cut(ids), id2label) == restated_strings(ids, id2label) == ["3040110", "5060708090"]


# ------------------------------------------------------------------------------------------ decode_attn host-side contract
def _chunks(R, H, Tk):
    """The key split of csrc/decode.cu restated: keys per chunk = ceil(Tk / max(1, 1024 // (R*H))) rounded up to 32, clamped
    to [64, 1024]."""
    want = 1 if R * H >= 1024 else 1024 // (R * H)
    kc = min(max(-(-(-(-Tk // want)) // 32) * 32, 64), 1024)
    return -(-Tk // kc)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    if not os.path.exists(L.LIB_PATH):
        __graft_entry__.build()
    return L.load()


def test_decode_attn_workspace_follows_the_key_split(lib):
    for R, H in ((1, 1), (3, 8), (32, 8), (129, 8), (4096, 16)):
        for Tk in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 500, 1000, 1023, 1024, 1025, 4097, 8192, 65536):
            for dv in (16, 128):
                nc = _chunks(R, H, Tk)
                want = 0 if nc == 1 else R * H * nc * (dv + 2) * 4
                assert lib.b200asr_decode_attn_ws_bytes(R, H, Tk, dv) == want, (R, H, Tk, dv)
    assert _chunks(32, 8, 200) == 4 and _chunks(32, 8, 16) == 1       # cfg2 decode: cross-attention split, self not
    for bad in ((0, 8, 10, 64), (1, 0, 10, 64), (1, 1, 0, 64), (1, 1, 65537, 64)):
        assert lib.b200asr_decode_attn_ws_bytes(*bad) == 0


def test_decode_attn_rejects_before_launching(lib):
    """Every rejection returns its code with nothing launched.  The pointers are never dereferenced on these paths."""
    p = 1 << 20                       # a 16-byte aligned fake address
    base = dict(q=p, k=p, v=p, out=p, ws=p, R=2, H=2, dk=64, dv=64, Tk=300, krs=128, kks=256, vrs=128, vks=256)
    cases = [
        (dict(q=None), -5), (dict(k=None), -5), (dict(v=None), -5), (dict(out=None), -5),
        (dict(ws=None), -5),                                   # 300 keys at R*H = 4 are split: the workspace is needed
        (dict(dk=48), -1), (dict(dv=8), -1), (dict(dk=256), -1), (dict(dv=0), -1),
        (dict(R=0), -1), (dict(H=0), -1), (dict(Tk=0), -1), (dict(Tk=65537), -1), (dict(kks=-4), -1), (dict(vrs=-4), -1),
        (dict(k=p + 4), -2), (dict(v=p + 8), -2), (dict(krs=130), -2), (dict(kks=258), -2), (dict(vrs=2), -2),
        (dict(vks=6), -2),
    ]
    n0 = lib.b200asr_launch_count()
    for change, code in cases:
        a = dict(base, **change)
        rc = lib.b200asr_decode_attn(a["q"], a["k"], a["v"], a["out"], a["ws"], a["R"], a["H"], a["dk"], a["dv"], a["Tk"],
                                     a["krs"], a["kks"], a["vrs"], a["vks"], 0.125, None)
        assert rc == code, (change, rc, L.last_error())
        assert "decode_attn" in L.last_error()
    assert lib.b200asr_launch_count() == n0


# ------------------------------------------------------------------------------------------ install() binding
@pytest.mark.skipif(ref_shim.reference_root() is None, reason="reference checkout not staged (oracle/make_ref.py)")
def test_install_binds_greedy_search_and_evaluate():
    """Runs in a subprocess because the reference parses flags at import (utils/constant.py:99)."""
    REF = ref_shim.reference_root()
    code = r'''
import sys, types
sys.path.insert(0, %r); sys.path.insert(0, %r)
sys.modules["Levenshtein"] = types.ModuleType("Levenshtein")
sys.argv = ["x", "--num-layers", "1", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
            "--dim-inner", "64", "--feat_extractor", "", "--tgt-max-len", "8"]
from utils import constant
import models.asr.transformer as tr
import importlib
import b200asr
modules = importlib.import_module(b200asr.__name__ + ".modules")
install = importlib.import_module(b200asr.__name__ + ".install")
greedy, evaluate = tr.Decoder.greedy_search, tr.Transformer.evaluate
b200asr.install()
assert tr.Decoder.greedy_search is modules.greedy_search and tr.Transformer.evaluate is modules.transformer_evaluate
assert install.original(tr.Decoder, "greedy_search") is greedy and install.original(tr.Transformer, "evaluate") is evaluate
b200asr.uninstall()
assert tr.Decoder.greedy_search is greedy and tr.Transformer.evaluate is evaluate
assert install.original(tr.Decoder, "greedy_search") is None
print("OK")
''' % (REF, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "OK" in out.stdout, out.stderr[-2000:]


def test_mirror_classes_carry_greedy_search_and_evaluate():
    assert b200asr.modules.Decoder.greedy_search is M.greedy_search
    assert b200asr.modules.Transformer.evaluate is M.transformer_evaluate
    m = b200asr.build_model(b200asr.ASRConfig(num_layers=1, vocab=40, feat_extractor="", tgt_max_len=20))
    m.eval()
    with pytest.raises(ValueError, match="trg_max_length"):          # checked before anything is launched
        m.decoder.greedy_search(torch.randn(2, 5, m.decoder.dim_model))
    m.train()
    with pytest.raises(NotImplementedError, match="install"):       # training mode: the reference's own method, absent here
        m.decoder.greedy_search(torch.randn(2, 5, m.decoder.dim_model))
