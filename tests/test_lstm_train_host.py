"""CPU tests of the LSTM LM training path's host side: the gate interleave of the prepared layout and its inverse, and the
install() binding of the reference's RNNModel.forward."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ref_shim


def _prepare(w, nhid, width):
    """lstm_prepare restated: PyTorch row g * nhid + u -> prepared row 4u + g of [4H][width], zero padded."""
    H = (nhid + 7) // 8 * 8
    out = np.zeros((4 * H, width), dtype=w.dtype)
    for g in range(4):
        for u in range(nhid):
            out[4 * u + g, :w.shape[1]] = w[g * nhid + u]
    return out


def _unprepare(wp, nhid, cols):
    """lstm_grad_unprepare restated: prepared row 4u + g -> PyTorch row g * nhid + u, padding dropped."""
    return np.stack([wp[4 * u + g, :cols] for g in range(4) for u in range(nhid)])


@pytest.mark.parametrize("nhid,ninp", [(8, 12), (13, 20), (650, 400)])
def test_interleave_and_its_inverse_round_trip(nhid, ninp):
    rng = np.random.default_rng(nhid)
    w = rng.standard_normal((4 * nhid, ninp)).astype(np.float32)
    I, H = (ninp + 7) // 8 * 8, (nhid + 7) // 8 * 8
    wp = _prepare(w, nhid, I)
    assert np.array_equal(_unprepare(wp, nhid, ninp), w)
    assert not wp[4 * nhid:].any() and not wp[:, ninp:].any()          # padded units and columns are 0
    for blk in range(0, 4 * H, 32):                                     # a 32-column epilogue piece: all four gates of 8 units
        units = {r // 4 for r in range(blk, blk + 32)}
        assert len(units) == 8 and all({4 * u + g for g in range(4)} <= set(range(blk, blk + 32)) for u in units)


@pytest.mark.skipif(ref_shim.reference_root() is None, reason="reference checkout not staged (oracle/make_ref.py)")
def test_install_binds_and_restores_rnn_model_forward_and_gru_runs_on_cpu():
    """Runs in a subprocess because the reference parses flags at import (utils/constant.py:99)."""
    REF = ref_shim.reference_root()
    code = r'''
import sys, types
sys.path.insert(0, %r); sys.path.insert(0, %r)
sys.modules["Levenshtein"] = types.ModuleType("Levenshtein")
sys.argv = ["x"]
import torch
import utils.lstm_utils as lu
import b200asr
orig = lu.RNNModel.forward
torch.manual_seed(0)
gru = lu.RNNModel("GRU", 30, 16, 16, 2, dropout=0.0).eval()
inp = torch.randint(0, 30, (6, 2))
want, _ = gru(inp, gru.init_hidden(2))
b200asr.install()
f = lu.RNNModel.forward
assert f is not orig and f.__name__ == "rnn_model_forward" and f.__module__.endswith("modules")
got, _ = gru(inp, gru.init_hidden(2))                 # not an LSTM: the reference's own forward, on the CPU
assert torch.equal(got, want)
lstm = lu.RNNModel("LSTM", 30, 16, 16, 2, dropout=0.0)
try:
    lstm(inp, lstm.init_hidden(2))
    raise SystemExit("expected the CUDA-only error")
except ValueError as e:
    assert "CUDA" in str(e)
b200asr.uninstall()
assert lu.RNNModel.forward is orig
out, _ = lstm(inp, lstm.init_hidden(2))
assert out.shape == (6, 2, 30)
print("OK")
''' % (REF, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "OK" in out.stdout, out.stderr[-2000:]
