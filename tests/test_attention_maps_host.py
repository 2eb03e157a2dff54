"""b200asr.attention_maps, the switch that makes the attention forwards return their probability maps, and the layout of
the maps (no GPU needed)."""
import importlib

import pytest
import torch

import b200asr

ops = importlib.import_module(b200asr.__name__ + ".ops")


@pytest.fixture(autouse=True)
def _restore_switch():
    before = ops.attention_maps_enabled()
    yield
    ops.attention_maps(before)


def test_off_by_default_and_exported():
    assert b200asr.attention_maps is ops.attention_maps
    assert "attention_maps" in b200asr.__all__
    assert ops.attention_maps_enabled() is False


def test_called_as_a_function_sets_the_state():
    b200asr.attention_maps(True)
    assert ops.attention_maps_enabled() is True
    b200asr.attention_maps(False)
    assert ops.attention_maps_enabled() is False


def test_with_block_restores_and_nests():
    with b200asr.attention_maps(True):
        assert ops.attention_maps_enabled()
        with b200asr.attention_maps(False):
            assert not ops.attention_maps_enabled()
            with b200asr.attention_maps(True):
                assert ops.attention_maps_enabled()
            assert not ops.attention_maps_enabled()
        assert ops.attention_maps_enabled()
    assert not ops.attention_maps_enabled()


def test_with_block_restores_after_an_exception():
    with pytest.raises(RuntimeError):
        with b200asr.attention_maps(True):
            with b200asr.attention_maps(True):
                raise RuntimeError("inside")
    assert not ops.attention_maps_enabled()
    b200asr.attention_maps(True)
    with pytest.raises(ValueError):
        with b200asr.attention_maps(False):
            raise ValueError("inside")
    assert ops.attention_maps_enabled()


def test_install_and_uninstall_leave_the_switch_alone():
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("reference checkout not staged (oracle/make_ref.py)")
    ref_shim.load(["--num-layers", "1"])
    for state in (True, False):
        b200asr.attention_maps(state)
        b200asr.install()
        try:
            assert ops.attention_maps_enabled() is state
        finally:
            b200asr.uninstall()
        assert ops.attention_maps_enabled() is state


@pytest.mark.parametrize("B,H,Tq,Tk", [(1, 1, 1, 1), (3, 2, 5, 7), (2, 4, 3, 1), (4, 3, 1, 6)])
def test_layout_is_the_order_of_mask_repeat(B, H, Tq, Tk):
    """maps_layout puts probability (b, h, t, j) where MultiHeadAttention's mask.repeat(H, 1, 1) puts mask[b, t, j] for head h
    (models/common_layers.py:189): row block h * B + b."""
    shape, (bs, hs, rs) = ops.maps_layout(B, H, Tq, Tk)
    mask = torch.arange(B * Tq * Tk).view(B, Tq, Tk)
    expect = torch.cat([mask] * H, dim=0)                   # restatement of mask.repeat(H, 1, 1)
    assert torch.equal(expect, mask.repeat(H, 1, 1))
    got = torch.full((H * B * Tq * Tk,), -1, dtype=torch.long)
    for b in range(B):
        for h in range(H):
            for t in range(Tq):
                for j in range(Tk):
                    got[b * bs + h * hs + t * rs + j] = mask[b, t, j]
    assert tuple(shape) == tuple(expect.shape)
    assert torch.equal(got.view(shape), expect)
