"""CPU check of the float64 CTC restatement the GPU tests compare against (tests/ctc_util.py): it reproduces the reference's
calculate_metrics(..., loss_type="ctc") of tests/golden/ctc.npz -- loss and d loss / d pred, including the inf loss and NaN
rows of an infeasible utterance -- and the fixture covers every edge case it was made for.  The one place where torch's CPU
backward is not the derivative (ctc_util.cpu_backward_differs: the last frame of an utterance whose last label is the blank)
is left out of the gradient comparison and checked to occur in the fixture."""
import pytest
import torch

from tests.ctc_util import cpu_backward_differs, ctc_float64, load_ctc_golden


@pytest.fixture(scope="module")
def golden():
    return load_ctc_golden()


def test_fixture_covers_the_edge_cases(golden):
    assert set(golden) == {"feasible", "repeats", "blank_label", "empty_target", "no_frames", "infeasible", "short_inputs"}
    gold = {k: c["gold"] for k, c in golden.items()}
    tl = {k: c["target_lengths"] for k, c in golden.items()}
    sizes = {k: c["sizes"] for k, c in golden.items()}
    T = golden["feasible"]["pred"].shape[1]
    rep = gold["repeats"]
    assert any(int(rep[b, i]) == int(rep[b, i + 1]) for b in range(rep.shape[0]) for i in range(int(tl["repeats"][b]) - 1))
    assert any(int(gold["blank_label"][b, i]) == 0 for b in range(3) for i in range(int(tl["blank_label"][b])))
    assert (tl["empty_target"] == 0).any()
    assert ((sizes["no_frames"] == 0) & (tl["no_frames"] == 0)).any()
    assert torch.isinf(golden["infeasible"]["loss"]) and torch.isnan(golden["infeasible"]["grad"]).any()
    assert (sizes["short_inputs"] < T).all()
    c = golden["blank_label"]
    assert cpu_backward_differs(c["gold"], c["sizes"], c["target_lengths"])
    for c in golden.values():                                   # the trainer's own sizes expression, trainer.py:81-82
        assert torch.equal(c["percentages"].clone().mul_(int(c["pred"].shape[1])).int(), c["sizes"])


@pytest.mark.parametrize("case", ["feasible", "repeats", "blank_label", "empty_target", "no_frames", "infeasible", "short_inputs"])
def test_float64_restatement_reproduces_reference(golden, case):
    c = golden[case]
    _, loss, grad = ctc_float64(c["pred"], c["gold"], c["sizes"], c["target_lengths"])
    want, gwant = c["loss"], c["grad"]
    if torch.isinf(want):
        assert torch.isinf(loss) and loss > 0
    else:
        assert abs(float(loss) - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
    nan = torch.isnan(gwant)
    assert torch.equal(torch.isnan(grad), nan)
    keep = ~nan
    for b, t in cpu_backward_differs(c["gold"], c["sizes"], c["target_lengths"]):
        keep[b, t] = False
    assert float((grad[keep] - gwant[keep]).abs().max()) <= 1e-12
    # NaN exactly on the rows t < T_b of an infeasible utterance; 0 on the rows t >= T_b of every utterance
    for b, Tb in enumerate(c["sizes"].tolist()):
        assert (gwant[b, Tb:] == 0).all()
        if case == "infeasible" and b == 1:
            assert nan[b, :Tb].all()
        else:
            assert not nan[b].any()
