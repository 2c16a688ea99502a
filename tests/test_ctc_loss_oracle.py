"""The float64 CTC oracle (tests/_oracle_ctc_loss.py) against torch's CPU ctc_loss in float64: per-sample losses and
gradients on every shared case, with the same non-finite pattern (an infeasible sample: loss inf, NaN on every frame
before its input length) and exact zeros on the frames past each input length."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _oracle_ctc_loss as O


def _torch_cpu(c):
    lp = torch.from_numpy(c["log_probs"]).requires_grad_()
    nll = F.ctc_loss(lp, torch.from_numpy(c["targets"]), torch.from_numpy(c["input_lengths"]),
                     torch.from_numpy(c["target_lengths"]), blank=c["blank"], reduction="none")
    nll.sum().backward()
    return nll.detach().numpy(), lp.grad.numpy()


@pytest.mark.parametrize("c", O.cases(), ids=lambda c: c["name"])
def test_oracle_matches_torch_cpu_float64(c):
    ref_nll, ref_grad = _torch_cpu(c)
    nll, grad = O.ctc_loss(c["log_probs"], c["targets"], c["input_lengths"], c["target_lengths"], c["blank"])
    assert np.array_equal(np.isfinite(nll), np.isfinite(ref_nll)) and np.array_equal(np.isnan(grad), np.isnan(ref_grad))
    fin = np.isfinite(ref_nll)
    assert np.allclose(nll[fin], ref_nll[fin], rtol=1e-12, atol=1e-10)
    assert np.array_equal(nll[~fin], ref_nll[~fin])
    ok = ~np.isnan(ref_grad)
    assert float(np.abs(grad[ok] - ref_grad[ok]).max()) <= 1e-12
    for n, il in enumerate(c["input_lengths"]):
        assert not grad[il:, n].any() and not ref_grad[il:, n].any()


def test_cases_cover_the_edges():
    cs = {c["name"]: c for c in O.cases()}
    mixed = cs["mixed_padded"]
    assert {1, mixed["log_probs"].shape[0]} <= set(mixed["input_lengths"].tolist())
    assert {0, 1} <= set(mixed["target_lengths"].tolist()) and cs["mixed_concat"]["targets"].ndim == 1
    b = cs["feasibility_boundary"]
    rep = list(b["targets"][0, :b["target_lengths"][0]])
    need = len(rep) + O.repeats(rep)
    assert O.repeats(rep) > 0 and list(b["input_lengths"][:2]) == [need, need - 1]
    nll, grad = O.ctc_loss(b["log_probs"], b["targets"], b["input_lengths"], b["target_lengths"])
    assert np.isfinite(nll[0]) and nll[1] == np.inf and np.isnan(grad[:need - 1, 1]).all()
    assert np.isfinite(grad[:, 0]).all()
    assert {c["blank"] for c in cs.values()} >= {0, 2, 4, 255}
    assert max(c["log_probs"].shape[2] for c in cs.values()) == 256
