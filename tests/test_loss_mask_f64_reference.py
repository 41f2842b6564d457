"""CPU: the float64 restatement of the masked loss (tests/loss_mask_f64.py, DESIGN D26) against float64 autograd of
D26's plain formula, against the unmasked restatement at an all-ones mask, and its ignored-pixel rules."""
import numpy as np
import pytest
import torch

import loss_f64
import loss_mask_f64 as lm
from project_f64 import F8


def _case(H, W, kind, seed=0):
    r, g = loss_f64.tie_images(H, W, seed)
    return torch.from_numpy(r), torch.from_numpy(g), torch.from_numpy(lm.make_mask(H, W, kind, seed + 1))


@pytest.mark.parametrize("H,W,kind", [(7, 5, "random"), (23, 31, "blobs"), (40, 33, "random"), (19, 26, "single"),
                                      (1, 1, "ones"), (12, 17, "ones")])
def test_restatement_equals_autograd_of_the_plain_formula(H, W, kind):
    r, g, m = _case(H, W, kind)
    ref = lm.loss(r, g, m, 0.2)
    y = r.to(F8).requires_grad_()
    total, l1, ssim = lm.plain_loss(y, g.to(F8), m, 0.2)
    total.backward()
    total, l1, ssim = (float(t.detach()) for t in (total, l1, ssim))
    assert abs(ref["loss"] - total) <= 1e-12 * max(1.0, abs(total))
    assert abs(ref["l1"] - l1) <= 1e-12 and abs(ref["ssim"] - ssim) <= 1e-12
    scale = float(y.grad.abs().max()) + 1e-300
    assert float((ref["v_rendered"] - y.grad).abs().max()) <= 1e-10 * scale + 1e-15
    assert ref["n"] == int((m != 0).sum())


@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (33, 47)])
def test_all_ones_mask_is_the_unmasked_restatement(H, W):
    r, g = loss_f64.tie_images(H, W, 3)
    r, g = torch.from_numpy(r), torch.from_numpy(g)
    a = lm.loss(r, g, torch.ones(H, W, dtype=torch.uint8), 0.2)
    b = loss_f64.loss(r, g, 0.2)
    for k in ("loss", "l1", "ssim", "B_loss", "B_l1", "B_ssim"):
        assert a[k] == b[k], k
    for k in ("v_rendered", "B_v_rendered", "d_mu", "d_e22", "d_e12", "B_d_mu"):
        assert torch.equal(a[k], b[k]), k


def test_ignored_pixels_get_zero_gradient_and_their_content_never_leaks():
    H, W = 29, 37
    r, g, m = _case(H, W, "blobs", 5)
    ref = lm.loss(r, g, m, 0.2)
    ign = (m == 0)
    assert int(ign.sum()) > 0
    assert torch.count_nonzero(ref["v_rendered"][ign]) == 0 and torch.count_nonzero(ref["B_v_rendered"][ign]) == 0
    assert torch.count_nonzero(ref["v_rendered"][~ign]) > 0
    # overwrite the ignored pixels of both images with junk, NaN and inf: every output stays the same
    rng = np.random.default_rng(9)
    r2, g2 = r.clone(), g.clone()
    junk = torch.from_numpy(rng.uniform(-5, 5, (int(ign.sum()), 3)).astype(np.float32))
    junk[0, 0], junk[1, 1], junk[2, 2] = float("nan"), float("inf"), -float("inf")
    r2[ign], g2[ign] = junk, junk.flip(0)
    ref2 = lm.loss(r2, g2, m, 0.2)
    for k in ("loss", "l1", "ssim"):
        assert ref[k] == ref2[k], k
    assert torch.equal(ref["v_rendered"], ref2["v_rendered"])


def test_normalisation_by_the_used_pixels():
    """A used pixel far from the mask boundary pulls as hard as in an unmasked image of the used pixels only: with the
    right half ignored, the L1 part of the loss of [H, 2W] equals that of the left [H, W] image alone."""
    H, W = 16, 24
    r, g = loss_f64.tie_images(H, 2 * W, 2)
    r, g = torch.from_numpy(r), torch.from_numpy(g)
    m = torch.zeros(H, 2 * W, dtype=torch.uint8)
    m[:, :W] = 1
    a = lm.loss(r, g, m, 0.0)
    b = loss_f64.loss(r[:, :W].contiguous(), g[:, :W].contiguous(), 0.0)
    assert abs(a["l1"] - b["l1"]) <= 1e-15 and abs(a["loss"] - b["loss"]) <= 1e-15


def test_no_used_pixel():
    r, g, m = _case(9, 11, "zero")
    ref = lm.loss(r, g, m, 0.2)
    assert (ref["loss"], ref["l1"], ref["ssim"], ref["n"]) == (0.0, 0.0, 1.0, 0)
    assert torch.count_nonzero(ref["v_rendered"]) == 0


def test_masks_are_seeded_and_of_their_kind():
    for kind in ("random", "blobs", "single", "zero", "ones"):
        a, b = lm.make_mask(20, 30, kind, 4), lm.make_mask(20, 30, kind, 4)
        assert np.array_equal(a, b) and a.dtype == np.uint8 and set(np.unique(a)) <= {0, 1}
    assert lm.make_mask(20, 30, "single", 1).sum() == 1
    assert 0 < lm.make_mask(50, 60, "blobs", 1).mean() < 1
