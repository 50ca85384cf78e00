"""CPU checks behind the image gradients: the fp64 closed form of d NCC / d y_true against fp64 autograd of the
reference restatement, and the C header / ctypes table entries of the two-sided NCC entry points."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import cases, ref_torch, spec_np

import image_grads_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _autograd(I, J, win):
    It = torch.from_numpy(I).double().requires_grad_(True)
    Jt = torch.from_numpy(J).double().requires_grad_(True)
    loss = ref_torch.ncc_loss(It, Jt, list(win))
    loss.backward()
    return float(loss.detach()), It.grad.numpy(), Jt.grad.numpy()


@pytest.mark.parametrize("shape,win", [((14, 17, 19), (9, 9, 9)), ((12, 13, 16), (5, 5, 5)), ((33, 41), (9, 9)), ((20, 23), (3, 3))],
                         ids=["3d-9", "3d-5", "2d-9", "2d-3"])
def test_ncc_grad_true_vs_fp64_autograd(shape, win):
    I, J = cases.volume_pair(21, shape, sigma=2.0)
    loss, gI, gJ = _autograd(I, J, win)
    assert abs(spec_np.ncc_loss(I, J, list(win)) - loss) <= 1e-12 * abs(loss)
    mine = image_grads_ref.ncc_grad_true(I, J, list(win))
    assert np.abs(mine - gI).max() <= 1e-10 * np.abs(gI).max()
    # the yardstick itself: the existing closed form for y_pred against the same autograd run
    assert np.abs(spec_np.ncc_grad_pred(I, J, list(win)) - gJ).max() <= 1e-10 * np.abs(gJ).max()


def test_ncc_grad_true_non_cubic_window():
    """ref_torch.ncc_loss pads every axis by win[0] // 2, so a window that is not a cube is differentiated numerically
    here: central differences of spec_np.ncc_loss (fp64) at a handful of voxels."""
    win = [3, 7, 5]
    I, J = cases.volume_pair(22, (9, 12, 11), sigma=1.5)
    g = image_grads_ref.ncc_grad_true(I, J, win)
    rng = np.random.default_rng(0)
    I64 = I.astype(np.float64)
    for _ in range(12):
        idx = (0, 0) + tuple(int(rng.integers(0, n)) for n in I.shape[2:])
        h = 1e-5
        up, dn = I64.copy(), I64.copy()
        up[idx] += h
        dn[idx] -= h
        fd = (spec_np.ncc_loss(up, J, win) - spec_np.ncc_loss(dn, J, win)) / (2 * h)
        assert abs(fd - g[idx]) <= 1e-6 * np.abs(g).max(), (idx, fd, g[idx])


def test_ncc_grad_true_is_grad_pred_with_the_images_swapped():
    I, J = cases.volume_pair(23, (11, 15, 13), sigma=2.0)
    a = image_grads_ref.ncc_grad_true(I, J, [5, 5, 5])
    b = spec_np.ncc_grad_pred(J, I, [5, 5, 5])
    assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max()


def test_dice_is_symmetric_in_its_arguments_clamp_included():
    """d Dice / d y_true by fp64 autograd equals d Dice / d y_pred with the tensors swapped, also for a label that is
    absent from both maps (bottom at the clamp floor): what lets one backward kernel serve both arguments."""
    g = torch.Generator().manual_seed(3)
    a = torch.rand((2, 4, 6, 7, 5), generator=g, dtype=torch.float64)
    b = torch.rand((2, 4, 6, 7, 5), generator=g, dtype=torch.float64)
    a[:, 2] = 0
    b[:, 2] = 0
    at, bt = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref_torch.dice_loss(at, bt).backward()
    a2, b2 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref_torch.dice_loss(b2, a2).backward()
    assert torch.equal(at.grad, a2.grad) and torch.equal(bt.grad, b2.grad)
    assert float(at.grad[:, 2].abs().max()) == 0.0      # the kernel's clamp branch: k1 * 0 - 0


def test_two_sided_ncc_entry_points_are_declared_consistently():
    """vxm_ncc_fwd2 / vxm_ncc_bwd2: declared in the header, present in the ctypes table with one entry per C parameter
    (pointers as void*, `which` and the sizes as int)."""
    import ctypes
    from voxelmorph_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    for name in ("vxm_ncc_fwd2", "vxm_ncc_bwd2"):
        m = re.search(r"\bint\s+%s\s*\(([^;]*?)\)\s*;" % name, hdr, re.S)
        assert m, name
        params = [p.strip() for p in m.group(1).split(",")]
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == len(params), (name, len(args), len(params))
        for p, a in zip(params, args):
            assert (a is ctypes.c_void_p) == ("*" in p), (name, p)
            assert "*" in p or p.startswith("int "), (name, p)
        assert "int which" in params
