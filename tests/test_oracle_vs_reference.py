"""Pin of the oracle restatements (oracle/spec_np.py, oracle/ref_torch.py) against outputs of the UNMODIFIED reference,
frozen by oracle/make_golden_live.py into tests/golden/reference_live.npz (same seeded inputs as below)."""
import numpy as np
import torch

from oracle import cases, ref_torch, spec_np


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def test_layers_live(golden):
    ref = golden("reference_live")
    shape = (10, 14, 12)
    src = cases.smooth_volume(1, shape)
    flow = cases.smooth_field(2, 3, shape, scale=5.0)
    lab = cases.label_volume(3, shape)
    assert np.array_equal(ref["layers/warp_lin"], spec_np.warp(src, flow))
    assert np.array_equal(ref["layers/warp_near"], spec_np.warp(lab, flow, mode="nearest"))
    assert np.array_equal(ref["layers/vecint5"], spec_np.vecint(flow, 5))
    for vr in (2, 0.5):
        r = ref["layers/resize_%g" % vr]
        assert np.array_equal(r, ref_torch.resize_transform(t(flow), vr).numpy())
        np.testing.assert_allclose(spec_np.resize_flow(flow, vr), r, rtol=0, atol=5e-6 * np.abs(flow).max())


def test_losses_live(golden):
    ref = golden("reference_live")
    I, J = cases.volume_pair(7, (16, 20, 18))
    assert abs(float(ref["losses/ncc"]) - spec_np.ncc_loss(I, J)) < 2e-6
    assert float(ref["losses/ncc"]) == np.float32(ref_torch.ncc_loss(t(I), t(J)).item())
    f = cases.smooth_field(8, 3, (8, 10, 12), scale=2.0)
    assert abs(float(ref["losses/grad_l2"]) - spec_np.grad_loss(f, "l2", 2)) < 1e-6
    assert abs(float(ref["losses/mse"]) - spec_np.mse_loss(I, J)) < 1e-7


def test_network_live(golden):
    import voxelmorph_b200 as vxm
    ref = golden("reference_live")
    kw = dict(inshape=(16, 16, 32), nb_unet_features=[[4, 8, 8, 8], [8, 8, 8, 8, 8, 4, 4]], bidir=True)
    cfg = vxm.networks.VxmDense(**kw).config
    sd = ref_torch.init_state_dict(cfg, seed=5, flow_std=2e-2)
    s, g = cases.volume_pair(9, kw["inshape"])
    with torch.no_grad():
        b = ref_torch.vxm_forward(sd, cfg, t(s), t(g))
    assert len(b) == sum(1 for k in ref if k.startswith("network/"))
    assert all(np.array_equal(ref["network/out%d" % i], y.numpy()) for i, y in enumerate(b))


def test_eval_helpers_live(golden):
    """Dice overlap and Jacobian determinant restatements vs reference py/utils.py:265-287, :473-516."""
    ref = golden("reference_live")
    rng = np.random.RandomState(5)
    a, b = rng.randint(0, 5, size=(9, 10, 11)), rng.randint(0, 6, size=(9, 10, 11))
    assert np.array_equal(ref["eval/dice"], spec_np.dice_overlap(a, b))
    assert np.array_equal(ref["eval/dice_labels"], spec_np.dice_overlap(a, b, [1, 3, 7], True))
    for shape in ((7, 9), (6, 7, 8)):
        disp = cases.smooth_field(11, len(shape), shape, scale=3.0)[0]        # (nd, *vol)
        disp = np.moveaxis(disp, 0, -1).astype(np.float64)
        np.testing.assert_allclose(spec_np.jacobian_determinant(disp), ref["eval/jacdet_%dd" % len(shape)], rtol=0, atol=1e-12)
