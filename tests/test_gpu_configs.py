"""BASELINE.json configs 4 and 5 as parity tests (they are test cases, not bench lines):
  config 4 — 3-D 256^3 inference-only SpatialTransformer + VecInt (sizes the numpy oracle still finishes in seconds);
  config 5 — semi-supervised composition (SURVEY 8(a) A12): flow rescaled to the segmentation resolution, LINEAR warp of
             the one-hot segmentation, Dice loss (+ autograd), and the nearest-neighbour label-map warp, bit-exact."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch, spec_np

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


@pytest.mark.parametrize("arith", ["fast", "exact"])
def test_config4_256cubed_warp_and_vecint(vxm, cuda, arith, monkeypatch):
    monkeypatch.setenv("VXM_B200_LINEAR_ARITH", arith)   # exact: bit-identical to the oracle; fast (default, benched): <= 2e-5
    full = (256, 256, 256)
    vol = cases.smooth_volume(301, full)
    lab = cases.label_volume(302, full)
    flow = cases.smooth_field(303, 3, full, scale=6.0)
    F = t(flow).to(cuda)
    lin = vxm.layers.SpatialTransformer(full)(t(vol).to(cuda), F).cpu().numpy()
    near = vxm.layers.SpatialTransformer(full, mode="nearest")(t(lab).to(cuda), F).cpu().numpy()
    # oracle on a 64-slice slab of the output (the gather may reach anywhere in the source volume)
    sl = slice(96, 160)
    ref_lin = spec_np.warp(vol, flow)[:, :, sl]
    if arith == "exact":
        assert np.array_equal(lin[:, :, sl], ref_lin)
    else:
        assert rel(lin[:, :, sl], ref_lin) <= 2e-5
    assert np.array_equal(near[:, :, sl], spec_np.warp(lab, flow, mode="nearest")[:, :, sl])
    # VecInt at 128^3 (int_downsize = 2 of a 256^3 volume), all steps in one launch, against the oracle
    half = (128, 128, 128)
    vel = cases.smooth_field(304, 3, half, scale=4.0)
    out = vxm.layers.VecInt(half, 7)(t(vel).to(cuda)).cpu().numpy()
    if arith == "exact":
        assert np.array_equal(out, spec_np.vecint(vel, 7))
    else:
        assert rel(out, spec_np.vecint(vel, 7)) <= 2e-5
    # batch of 2 at 256^3: entries independent (size-independent property)
    vb = torch.cat([t(flow), t(flow).flip(0) * 0.5], 0).to(cuda)
    o = vxm.layers.VecInt(full, 3)(vb)
    assert torch.equal(o[:1], vxm.layers.VecInt(full, 3)(vb[:1]))


def test_config5_semisupervised_composition(vxm, cuda):
    shape = (32, 48, 40)
    half = tuple(s // 2 for s in shape)
    nlab = 30
    lab_m = cases.label_volume(311, shape, nlab)
    lab_f = cases.label_volume(312, shape, nlab)
    pos_flow = cases.smooth_field(313, 3, shape, scale=3.0)

    def onehot(lab):
        oh = (lab[:, 0, ::2, ::2, ::2][:, None] == np.arange(nlab, dtype=np.float32)[None, :, None, None, None])
        return oh.astype(np.float32)

    seg_m, seg_f = onehot(lab_m), onehot(lab_f)           # (1, 30, 16, 24, 20), generators.py:163-167 sub-sampling
    # --- oracle: ResizeTransform(2) -> linear warp of the prob-seg -> Dice, with autograd through the flow
    fc = t(pos_flow).double().requires_grad_(True)
    seg_flow_c = ref_torch.resize_transform(fc, 2)
    warped_c = ref_torch.spatial_transform(t(seg_m).double(), seg_flow_c)
    loss_c = ref_torch.dice_loss(t(seg_f).double(), warped_c)
    loss_c.backward()
    # --- GPU path
    fg = t(pos_flow).to(cuda).requires_grad_(True)
    seg_flow_g = vxm.layers.ResizeTransform(2, 3)(fg)
    warped_g = vxm.layers.SpatialTransformer(half)(t(seg_m).to(cuda), seg_flow_g)
    loss_g = vxm.losses.Dice().loss(t(seg_f).to(cuda), warped_g)
    loss_g.backward()
    assert rel(warped_g.detach().cpu().numpy(), warped_c.detach().numpy()) <= 1e-5
    assert abs(float(loss_g) - float(loss_c)) <= 1e-5 * abs(float(loss_c))
    assert rel(fg.grad.cpu().numpy(), fc.grad.numpy()) <= 1e-4
    # --- label-map propagation (evaluation): nearest-neighbour warp at full resolution, bit-exact
    moved = vxm.layers.SpatialTransformer(shape, mode="nearest")(t(lab_m).to(cuda), t(pos_flow).to(cuda)).cpu().numpy()
    assert np.array_equal(moved, spec_np.warp(lab_m, pos_flow, mode="nearest"))
    assert set(np.unique(moved)).issubset(set(np.unique(lab_m)) | {0.0})


def test_config5_semisupervised_model_training_step(vxm, cuda, monkeypatch):
    """The semi-supervised front end (networks.VxmDenseSemiSupervisedSeg, "next" row N2) against the oracle composition of
    the reference's torch pieces (SURVEY 8(a) A12): outputs, the three-term loss [image, Grad, Dice] with weights
    [1, 0.01, 0.01] (scripts/tf/train_semisupervised_seg.py:117-140) and parameter gradients."""
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "f32")
    from test_oracle import full_cfg
    shape = (32, 32, 32)
    nlab = 6
    model = vxm.networks.VxmDenseSemiSupervisedSeg(shape, nlab, nb_unet_features=[[8, 16, 16, 16], [16, 16, 16, 16, 16, 8, 8]])
    cfg = model.vxm_model.config
    sd = ref_torch.init_state_dict(cfg, seed=21, flow_std=2e-2)
    model.vxm_model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(401, shape, sigma=1.5)
    lab_m, lab_f = cases.label_volume(402, shape, nlab), cases.label_volume(403, shape, nlab)
    oh = lambda lab: (lab[:, 0, ::2, ::2, ::2][:, None] == np.arange(nlab, dtype=np.float32)[None, :, None, None, None]).astype(np.float32)  # noqa: E731
    seg_m, seg_f = oh(lab_m), oh(lab_f)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    y, pre, yseg = model(S, T, t(seg_m).to(cuda))
    loss = vxm.losses.MSE().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, pre) \
        + 0.01 * vxm.losses.Dice().loss(t(seg_f).to(cuda), yseg)
    loss.backward()
    # oracle (fp64): VxmDense forward in both modes gives preint and pos_flow; seg branch composed from the torch pieces
    sdc = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    yc, prec = ref_torch.vxm_forward(sdc, cfg, t(s).double(), t(tr).double())
    _, posc = ref_torch.vxm_forward(sdc, cfg, t(s).double(), t(tr).double(), registration=True)
    ysegc = ref_torch.spatial_transform(t(seg_m).double(), ref_torch.resize_transform(posc, 2))
    lossc = ref_torch.mse_loss(t(tr).double(), yc) + 0.01 * ref_torch.grad_loss(prec, "l2", 2) + 0.01 * ref_torch.dice_loss(t(seg_f).double(), ysegc)
    lossc.backward()
    assert rel(y.detach().cpu().numpy(), yc.detach().numpy()) <= 1e-4
    assert rel(yseg.detach().cpu().numpy(), ysegc.detach().numpy()) <= 1e-4
    assert abs(float(loss) - float(lossc)) <= 1e-4 * abs(float(lossc))
    params = dict(model.vxm_model.named_parameters())
    for k in ("flow.weight", "unet_model.encoder.0.0.main.weight", "unet_model.remaining.0.main.bias"):
        assert rel(params[k].grad.cpu().numpy(), sdc[k].grad.numpy()) <= 2e-3, k
    # checkpoint round trip of the wrapper
    import os
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "semi.pt")
        model.save(p)
        m2 = vxm.networks.VxmDenseSemiSupervisedSeg.load(p, "cuda").to(cuda)
        assert m2.config["nb_labels"] == nlab and m2.config["inshape"] == shape
        with torch.no_grad():
            model.eval()
            m2.eval()
            a = model(S, T, t(seg_m).to(cuda))
            b = m2(S, T, t(seg_m).to(cuda))
        assert all(torch.equal(x, z) for x, z in zip(a, b))


def test_jacobian_determinant_on_device(vxm, cuda):
    """Device Jacobian determinant / fold count ("next" row N3) against the host restatement of py/utils.py:473-516."""
    from voxelmorph_b200 import utils
    for shape, sc in (((24, 20, 28), 2.0), ((24, 20, 28), 12.0), ((18, 22), 6.0)):
        nd = len(shape)
        f = cases.smooth_field(500 + nd, nd, shape, scale=sc)        # (1, nd, *shape)
        F = t(f).to(cuda)
        det, folds = utils.jacobian_determinant_device(F, return_folds=True)
        ref = utils.jacobian_determinant(np.moveaxis(f[0], 0, -1))
        assert rel(det[0].cpu().numpy(), ref) <= 1e-5
        clear = np.abs(ref) > 1e-4                                     # the sign of a determinant at rounding level is not defined
        assert np.array_equal((det[0].cpu().numpy() <= 0)[clear], (ref <= 0)[clear])
        assert abs(folds - int((ref <= 0).sum())) <= int((~clear).sum())
        assert utils.count_folds(F) == folds
    assert utils.count_folds(torch.zeros(1, 3, 8, 8, 8, device=cuda)) == 0
