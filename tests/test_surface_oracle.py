"""CPU checks behind VxmDenseSemiSupervisedPointCloud: the two fp64 restatements of the point warp and the distance
lookup (tests/surface_ref.py) against each other, the model's stored config and checkpoint keys, the refusals of the
layer functions that need no device, and the C header / ctypes entries of the surface kernels."""
import os
import re

import pytest
import torch

import surface_ref as sr
from conftest import ROOT

F64 = torch.float64


def surface_points(g, B, N, shape, L):
    """(B, N, nd+1) points covering every regime: inside, on integer coordinates, exactly on the border and outside
    the volume, with the label column spanning the first and the last label."""
    nd = len(shape)
    cols = []
    for n in shape:
        kind = torch.randint(0, 4, (B, N), generator=g)
        inside = torch.rand(B, N, generator=g, dtype=F64) * (n - 1)
        integer = torch.randint(0, n, (B, N), generator=g).to(F64)
        border = torch.where(torch.rand(B, N, generator=g) < 0.5, 0.0, float(n - 1)).to(F64)
        outside = torch.where(torch.rand(B, N, generator=g) < 0.5, -1.75, n + 0.6).to(F64)
        cols.append(torch.stack([inside, integer, border, outside])[kind, torch.arange(B)[:, None], torch.arange(N)])
    lab = torch.randint(0, L, (B, N), generator=g).to(F64)
    lab[:, 0], lab[:, -1] = 0, L - 1
    return torch.stack(cols + [lab], -1)


CASES = [((9, 7), 3), ((1, 6), 2), ((6, 5, 4), 3), ((1, 5, 4), 1), ((4, 1, 6), 2), ((5, 6, 7), 5)]


@pytest.mark.parametrize("shape,L", CASES)
@pytest.mark.parametrize("r", [1.0, 0.5])
def test_point_warp_closed_form_matches_tf_graph(shape, L, r):
    g = torch.Generator().manual_seed(hash((shape, L)) % 1000)
    B, N, nd = 2, 200, len(shape)
    pts = surface_points(g, B, N, shape, L)
    flow = torch.randn(B, nd, *shape, generator=g, dtype=F64).requires_grad_(True)
    gout = torch.randn(B, N, nd + 1, generator=g, dtype=F64)
    out_tf = sr.point_warp_tf(pts, flow, r)
    out_tf.backward(gout)
    out = sr.point_warp(pts, flow.detach(), r)
    assert torch.equal(out[..., -1], pts[..., -1])
    assert (out - out_tf.detach()).abs().max() < 1e-12
    gflow = sr.point_warp_flow_grad(pts, gout, tuple(flow.shape), r)
    assert (gflow - flow.grad).abs().max() < 1e-12


@pytest.mark.parametrize("shape,L", CASES)
def test_value_at_closed_form_matches_tf_graph(shape, L):
    g = torch.Generator().manual_seed(1 + hash((shape, L)) % 1000)
    B, N, nd = 2, 200, len(shape)
    q = surface_points(g, B, N, shape, L).requires_grad_(True)
    sdt = torch.randn(B, L, *shape, generator=g, dtype=F64)
    sdt[0, 0].flatten()[0] = 0.0                      # a zero value: sign(0) = 0
    gout = torch.randn(B, N, 1, generator=g, dtype=F64)
    v_tf = sr.value_at_tf(sdt, q)
    v_tf.backward(gout)
    v = sr.value_at(sdt, q.detach())
    assert v.shape == v_tf.shape == (B, N, 1)
    assert (v - v_tf.detach()).abs().max() < 1e-12
    gq = sr.value_at_grad(sdt, q.detach(), gout)
    assert (gq[..., :nd] - q.grad[..., :nd]).abs().max() < 1e-12
    assert torch.equal(gq[..., nd], torch.zeros(B, N, dtype=F64))


def test_interp_border_semantics():
    """Worked values of the clamped interpolation on one axis of size 4."""
    vol = torch.tensor([[1.0], [3.0], [7.0], [15.0]], dtype=F64)
    loc = torch.tensor([[-2.0], [0.0], [1.0], [2.5], [3.0], [9.0]], dtype=F64)
    v, dv = sr._interp(vol, loc)
    assert v[:, 0].tolist() == [1.0, 1.0, 3.0, 11.0, 15.0, 15.0]
    assert dv[0, :, 0].tolist() == [0.0, 2.0, 4.0, 8.0, 0.0, 0.0]


SMALL = dict(inshape=(8, 8, 8), nb_surface_points=16, nb_labels_sample=3, nb_unet_features=[[8, 16], [16, 8, 8]])


def _model(**kw):
    from voxelmorph_b200 import networks
    kw = dict(SMALL, **kw)
    return networks.VxmDenseSemiSupervisedPointCloud(kw.pop("inshape"), **kw)


@pytest.mark.parametrize("use_probs", [False, True])
def test_checkpoint_keys_and_config(tmp_path, use_probs):
    from voxelmorph_b200 import networks
    torch.manual_seed(0)
    m = _model(use_probs=use_probs, sdt_vol_resize=0.5, int_steps=5)
    inner = (networks.VxmDenseProbabilistic if use_probs else networks.VxmDense)(
        (8, 8, 8), nb_unet_features=SMALL["nb_unet_features"], bidir=True, int_steps=5)
    assert type(m.vxm_model) is type(inner) and m.vxm_model.bidir
    assert set(m.state_dict()) == {"vxm_model." + k for k in inner.state_dict()}
    assert m.config == dict(inshape=(8, 8, 8), nb_surface_points=16, nb_labels_sample=3,
                            nb_unet_features=SMALL["nb_unet_features"], sdt_vol_resize=0.5, surf_bidir=True,
                            use_probs=use_probs, int_steps=5)
    assert m.sdt_shape == (4, 4, 4)
    path = os.path.join(str(tmp_path), "m.pt")
    m.save(path)
    r = networks.VxmDenseSemiSupervisedPointCloud.load(path, "cpu")
    assert r.config == m.config
    for k, v in m.state_dict().items():
        assert torch.equal(r.state_dict()[k], v), k


def test_layer_refusals_without_a_device():
    from voxelmorph_b200 import _lib, layers
    pts = torch.zeros(1, 4, 4)
    flow = torch.zeros(1, 3, 4, 4, 4)
    sdt = torch.zeros(1, 2, 4, 4, 4)
    with pytest.raises(_lib.VxmError, match="points must not require a gradient"):
        layers.point_spatial_transformer(pts.clone().requires_grad_(True), flow)
    with pytest.raises(_lib.VxmError, match="sdt must not require a gradient"):
        layers.value_at_location(sdt.clone().requires_grad_(True), pts)
    with pytest.raises(_lib.VxmError, match="CUDA tensors are required"):
        layers.point_spatial_transformer(pts, flow)
    with pytest.raises(_lib.VxmError, match="CUDA tensors are required"):
        layers.value_at_location(sdt, pts)


def test_forward_arity_is_checked():
    m = _model(surf_bidir=False)
    x = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(TypeError, match=re.escape("subj_dt, atl_surf")):
        m(x, x, x, x, x, x)


def test_c_declarations_match_ctypes():
    from voxelmorph_b200 import _lib
    header = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    for name in ("vxm_point_warp_workspace_bytes", "vxm_point_warp_fwd", "vxm_point_warp_bwd", "vxm_value_at_fwd",
                 "vxm_value_at_bwd"):
        m = re.search(r"\b%s\(([^;]*)\);" % name, header)
        assert m, name
        nargs = len([a for a in m.group(1).split(",") if a.strip()])
        assert nargs == len(_lib.SIGNATURES[name][1]), name
