"""CPU checks behind TemplateCreation: the fp64 MeanStream restatement against its closed forms and fp64 autograd, the
template_creation generator against this repo's volgen, the model's checkpoint round trip and state_dict keys, the
data-parallel refusal, and the C header / ctypes entries of the MeanStream kernels."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import template_ref
from conftest import ROOT
from test_generators import make_dataset


def _trajectory(B, cap, steps, shape=(2, 3, 4), seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((B,) + shape, generator=g, dtype=torch.float64) for _ in range(steps)]


@pytest.mark.parametrize("B", [1, 2])
def test_mean_stream_closed_forms_across_the_cap(B):
    """cap = 3, 8 steps: below the cap the state is the plain running mean of every sample seen, past it the update is
    m (1 - B / cap) + mean_b B / cap; the output is min(1, n' / cap) m' for every batch entry."""
    cap = 3
    xs = _trajectory(B, cap, 8)
    mean, count = torch.zeros(xs[0].shape[1:], dtype=torch.float64), 0.0
    seen = []
    for x in xs:
        out, m1, n1 = template_ref.mean_stream(x, mean, count, cap)
        seen.extend(x)
        assert n1 == count + B
        if n1 <= cap:
            want = torch.stack(seen).mean(0)
        else:
            want = mean * (1 - B / cap) + x.mean(0) * B / cap
        assert torch.allclose(m1, want, rtol=0, atol=1e-14)
        assert out.shape == x.shape
        for b in range(B):
            assert torch.allclose(out[b], min(1.0, n1 / cap) * want, rtol=0, atol=1e-14)
        mean, count = m1, n1
    assert count == 8 * B


@pytest.mark.parametrize("B,count", [(1, 0.0), (2, 0.0), (2, 5.0), (1, 40.0)])
def test_mean_stream_gradient_vs_fp64_autograd(B, count):
    """Autograd of the restatement equals the closed form min(1, n'/cap) alpha / B * sum_b' gout_b' for every x_b, and
    nothing reaches the state."""
    cap = 7.0
    g = torch.Generator().manual_seed(B)
    x = torch.randn((B, 3, 5, 6), generator=g, dtype=torch.float64, requires_grad=True)
    mean = torch.randn((3, 5, 6), generator=g, dtype=torch.float64, requires_grad=True)
    gout = torch.randn((B, 3, 5, 6), generator=g, dtype=torch.float64)
    out, _, n1 = template_ref.mean_stream(x, mean, count, cap)
    (out * gout).sum().backward()
    alpha = B / min(n1, cap)
    want = (min(1.0, n1 / cap) * alpha / B) * gout.sum(0)
    for b in range(B):
        assert torch.allclose(x.grad[b], want, rtol=1e-15, atol=0)
    assert mean.grad is None


@pytest.mark.parametrize("shape", [(12, 16, 16), (16, 24)])
def test_template_forward_is_the_bidirectional_vxm_forward(shape):
    """template_ref.template_forward composes the oracle's bidirectional VxmDense with the atlas as the moving image:
    y_source, y_target and pos_flow equal ref_torch.vxm_forward's on the same parameters, for B = 2."""
    from oracle import cases, ref_torch
    from test_oracle import full_cfg
    cfg = full_cfg(dict(inshape=shape, nb_unet_features=[[8, 8], [8, 8, 8]], bidir=True, int_steps=4))
    inner = ref_torch.init_state_dict(cfg, seed=4, dtype=torch.float64, flow_std=2e-2)
    atlas = torch.from_numpy(cases.volume_pair(5, shape)[0]).double()
    imgs = torch.cat([torch.from_numpy(cases.volume_pair(6 + b, shape)[1]).double() for b in range(2)])
    sd = dict({"vxm_model." + k: v for k, v in inner.items()}, atlas=atlas)
    tcfg = dict(cfg, mean_cap=3)
    (y_s, y_t, ms, pos), (m1, n1) = template_ref.template_forward(sd, tcfg, imgs, torch.zeros((len(shape),) + shape, dtype=torch.float64), 0.0)
    want = ref_torch.vxm_forward(inner, cfg, atlas.expand_as(imgs), imgs)
    _, want_pos = ref_torch.vxm_forward(inner, cfg, atlas.expand_as(imgs), imgs, registration=True)
    assert torch.equal(y_s, want[0]) and torch.equal(y_t, want[1]) and torch.equal(pos, want_pos)
    assert n1 == 2 and ms.shape == pos.shape and float(pos.abs().max()) > 0
    loss = template_ref.template_loss((y_s, y_t, ms, pos), atlas.expand_as(imgs), imgs, w_img=0.5)
    assert torch.isfinite(loss)


@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("batch_size", [1, 2])
def test_template_creation_generator_follows_volgen(tmp_path, bidir, batch_size):
    from voxelmorph_b200 import generators as G
    files = make_dataset(tmp_path, shape=(6, 8, 10))
    np.random.seed(11)
    gen = G.template_creation(files, bidir=bidir, batch_size=batch_size)
    items = [next(gen) for _ in range(5)]
    state = np.random.get_state()[1].copy()
    np.random.seed(11)
    vg = G.volgen(files, batch_size=batch_size)
    scans = [next(vg)[0] for _ in range(5)]
    assert np.array_equal(np.random.get_state()[1], state)      # exactly volgen's draws
    for (inv, outv), scan in zip(items, scans):
        assert len(inv) == 1 and len(outv) == (4 if bidir else 3)
        assert np.array_equal(inv[0], scan) and np.array_equal(outv[0], scan)
        for z in outv[1:]:
            assert z.shape == (1, 6, 8, 10, 3) and z.dtype == np.float32 and not z.any()


def test_reference_import_surface_has_the_template_pieces():
    """`import voxelmorph as vxm` (in a process of its own: it selects the default engine) reaches the generator and the
    model under the reference's names."""
    from test_shim import run_py
    r = run_py(["-c", "import voxelmorph as vxm, voxelmorph_b200 as v\n"
                      "assert vxm.generators.template_creation is v.generators.template_creation\n"
                      "assert vxm.networks.TemplateCreation is v.networks.TemplateCreation\n"
                      "assert vxm.torch.networks.TemplateCreation is v.networks.TemplateCreation\n"],
               env={"VXM_BACKEND": "pytorch"}, cwd=ROOT)
    assert r.returncode == 0, r.stderr


def _model(**kw):
    from voxelmorph_b200 import networks
    return networks.TemplateCreation((8, 8, 8), nb_unet_features=[[8, 8], [8, 8, 8]], mean_cap=50, **kw)


def test_template_checkpoint_round_trip(tmp_path):
    from voxelmorph_b200 import networks
    m = _model(int_steps=5)
    keys = set(m.state_dict())
    assert {"atlas", "mean_stream.mean", "mean_stream.count"} <= keys
    assert all(k in ("atlas", "mean_stream.mean", "mean_stream.count") or k.startswith("vxm_model.") for k in keys)
    assert m.atlas.shape == (1, 1, 8, 8, 8) and float(m.atlas.detach().abs().max()) < 1e-5
    assert m.mean_stream.mean.shape == (3, 8, 8, 8) and m.mean_stream.cap == 50
    assert m.vxm_model.bidir and m.vxm_model.config["src_feats"] == 1 and m.vxm_model.config["int_steps"] == 5
    with torch.no_grad():
        m.mean_stream.mean.normal_()
        m.mean_stream.count.fill_(17)
    m.set_atlas(np.arange(512, dtype=np.float32).reshape(8, 8, 8))
    path = os.path.join(str(tmp_path), "t.pt")
    m.save(path)
    r = networks.TemplateCreation.load(path, "cpu")
    assert r.config == m.config and set(r.state_dict()) == keys
    for k, v in m.state_dict().items():
        assert torch.equal(r.state_dict()[k], v), k
    assert np.array_equal(r.get_atlas(), np.arange(512, dtype=np.float32).reshape(8, 8, 8))


def test_set_atlas_shapes_keep_the_parameter():
    m = _model(atlas_feats=2)
    p = m.atlas
    a = torch.randn(1, 2, 8, 8, 8)
    m.set_atlas(a)
    assert m.atlas is p and torch.equal(p.detach(), a)
    m.set_atlas(a[0].numpy() * 2)
    assert m.atlas is p and torch.equal(p.detach(), 2 * a)
    assert m.get_atlas().shape == (2, 8, 8, 8)
    with pytest.raises(ValueError):
        m.set_atlas(np.zeros((8, 8, 8), np.float32))      # a bare volume needs C == 1


def test_template_refuses_data_parallel(monkeypatch):
    from voxelmorph_b200 import _lib
    m = _model()
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(_lib.VxmError, match="mean stream"):
        m(torch.zeros(1, 1, 8, 8, 8))


def test_mean_stream_entry_points_are_declared_consistently():
    from voxelmorph_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    for name in ("vxm_mean_stream_fwd", "vxm_mean_stream_bwd"):
        m = re.search(r"\bint\s+%s\s*\(([^;]*?)\)\s*;" % name, hdr, re.S)
        assert m, name
        params = [p.strip() for p in m.group(1).split(",")]
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == len(params), (name, len(args), len(params))
        kinds = {ctypes.c_void_p: "*", ctypes.c_int: "int ", ctypes.c_size_t: "size_t ", ctypes.c_float: "float "}
        for p, a in zip(params, args):
            assert kinds[a] in p or (a is ctypes.c_void_p and "*" in p), (name, p)
