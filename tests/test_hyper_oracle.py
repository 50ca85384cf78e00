"""CPU checks behind HyperVxmDense: the fp64 restatement (tests/hyper_ref.py) against the closed-form gradients of the
generated weights and a literal per-layer Dense, the flat layout of the package's model, its checkpoint keys, stored
config and initialisation, its refusals, the hypermorph generator against a literal restatement of the training
script's, the loss helper, and the C header / ctypes entries of the hypernetwork kernels."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import hyper_ref
from conftest import ROOT
from test_oracle import full_cfg

SMALL = dict(inshape=(8, 8, 8), nb_unet_features=[[8, 16], [16, 8, 8]])


def _model(**kw):
    from voxelmorph_b200 import networks
    kw = dict(SMALL, **kw)
    return networks.HyperVxmDense(kw.pop("inshape"), **kw)


def test_restatement_gradients_are_the_closed_forms():
    g = torch.Generator().manual_seed(0)
    U, N = 7, 53
    A = torch.randn(U, N, generator=g, dtype=torch.float64, requires_grad=True)
    a = torch.randn(N, generator=g, dtype=torch.float64, requires_grad=True)
    h = torch.rand(U, generator=g, dtype=torch.float64, requires_grad=True)
    dW = torch.randn(N, generator=g, dtype=torch.float64)
    (a + h @ A).backward(dW)
    assert torch.allclose(A.grad, torch.outer(h.detach(), dW), rtol=0, atol=1e-14)
    assert torch.equal(a.grad, dW)
    assert torch.allclose(h.grad, A.detach() @ dW, rtol=0, atol=1e-12)


@pytest.mark.parametrize("kw", [{}, dict(inshape=(8, 12), nb_unet_features=[[16, 16], [16, 16, 8]]),
                                dict(unet_half_res=True), dict(nb_unet_features=[[64, 64], [64, 64, 64]])])
def test_flat_layout_is_a_per_layer_dense(kw):
    """Each convolution's weight and bias are the Dense map of h through that layer's own block of columns, in the U-Net's
    execution order; the package's views and offsets are the restatement's."""
    m = _model(**kw).double()
    cfg = full_cfg(dict(m.config, **dict(SMALL, **kw)))
    lay, N = hyper_ref.layout(cfg)
    assert N == m.hyper.hyper_bias.numel() == m.hyper.hyper_kernel.shape[1]
    assert [(ow, ob) for _, _, ow, ob in lay] == m.hyper.offsets
    assert [s for _, s, _, _ in lay] == m.hyper.shapes
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        m.hyper.hyper_bias.copy_(torch.randn(N, generator=g, dtype=torch.float64))
    A, a = m.hyper.hyper_kernel.detach(), m.hyper.hyper_bias.detach()
    h = torch.rand(A.shape[0], generator=g, dtype=torch.float64)
    wflat = a + h @ A
    views = m.hyper.views(wflat)
    sd = hyper_ref.generated_state_dict(wflat, cfg)
    for (k, s, ow, ob), (w, b) in zip(lay, views):
        # literal Dense of this layer alone: kernel (U, Cout Cin 27) and bias columns, reshaped as TF's HyperConv does
        kw_, kb_ = A[:, ow:ob], A[:, ob:ob + s[0]]
        want_w = (h @ kw_ + a[ow:ob]).reshape(s)
        want_b = h @ kb_ + a[ob:ob + s[0]]
        assert torch.equal(w, want_w) and torch.equal(b, want_b), k
        assert torch.equal(sd[k + ".weight"], want_w) and torch.equal(sd[k + ".bias"], want_b), k
    convs = m._convs
    assert len(convs) == len(lay) and all(tuple(c.weight.shape) == s for c, (_, s, _, _) in zip(convs, lay))


def test_checkpoint_keys_config_and_round_trip(tmp_path):
    from voxelmorph_b200 import networks
    m = _model(nb_hyp_params=2, nb_hyp_layers=3, nb_hyp_units=32, int_steps=5, bidir=True)
    keys = set(m.state_dict())
    want = {"hyper.hyper_kernel", "hyper.hyper_bias", "flow.weight", "flow.bias"} | \
        {"hyper.hypernet.%d.%s" % (i, n) for i in range(3) for n in ("weight", "bias")}
    assert keys == want
    assert not list(m.unet_model.parameters())
    assert m.hyper.hypernet[0].weight.shape == (32, 2) and m.hyper.hypernet[2].weight.shape == (32, 32)
    assert m.config == dict(inshape=(8, 8, 8), nb_hyp_params=2, nb_hyp_layers=3, nb_hyp_units=32, int_steps=5, bidir=True,
                            nb_unet_features=SMALL["nb_unet_features"])
    with torch.no_grad():
        m.hyper.hyper_bias.normal_()
    path = os.path.join(str(tmp_path), "h.pt")
    m.save(path)
    r = networks.HyperVxmDense.load(path, "cpu")
    assert r.config == m.config and set(r.state_dict()) == keys and r.bidir
    for k, v in m.state_dict().items():
        assert torch.equal(r.state_dict()[k], v), k


def test_default_sizes():
    m = _model(inshape=(16, 16, 16), nb_unet_features=None)
    assert m.hyper.hyper_kernel.shape == (128, 326032)
    assert sum(p.numel() for p in m.hyper.hypernet.parameters()) == 82816
    assert sum(p.numel() for p in m.flow.parameters()) == 1299


def test_initialisation_statistics():
    torch.manual_seed(0)
    m = _model(inshape=(16, 16, 16), nb_unet_features=None)
    U = 128
    for i, lin in enumerate(m.hyper.hypernet):
        lim = np.sqrt(6 / (lin.in_features + lin.out_features))
        w = lin.weight.detach()
        assert 0.9 * lim < float(w.abs().max()) <= lim * (1 + 1e-6) and not lin.bias.any(), i
        if w.numel() > 1000:          # uniform(-lim, lim): variance lim^2 / 3
            assert abs(float(w.var()) / (lim * lim / 3) - 1) < 0.1, i
    A = m.hyper.hyper_kernel.detach()
    assert not m.hyper.hyper_bias.any()
    for s, (ow, ob) in zip(m.hyper.shapes, m.hyper.offsets):
        lw, lb = np.sqrt(6 / (U + 27 * s[0] * s[1])), np.sqrt(6 / (U + s[0]))
        blk_w, blk_b = A[:, ow:ob], A[:, ob:ob + s[0]]
        assert 0.99 * lw < float(blk_w.abs().max()) <= lw * (1 + 1e-6), s
        assert 0.8 * lb < float(blk_b.abs().max()) <= lb * (1 + 1e-6), s
        assert abs(float(blk_w.var()) / (lw * lw / 3) - 1) < 0.05, s
        assert abs(float(blk_w.mean())) < 0.05 * lw, s


def test_refusals():
    from voxelmorph_b200 import _lib
    m = _model()
    x = torch.zeros(1, 1, 8, 8, 8)
    for bad in (torch.zeros(2, 1), torch.zeros(1, 2), torch.zeros(1), torch.zeros(1, 1, 1)):
        with pytest.raises(_lib.VxmError, match=re.escape("got %s" % (tuple(bad.shape),))):
            m(x, x, bad)
    with pytest.raises(NotImplementedError, match="use_probs"):
        _model(use_probs=True)
    with pytest.raises(ValueError, match="nb_hyp_units"):
        _model(nb_hyp_units=300)


def _script_hyp_generator(base_generator, batch_size, oversample_rate):
    """scripts/tf/train_hypermorph.py:107-121, literally."""
    def random_hyperparam():
        if np.random.rand() < oversample_rate:
            return np.random.choice([0, 1])
        else:
            return np.random.rand()
    while True:
        hyp = np.expand_dims([random_hyperparam() for _ in range(batch_size)], -1)
        inputs, outputs = next(base_generator)
        inputs = (*inputs, hyp)
        yield (inputs, outputs)


def _base():
    """a base generator that draws from np.random too, so that the interleaving is checked"""
    while True:
        v = np.random.rand(1, 4, 4, 1).astype(np.float32)
        yield ([v, v + 1], [v])


@pytest.mark.parametrize("rate", [0.2, 0.7])
def test_generator_draws_follow_the_script(rate):
    from voxelmorph_b200 import generators
    np.random.seed(11)
    want = [next(g) for g in [_script_hyp_generator(_base(), 1, rate)] for _ in range(40)]
    state = np.random.get_state()[1].copy()
    np.random.seed(11)
    gen = generators.hypermorph(_base(), oversample_rate=rate)
    got = [next(gen) for _ in range(40)]
    assert np.array_equal(np.random.get_state()[1], state)
    lams = []
    for (wi, wo), (gi, go) in zip(want, got):
        assert isinstance(gi, tuple) and len(gi) == 3
        assert gi[2].shape == (1, 1) and gi[2].dtype == np.float32
        assert gi[2][0, 0] == np.float32(wi[2][0, 0])
        assert np.array_equal(gi[0], wi[0]) and np.array_equal(gi[1], wi[1]) and np.array_equal(go[0], wo[0])
        lams.append(float(gi[2][0, 0]))
    assert any(v in (0.0, 1.0) for v in lams) and any(0 < v < 1 for v in lams)


def test_shim_exports():
    import importlib
    os.environ.setdefault("VXM_BACKEND", "pytorch")
    vxm = importlib.import_module("voxelmorph")
    from voxelmorph_b200 import generators, networks
    assert vxm.networks.HyperVxmDense is networks.HyperVxmDense
    assert vxm.generators.hypermorph is generators.hypermorph


def test_loss_helper_weighs_by_lambda():
    from voxelmorph_b200 import losses
    img = torch.tensor(3.0, requires_grad=True)
    reg = torch.tensor(5.0, requires_grad=True)
    hyp = torch.tensor([[0.25]], requires_grad=True)
    loss = losses.hyper_loss(hyp, img, reg)
    loss.backward()
    assert float(loss) == 0.75 * 3 + 0.25 * 5
    assert float(img.grad) == 0.75 and float(reg.grad) == 0.25 and hyp.grad is None


NAMES = (("vxm_hyper_workspace_bytes", "size_t"), ("vxm_hyper_mlp_fwd", "int"), ("vxm_hyper_mlp_bwd", "int"),
         ("vxm_hyper_weights_fwd", "int"), ("vxm_hyper_weights_bwd", "int"))


def test_entry_points_are_declared_consistently():
    from voxelmorph_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    kinds = {ctypes.c_void_p: "*", ctypes.c_int: "int ", ctypes.c_size_t: "size_t ", ctypes.c_float: "float "}
    for name, restype in NAMES:
        m = re.search(r"\b%s\s+%s\s*\(([^;]*?)\)\s*;" % (restype, name), hdr, re.S)
        assert m, name
        params = [p.strip() for p in m.group(1).split(",")]
        res, args = _lib.SIGNATURES[name]
        assert res is (ctypes.c_int if restype == "int" else ctypes.c_size_t) and len(args) == len(params), name
        for p, a in zip(params, args):
            assert kinds[a] in p, (name, p)


def test_entry_points_are_exported_and_refuse_bad_sizes():
    """The size checks run on the host, before any launch: they answer without a GPU."""
    from voxelmorph_b200 import _lib
    lib = _lib.load()
    for name, _ in NAMES:
        assert hasattr(lib, name), name
    assert lib.vxm_hyper_workspace_bytes(128, 326032) == 4 * 128 * 319
    assert lib.vxm_hyper_workspace_bytes(257, 10) == 0 and lib.vxm_hyper_workspace_bytes(8, 0) == 0
    p = ctypes.c_void_p(256)
    arr = (ctypes.c_void_p * 8)(*([256] * 8))
    ptrs = ctypes.cast(arr, ctypes.c_void_p)
    assert lib.vxm_hyper_mlp_fwd(p, ptrs, ptrs, p, p, 17, 128, 6, None) != 0 and "P = 17" in _lib.last_error()
    assert lib.vxm_hyper_mlp_fwd(p, ptrs, ptrs, p, p, 1, 257, 6, None) != 0 and "U = 257" in _lib.last_error()
    assert lib.vxm_hyper_mlp_fwd(p, ptrs, ptrs, p, p, 1, 128, 9, None) != 0 and "9 layers" in _lib.last_error()
    assert lib.vxm_hyper_mlp_fwd(p, ptrs, ptrs, p, p, 0, 128, 6, None) != 0 and "P = 0" in _lib.last_error()
    assert lib.vxm_hyper_mlp_bwd(p, p, ptrs, p, ptrs, ptrs, 1, 128, 6, 2, None) != 0 and "accumulate" in _lib.last_error()
    assert lib.vxm_hyper_mlp_fwd(None, ptrs, ptrs, p, p, 1, 128, 6, None) != 0 and "null pointer" in _lib.last_error()
    assert lib.vxm_hyper_weights_fwd(p, p, p, p, 0, 100, None) != 0 and "U = 0" in _lib.last_error()
    assert lib.vxm_hyper_weights_fwd(p, p, p, p, 8, 0, None) != 0 and "N = 0" in _lib.last_error()
    assert lib.vxm_hyper_weights_bwd(p, p, p, p, p, p, p, 300, 10, 0, None) != 0 and "U = 300" in _lib.last_error()
    assert lib.vxm_hyper_weights_bwd(p, p, p, p, p, p, p, 8, 10, 3, None) != 0 and "accumulate" in _lib.last_error()
