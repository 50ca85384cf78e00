"""CPU checks behind ConditionalTemplateCreation: the fp64 restatement (tests/cond_template_ref.py) against a literal
Keras-order Dense and TF's EluGrad, the conditional_template_creation generator and load_pheno_csv against the
unmodified reference's (frozen in tests/golden/cond_template_generator.npz by oracle/make_golden_cond_template.py), the
model's refusals, checkpoint keys and initialisation, and the C header / ctypes entries of the decoder kernels."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

import cond_template_ref
from conftest import ROOT
from test_generators import assert_same, flatten, make_dataset

INSHAPE = (6, 8, 10)


def make_pheno_dataset(d):
    """Five npz volumes (test_generators.make_dataset), an attribute csv that lists four of them (vol03 is pruned by
    load_pheno_csv), and a (1, *vol, 1) atlas."""
    files = make_dataset(d, n=5, shape=INSHAPE, with_seg=False)
    rng = np.random.RandomState(99)
    csv_path = os.path.join(str(d), "pheno.csv")
    with open(csv_path, "w") as f:
        f.write("subject,age,sex\n")
        for i, name in enumerate(files):
            if i != 3:
                f.write("%s,%.4f,%d\n" % (os.path.basename(name), rng.uniform(20, 90), i % 2))
    atlas = rng.rand(1, *INSHAPE, 1).astype(np.float32)
    return files, csv_path, atlas


GEN_CASES = {
    "b1": dict(batch_size=1),
    "b3": dict(batch_size=3),
    "b2_pad": dict(batch_size=2, pad_shape=(8, 8, 12)),
}


def run_gen(mod, files, atlas, attributes, kw, steps=6, seed=5):
    """Six yields and the np.random state after them (the generator's only draws)."""
    np.random.seed(seed)
    kw = dict(kw)
    if "pad_shape" in kw:
        atlas = np.zeros((1,) + tuple(kw["pad_shape"]) + (1,), np.float32) + atlas.mean()
    gen = mod.conditional_template_creation(files, atlas, attributes, **kw)
    items = [next(gen) for _ in range(steps)]
    return items, np.random.get_state()[1].copy()


@pytest.mark.parametrize("name", sorted(GEN_CASES))
def test_generator_matches_the_reference(tmp_path, golden, name):
    from voxelmorph_b200 import generators, pyutils
    ref = golden("cond_template_generator")
    files, csv_path, atlas = make_pheno_dataset(tmp_path)
    attributes, kept = pyutils.load_pheno_csv(csv_path, files)
    assert [os.path.basename(f) for f in kept] == ["vol00.npz", "vol01.npz", "vol02.npz", "vol04.npz"]
    items, state = run_gen(generators, kept, atlas, attributes, GEN_CASES[name])
    arrs = []
    assert flatten(items, arrs) == json.loads(str(ref["structure"]))[name]
    assert_same(arrs, [ref["%s/%d" % (name, i)] for i in range(len(arrs))])
    assert np.array_equal(state, ref["%s/state" % name])              # exactly the reference's draws
    for (pheno, atl, vols), (v2, *zeros) in items:
        B = GEN_CASES[name]["batch_size"]
        assert pheno.dtype == atl.dtype == vols.dtype == np.float32 and pheno.shape == (B, 2)
        assert v2 is vols and len(zeros) == 3 and all(z.dtype == np.float32 and not z.any() for z in zeros)
        assert zeros[0].shape == (B,) + vols.shape[1:-1] + (3,)


def test_reference_import_surface_has_the_conditional_template():
    from test_shim import run_py
    r = run_py(["-c", "import voxelmorph as vxm, voxelmorph_b200 as v\n"
                      "assert vxm.generators.conditional_template_creation is v.generators.conditional_template_creation\n"
                      "assert vxm.networks.ConditionalTemplateCreation is v.networks.ConditionalTemplateCreation\n"
                      "assert vxm.torch.networks.ConditionalTemplateCreation is v.networks.ConditionalTemplateCreation\n"
                      "assert vxm.py.utils.load_pheno_csv is not None\n"],
               env={"VXM_BACKEND": "pytorch"}, cwd=ROOT)
    assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("vol", [(4, 5, 6), (7, 9)])
def test_keras_order_dense_gives_the_same_template(vol):
    """A literal Keras Dense ((P, V F) kernel, F fastest), ELU, Reshape and channels-last 1x1 convolution gives the decoder
    output and the template of the (P, F, *vol) layout after PhenoDecoder.from_keras."""
    from voxelmorph_b200 import layers
    P, F, B, A = 3, 4, 2, 1
    V = int(np.prod(vol))
    g = torch.Generator().manual_seed(1)
    kernel = torch.randn(P, V * F, generator=g, dtype=torch.float64)
    kbias = torch.randn(V * F, generator=g, dtype=torch.float64)
    like_w = torch.randn((F, F) + (1,) * len(vol), generator=g, dtype=torch.float64)
    like_b = torch.randn(F, generator=g, dtype=torch.float64)
    pheno = torch.randn(B, P, generator=g, dtype=torch.float64)
    W, bias = layers.PhenoDecoder.from_keras(kernel, kbias, vol)
    assert W.shape == (P, F) + vol and bias.shape == (F,) + vol
    # element (p, f, v) is Keras column v F + f
    assert float(W[2, 3].reshape(-1)[5]) == float(kernel[2, 5 * F + 3]) and float(bias[1].reshape(-1)[7]) == float(kbias[7 * F + 1])
    want = cond_template_ref.keras_dense(pheno, kernel, kbias, vol, like_w, like_b)
    got = cond_template_ref.decoder(pheno, W, bias, like_w, like_b)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)
    sd = {"pheno_decoder.weight": W, "pheno_decoder.bias": bias, "pheno_decoder.like_weight": like_w,
          "pheno_decoder.like_bias": like_b}
    for i in range(2):
        sd["extra_convs.%d.weight" % i] = 0.2 * torch.randn((F, F) + (3,) * len(vol), generator=g, dtype=torch.float64)
        sd["extra_convs.%d.bias" % i] = torch.randn(F, generator=g, dtype=torch.float64)
    sd["atlas_gen.weight"] = torch.randn((A, F) + (3,) * len(vol), generator=g, dtype=torch.float64)
    sd["atlas_gen.bias"] = torch.randn(A, generator=g, dtype=torch.float64)
    atlas = torch.randn((1, A) + vol, generator=g, dtype=torch.float64)
    t_layout = cond_template_ref.generator(sd, pheno, atlas, 2)
    x = want
    for i in range(2):
        x = cond_template_ref.conv(x, sd["extra_convs.%d.weight" % i], sd["extra_convs.%d.bias" % i])
    t_keras = atlas + cond_template_ref.conv(x, sd["atlas_gen.weight"], sd["atlas_gen.bias"])
    assert t_layout.shape == (B, A) + vol and torch.allclose(t_layout, t_keras, rtol=1e-12, atol=1e-12)


def test_decoder_gradient_is_tf_elugrad():
    """Autograd of the restatement equals the closed forms: g_pre = (like_w^T g_out)(h < 0 ? h + 1 : 1), gW = pheno^T g_pre,
    gbias = sum_b g_pre, g_like_w = sum_{b,v} g_out h^T, g_like_b = sum_{b,v} g_out."""
    P, F, B, vol = 2, 3, 3, (5, 6, 7)
    g = torch.Generator().manual_seed(2)
    params = [torch.randn((P, F) + vol, generator=g, dtype=torch.float64), torch.randn((F,) + vol, generator=g, dtype=torch.float64),
              torch.randn(F, F, 1, 1, 1, generator=g, dtype=torch.float64), torch.randn(F, generator=g, dtype=torch.float64)]
    params = [p.requires_grad_(True) for p in params]
    pheno = torch.randn(B, P, generator=g, dtype=torch.float64)
    gout = torch.randn((B, F) + vol, generator=g, dtype=torch.float64)
    (cond_template_ref.decoder(pheno, *params) * gout).sum().backward()
    W, bias, lw, lb = [p.detach() for p in params]
    pre = bias + torch.einsum("bp,pf...->bf...", pheno, W)
    h = torch.where(pre > 0, pre, torch.expm1(pre))
    assert (pre < 0).any() and (pre > 0).any()
    gpre = torch.einsum("gf,bg...->bf...", lw.reshape(F, F), gout) * torch.where(h < 0, h + 1, torch.ones_like(h))
    want = [torch.einsum("bp,bf...->pf...", pheno, gpre), gpre.sum(0),
            torch.einsum("bg...,bf...->gf", gout, h).reshape(F, F, 1, 1, 1), gout.sum(dim=(0, 2, 3, 4))]
    for p, w in zip(params, want):
        assert torch.allclose(p.grad, w, rtol=1e-12, atol=1e-12)


def _model(**kw):
    from voxelmorph_b200 import networks
    kw = dict(dict(pheno_input_shape=(2,), nb_unet_features=[[8, 8], [8, 8, 8]], conv_nb_features=4), **kw)
    return networks.ConditionalTemplateCreation(kw.pop("inshape", (8, 8, 8)), **kw)


@pytest.mark.parametrize("kw,match", [(dict(conv_nb_levels=1), "conv_nb_levels"), (dict(templcondsi=True), "templcondsi"),
                                      (dict(conv_image_shape=(8, 8, 8, 8)), "conv_image_shape"),
                                      (dict(conv_size=5), "conv_size")])
def test_refusals(kw, match):
    with pytest.raises(NotImplementedError, match=match):
        _model(**kw)
    _model(conv_image_shape=(8, 8, 8, 4))       # the default shape, spelled out, is accepted


def test_refuses_data_parallel(monkeypatch):
    from voxelmorph_b200 import _lib
    m = _model()
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(_lib.VxmError, match="mean stream"):
        m(torch.zeros(1, 2), torch.zeros(1, 1, 8, 8, 8), torch.zeros(1, 1, 8, 8, 8))


def test_checkpoint_keys_initialisation_and_round_trip(tmp_path):
    from voxelmorph_b200 import networks
    m = _model(extra_conv_layers=2, mean_cap=40, int_steps=5, atlas_feats=2, src_feats=1)
    keys = set(m.state_dict())
    want = {"pheno_decoder.weight", "pheno_decoder.bias", "pheno_decoder.like_weight", "pheno_decoder.like_bias",
            "extra_convs.0.weight", "extra_convs.0.bias", "extra_convs.1.weight", "extra_convs.1.bias",
            "atlas_gen.weight", "atlas_gen.bias", "mean_stream.mean", "mean_stream.count"}
    assert want <= keys and all(k in want or k.startswith("vxm_model.") for k in keys)
    pd = m.pheno_decoder
    assert pd.weight.shape == (2, 4, 8, 8, 8) and pd.bias.shape == (4, 8, 8, 8) and pd.like_weight.shape == (4, 4, 1, 1, 1)
    # Keras defaults: glorot-uniform kernels, zero biases; atlas_gen ~ N(0, 1e-7)
    lim_dense, lim_like, lim_conv = np.sqrt(6 / (2 + 512 * 4)), np.sqrt(6 / 8), np.sqrt(6 / (27 * 8))
    assert 0.9 * lim_dense < float(pd.weight.detach().abs().max()) <= lim_dense
    assert 0.5 * lim_like < float(pd.like_weight.detach().abs().max()) <= lim_like
    assert 0.9 * lim_conv < float(m.extra_convs[1].weight.detach().abs().max()) <= lim_conv
    assert not pd.bias.any() and not pd.like_bias.any() and not m.extra_convs[0].bias.any()
    assert m.atlas_gen.weight.shape == (2, 4, 3, 3, 3) and 0 < float(m.atlas_gen.weight.detach().abs().max()) < 1e-6
    assert 0 < float(m.atlas_gen.bias.detach().abs().max()) < 1e-6
    assert m.vxm_model.bidir and m.vxm_model.config["src_feats"] == 2 and m.vxm_model.config["trg_feats"] == 1
    assert m.mean_stream.cap == 40 and m.mean_stream.mean.shape == (3, 8, 8, 8)
    with torch.no_grad():
        m.mean_stream.count.fill_(7)
    path = os.path.join(str(tmp_path), "c.pt")
    m.save(path)
    r = networks.ConditionalTemplateCreation.load(path, "cpu")
    assert r.config == m.config and set(r.state_dict()) == keys
    for k, v in m.state_dict().items():
        assert torch.equal(r.state_dict()[k], v), k
    n = _model(use_mean_stream=False, inshape=(8, 12))
    assert n.mean_stream is None and not any(k.startswith("mean_stream") for k in n.state_dict())
    assert n.pheno_decoder.like_weight.shape == (4, 4, 1, 1) and n.atlas_gen.weight.shape == (1, 4, 3, 3)


def test_decoder_entry_points_are_declared_consistently():
    from voxelmorph_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    kinds = {ctypes.c_void_p: "*", ctypes.c_int: "int ", ctypes.c_size_t: "size_t ", ctypes.c_float: "float "}
    for name, restype in (("vxm_pheno_decoder_workspace_bytes", "size_t"), ("vxm_pheno_decoder_fwd", "int"),
                          ("vxm_pheno_decoder_bwd", "int")):
        m = re.search(r"\b%s\s+%s\s*\(([^;]*?)\)\s*;" % (restype, name), hdr, re.S)
        assert m, name
        params = [p.strip() for p in m.group(1).split(",")]
        res, args = _lib.SIGNATURES[name]
        assert res is (ctypes.c_int if restype == "int" else ctypes.c_size_t) and len(args) == len(params), name
        for p, a in zip(params, args):
            assert kinds[a] in p, (name, p)
