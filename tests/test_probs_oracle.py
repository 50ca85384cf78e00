"""Probabilistic VoxelMorph on the CPU: the KL closed form against a literal transcription of the reference's TF loss, its
gradient against autograd, the noise stream's restatement, the model's constructor, config and key set, and the
wrappers' refusal of use_probs."""
import numpy as np
import pytest
import torch

import probs_ref

# odd sizes, size-2 and size-1 axes (a size-1 axis has no neighbours along it and no differences)
KL_SHAPES = [(2, 6, 5, 7, 9), (1, 6, 2, 5, 3), (1, 6, 1, 4, 6), (3, 4, 7, 5), (2, 4, 1, 6), (1, 6, 1, 1, 5)]


def _params(shape, seed):
    g = np.random.default_rng(seed)
    p = g.standard_normal(shape)
    nd = len(shape) - 2
    p[:, nd:] = p[:, nd:] - 2.0          # log variances around e^-2
    return p


@pytest.mark.parametrize("lam", [10.0, 0.3])
@pytest.mark.parametrize("shape", KL_SHAPES)
def test_kl_closed_form_matches_literal_transcription(shape, lam):
    p = _params(shape, 1)
    want = float(probs_ref.kl_literal(torch.from_numpy(p), lam))
    got = probs_ref.kl_loss(p, lam)
    assert abs(got - want) <= 1e-13 * abs(want), (got, want)


def test_kl_degree_is_the_adjacency_conv():
    assert probs_ref.degree((4, 5, 6))[1:-1, 1:-1, 1:-1].min() == 6
    assert probs_ref.degree((1, 3))[0].tolist() == [1, 2, 1]
    assert probs_ref.degree((2, 1, 2)).max() == 2


@pytest.mark.parametrize("shape", KL_SHAPES)
def test_kl_grad_matches_autograd(shape):
    p = _params(shape, 2)
    t = torch.from_numpy(p).requires_grad_(True)
    probs_ref.kl_torch(t, 10.0).backward()
    g, mag = probs_ref.kl_grad(p, 10.0)
    assert np.abs(g - t.grad.numpy()).max() <= 1e-13 * np.abs(g).max()
    assert (mag >= np.abs(g) - 1e-18).all()
    assert abs(float(probs_ref.kl_torch(t, 10.0)) - probs_ref.kl_loss(p, 10.0)) <= 1e-13 * abs(probs_ref.kl_loss(p, 10.0))


def test_philox_known_answer():
    # Random123's published known-answer vectors for philox4x32_10 (kat_vectors)
    w = probs_ref.philox4x32_10([np.uint32([0])] * 4, (0, 0))
    assert [int(x[0]) for x in w] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    w = probs_ref.philox4x32_10([np.uint32([0xFFFFFFFF])] * 4, (0xFFFFFFFF, 0xFFFFFFFF))
    assert [int(x[0]) for x in w] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    w = probs_ref.philox4x32_10([np.uint32([0x243F6A88]), np.uint32([0x85A308D3]), np.uint32([0x13198A2E]),
                                 np.uint32([0x03707344])], (0xA4093822, 0x299F31D0))
    assert [int(x[0]) for x in w] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_noise_stream_is_deterministic_and_keyed():
    a = probs_ref.normal_stream(1001, 123, 0)
    assert np.array_equal(a, probs_ref.normal_stream(1001, 123, 0))
    assert np.array_equal(a[:37], probs_ref.normal_stream(37, 123, 0))          # a prefix: no dependence on n
    others = [probs_ref.normal_stream(1001, s, c) for s, c in ((124, 0), (123, 1), (123 + (1 << 32), 0), (123, 1 << 32))]
    for o in others:
        assert np.abs(o - a).max() > 1.0
    assert np.isfinite(a).all() and np.abs(a).max() <= np.sqrt(2 * 24 * np.log(2)) + 1e-12
    big = probs_ref.normal_stream(400_000, 5, 7)
    m, v = probs_ref.standard_error_bounds(big)
    assert abs(big.mean()) <= m and abs(big.var() - 1) <= v


def test_rank_seed_mixes_the_rank():
    import voxelmorph_b200 as vxm
    seeds = [vxm.networks.rank_seed(42, r) for r in range(8)]
    assert seeds[0] == 42 and len(set(seeds)) == 8
    assert all(0 <= s < (1 << 63) for s in seeds)
    assert vxm.networks.rank_seed(43, 1) != seeds[1]


def test_probabilistic_constructor_config_and_keys(tmp_path):
    import voxelmorph_b200 as vxm
    torch.manual_seed(3)
    m = vxm.networks.VxmDenseProbabilistic((16, 16, 16), bidir=True, int_steps=5)
    torch.manual_seed(3)
    plain = vxm.networks.VxmDense((16, 16, 16), bidir=True, int_steps=5)
    assert "use_probs" not in m.config and m.config["int_steps"] == 5 and m.config["bidir"] is True
    assert list(m.state_dict()) == list(plain.state_dict()) + ["log_sigma.weight", "log_sigma.bias"]
    # the U-Net and flow head are drawn as VxmDense draws them, then the log-variance head, then the seed
    for k, v in plain.state_dict().items():
        assert torch.equal(v, m.state_dict()[k]), k
    assert m.log_sigma.weight.shape == (3, 16, 3, 3, 3) and torch.equal(m.log_sigma.bias, torch.full((3,), -10.0))
    assert float(m.log_sigma.weight.abs().max()) < 1e-8
    assert m.noise_state.dtype == torch.int64 and m.noise_state.tolist()[1] == 0
    names = [n for n, _ in m.named_parameters()]
    assert names.index("log_sigma.weight") == names.index("flow.bias") + 1
    # torch.manual_seed reproduces the seed; a later model draws another
    torch.manual_seed(3)
    again = vxm.networks.VxmDenseProbabilistic((16, 16, 16), bidir=True, int_steps=5)
    assert torch.equal(again.noise_state, m.noise_state)
    assert not torch.equal(vxm.networks.VxmDenseProbabilistic((16, 16, 16)).noise_state, m.noise_state)
    # checkpoint round trip through modelio (noise_state is not in the file)
    p = tmp_path / "m.pt"
    m.save(p)
    assert "noise_state" not in torch.load(p)["model_state"]
    m2 = vxm.networks.VxmDenseProbabilistic.load(p, "cpu")
    assert m2.config == m.config
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    with pytest.raises(TypeError):
        vxm.networks.VxmDenseProbabilistic((16, 16), use_probs=True)
    m2d = vxm.networks.VxmDenseProbabilistic((32, 32))
    assert m2d.log_sigma.weight.shape == (2, 16, 3, 3)


def test_log_sigma_init_statistics():
    import voxelmorph_b200 as vxm
    torch.manual_seed(11)
    m = vxm.networks.VxmDenseProbabilistic((16, 16, 16), nb_unet_features=[[16, 32], [32, 32, 64]])
    w = m.log_sigma.weight.detach().double()
    n = w.numel()                                         # 3 * 64 * 27
    assert abs(float(w.mean())) <= 5 * 1e-10 / n ** 0.5
    assert abs(float(w.std()) / 1e-10 - 1) <= 5 * (0.5 / n) ** 0.5


def test_wrappers_still_refuse_use_probs():
    import voxelmorph_b200 as vxm
    with pytest.raises(NotImplementedError, match="Flow variance"):
        vxm.networks.VxmDense((16, 16, 16), use_probs=True)
    with pytest.raises(NotImplementedError, match="Flow variance"):
        vxm.networks.TemplateCreation((16, 16, 16), use_probs=True)
    with pytest.raises(NotImplementedError, match="Flow variance"):
        vxm.networks.VxmDenseSemiSupervisedSeg((16, 16, 16), nb_labels=2, use_probs=True)


def test_kl_and_mse_surface():
    import voxelmorph_b200 as vxm
    assert vxm.losses.MSE().image_sigma == 1.0 and vxm.losses.MSE(0.02).image_sigma == 0.02
    with pytest.raises(vxm._lib.VxmError, match="flow_vol_shape"):
        vxm.losses.KL(10, flow_vol_shape=(8, 8, 8)).loss(None, torch.zeros(1, 6, 8, 8, 9))
    with pytest.raises(vxm._lib.VxmError):
        vxm.losses.KL(10).loss(None, torch.zeros(1, 6, 8, 8, 8))          # CPU tensors: no fallback
