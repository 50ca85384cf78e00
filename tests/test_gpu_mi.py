"""MutualInformation on the GPU (csrc/mi.cu): loss and gradients against the fp64 closed form of tests/mi_ref.py fed the
same fp32 inputs, one-sided calls, bit-reproducibility, peak memory at full size, the graphed training step, and a
cross-contrast registration.  Run with -s to see every measured error next to its bound."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

from mi_ref import make_case, mi_closed_form
from test_mi_oracle import CASES
from test_oracle import full_cfg

pytestmark = pytest.mark.gpu

LOSS_TOL = 1e-6      # absolute, on the loss (the measured maximum is 5.4e-8)
GRAD_TOL = 5e-5      # voxelwise, relative to max |g64| (floored at 1 / V, the scale of one voxel's share)
FULL = (160, 192, 224)


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


def _kw_to_loss(kw):
    kw = dict(kw)
    if "alpha" in kw:
        kw["soft_bin_alpha"] = kw.pop("alpha")
    return kw


def _run(vxm, cuda, x, y, kw, sides=(True, True)):
    X = torch.from_numpy(x).to(cuda).requires_grad_(sides[0])
    Y = torch.from_numpy(y).to(cuda).requires_grad_(sides[1])
    loss = vxm.losses.MutualInformation(**_kw_to_loss(kw)).loss(X, Y)
    loss.backward()
    torch.cuda.synchronize()
    return (float(loss), None if X.grad is None else X.grad.double().cpu().numpy(),
            None if Y.grad is None else Y.grad.double().cpu().numpy())


def _check(name, got, ref, V, sides=(True, True)):
    l, gx, gy = got
    l64, gx64, gy64 = ref
    dl = abs(l - l64)
    msg = "[mi %s] loss %.7f (fp64 %.7f) |dl| %.2e (bound %.0e)" % (name, l, l64, dl, LOSS_TOL)
    assert np.isfinite(l)
    assert dl <= LOSS_TOL, msg
    for side, g, g64 in (("y_true", gx, gx64), ("y_pred", gy, gy64)):
        want = sides[0] if side == "y_true" else sides[1]
        if not want:
            assert g is None
            continue
        assert np.all(np.isfinite(g))
        scale = max(float(np.abs(g64).max()), 1.0 / V)
        err = float(np.abs(g - g64).max()) / scale
        msg += " | %s %.2e" % (side, err)
        assert err <= GRAD_TOL, msg
    print("\n" + msg + " (bound %.0e)" % GRAD_TOL)


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0] for c in CASES])
def test_mi_matches_fp64(vxm, cuda, idx):
    name, shape, n, kw, extra = CASES[idx]
    x, y = make_case(100 + idx, shape, n=n, **extra)
    _check(name, _run(vxm, cuda, x, y, kw), mi_closed_form(x, y, **kw), x[0].size)


ONE_SIDED = ["3d_b23_n3", "centres_alpha_clip", "ties", "2d_b64_n2"]


@pytest.mark.parametrize("name", ONE_SIDED)
@pytest.mark.parametrize("sides", [(False, True), (True, False)], ids=["y_true_detached", "y_pred_detached"])
def test_mi_one_sided(vxm, cuda, name, sides):
    idx = [c[0] for c in CASES].index(name)
    _, shape, n, kw, extra = CASES[idx]
    x, y = make_case(100 + idx, shape, n=n, **extra)
    _check(name + str(sides), _run(vxm, cuda, x, y, kw, sides), mi_closed_form(x, y, **kw), x[0].size, sides)


@pytest.fixture(scope="module")
def full_pair():
    # skull-stripped look: millions of voxels tied at 0 in both images
    return make_case(2024, FULL, n=1, ties=True)


@pytest.mark.parametrize("bins", [16, 32])
def test_mi_full_size(vxm, cuda, full_pair, bins):
    x, y = full_pair
    _check("full B=%d" % bins, _run(vxm, cuda, x, y, dict(nb_bins=bins)),
           mi_closed_form(x, y, nb_bins=bins, chunk=1 << 20), x[0].size)


def test_mi_bit_reproducible(vxm, cuda, full_pair):
    small = make_case(5, (9, 11, 13), n=3, ties=True)
    for (x, y), kw in ((full_pair, dict(nb_bins=32)), (small, dict(nb_bins=23)), (small, dict(nb_bins=7, min_clip=0.1))):
        a = _run(vxm, cuda, x, y, kw)
        b = _run(vxm, cuda, x, y, kw)
        assert a[0] == b[0]
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_mi_peak_memory_full_size(vxm, cuda, full_pair):
    x, y = full_pair
    X = torch.from_numpy(x).to(cuda).requires_grad_(True)
    Y = torch.from_numpy(y).to(cuda).requires_grad_(True)
    mi = vxm.losses.MutualInformation(nb_bins=32)
    mi.loss(X, Y).backward()             # warm the reduce workspace and the library
    X.grad = Y.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(cuda)
    torch.cuda.reset_peak_memory_stats(cuda)
    mi.loss(X, Y).backward()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated(cuda) - base - X.numel() * 4 - Y.numel() * 4
    print("\n[mi peak memory] %.2f MiB beyond the inputs and gradients (bound 64 MiB; [V, B] weights alone: %.0f MB)"
          % (extra / 2 ** 20, X.numel() * 32 * 4 / 1e6))
    assert extra < 64 * 2 ** 20


def test_graphed_mi_step_matches_eager(vxm, cuda, monkeypatch):
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
    cfg = full_cfg(kw)
    s, tr = cases.volume_pair(95, kw["inshape"], sigma=1.5)
    lo, hi = min(s.min(), tr.min()), max(s.max(), tr.max())
    s, tr = (s - lo) / (hi - lo), (tr - lo) / (hi - lo)   # MutualInformation's default bins assume [0, 1]
    S, T = (torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(cuda) for v in (s, tr))

    def make():
        m = vxm.networks.VxmDense(**kw)
        m.load_state_dict(ref_torch.init_state_dict(cfg, seed=5, flow_std=2e-2), strict=False)
        m.to(cuda).train()
        return m, vxm.optim.FusedAdam(m.parameters(), lr=1e-3)

    m1, o1 = make()
    eager = []
    for _ in range(3):
        o1.zero_grad()
        y, flow = m1(S, T)
        loss = vxm.losses.MutualInformation().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
        loss.backward()
        o1.step()
        eager.append(float(loss))
    m2, o2 = make()
    step = GraphedTrainStep(m2, o2, image_loss="mi", warmup=3).capture(S, T)
    graphed = [float(step(S, T)) for _ in range(3)]
    print("\n[graphed mi step] %s vs eager %s" % (graphed, eager))
    for i in range(3):
        assert abs(graphed[i] - eager[i]) <= 2e-3 * abs(eager[i]), (i, graphed, eager)


def _contrast_pair(golden):
    g = golden("realseg_crop")
    seg = g["seg"][0, 0, :, :, 4:36].astype(np.int64)     # 32 x 48 x 32: four U-Net levels
    moved = g["moved"][0, 0, :, :, 4:36].astype(np.int64)
    rng = np.random.default_rng(11)
    labels = np.unique(seg)
    lut_s, lut_t = np.zeros(256), np.zeros(256)
    lut_s[labels] = rng.uniform(0.15, 1.0, labels.size)
    lut_t[labels] = rng.uniform(0.15, 1.0, labels.size)    # an independent draw: no monotonic map between the two
    lut_s[0] = lut_t[0] = 0.0                                # background stays at 0 in both
    src = lut_s[seg]
    trg = np.clip(lut_t[moved] + 0.03 * rng.standard_normal(moved.shape), 0.0, 1.0)
    return seg, moved, src.astype(np.float32), trg.astype(np.float32)


def _train_and_dice(vxm, cuda, golden, image_loss, steps=200, lr=1e-3):
    seg, moved, src, trg = _contrast_pair(golden)
    torch.manual_seed(0)
    S = torch.from_numpy(src[None, None]).to(cuda)
    T = torch.from_numpy(trg[None, None]).to(cuda)
    model = vxm.networks.VxmDense(inshape=src.shape).to(cuda).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=lr)
    img = image_loss().loss
    grad = vxm.losses.Grad("l2", loss_mult=2).loss
    for _ in range(steps):
        opt.zero_grad()
        y, flow = model(S, T)
        loss = img(T, y) + 0.01 * grad(None, flow)
        loss.backward()
        opt.step()
    model.eval()
    with torch.no_grad():
        _, pos = model(S, T, registration=True)
        warp = vxm.layers.SpatialTransformer(src.shape, mode="nearest").to(cuda)
        wseg = warp(torch.from_numpy(seg[None, None].astype(np.float32)).to(cuda), pos)
    wseg = np.rint(wseg.cpu().numpy()[0, 0]).astype(np.int64)
    labels = [l for l in np.unique(moved) if l != 0 and (moved == l).sum() >= 50]
    before = float(np.mean(vxm.utils.dice(seg, moved, labels=labels)))
    after = float(np.mean(vxm.utils.dice(wseg, moved, labels=labels)))
    return before, after


def test_mi_registers_across_contrasts(vxm, cuda, golden):
    before, after = _train_and_dice(vxm, cuda, golden, vxm.losses.MutualInformation)
    _, ncc_after = _train_and_dice(vxm, cuda, golden, vxm.losses.NCC)
    print("\n[cross-contrast] mean label Dice: unregistered %.4f, MI + Grad %.4f, NCC + Grad %.4f (measurement)"
          % (before, after, ncc_after))
    # measured on an H100 80GB HBM3 at 700 W over two runs (training is not bit-reproducible): 0.6152 -> 0.6276 and
    # 0.6219 with MI (+0.012, +0.007), 0.5448 and 0.5375 with NCC; the bar keeps 3x headroom on the smaller gain
    assert after >= before + 0.002, (before, after)
