"""Freeze outputs of the UNMODIFIED reference (voxelmorph at $VXM_REFERENCE_ROOT, torch CPU fp32)
into tests/golden/*.npz.

TEST INFRASTRUCTURE ONLY (needs the reference tree, see oracle/ref_import.py):

    VXM_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden

Inputs come from oracle/cases.py (seeded, exact arithmetic) and are stored beside the
outputs.  The fixtures pin (i) the restatements in oracle/spec_np.py and oracle/ref_torch.py
(`pytest -m "not gpu"`) and (ii) the CUDA kernels (`pytest -m gpu`).
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import cases, ref_import, ref_torch  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SMALL_FEATS = [[4, 8, 8, 8], [8, 8, 8, 8, 8, 4, 4]]


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def save_split(name, out, parts=2):
    """tests/golden/<name>.npz and <name>.part2.npz ...: the arrays dealt round-robin over `parts` files, each well under
    1 MB (tests/conftest.py's `golden` fixture merges them)."""
    keys = list(out)
    for p in range(parts):
        fn = name + (".npz" if p == 0 else ".part%d.npz" % (p + 1))
        np.savez_compressed(os.path.join(GOLD, fn), **{k: out[k] for k in keys[p::parts]})


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    vxm = ref_import.import_reference()
    NCC = ref_import.reference_ncc_class(vxm)
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(8)

    # ---- layers -------------------------------------------------------------------------
    shape = (12, 20, 16)
    out = {}
    src = np.concatenate([cases.smooth_volume(s, shape) for s in (1, 2, 3)], axis=1)
    src = np.concatenate([src, src[:, ::-1] * np.float32(0.5)], axis=0)           # (2,3,...)
    flow = np.concatenate([cases.smooth_field(11, 3, shape, scale=4.0),
                           cases.smooth_field(12, 3, shape, scale=9.0)], axis=0)  # (2,3,...) incl. OOB
    lab = np.concatenate([cases.label_volume(5, shape), cases.label_volume(6, shape)], axis=0)
    st = vxm.layers.SpatialTransformer(shape)
    stn = vxm.layers.SpatialTransformer(shape, mode="nearest")
    out.update(src=src, flow=flow, lab=lab,
               warp_lin=st(t(src), t(flow)).numpy(),
               warp_near=stn(t(lab), t(flow)).numpy())
    # integer shifts and exact .5 ties (round-half-even) for nearest
    tie = np.zeros((1, 3) + shape, np.float32)
    tie[:, 0] = 0.5
    tie[:, 1] = -1.5
    tie[:, 2] = 2.0
    out.update(tie_flow=tie, warp_near_tie=stn(t(lab[:1]), t(tie)).numpy(),
               warp_lin_tie=st(t(src[:1]), t(tie)).numpy())
    # 2-D
    s2 = (20, 28)
    src2 = cases.smooth_volume(21, s2)
    flow2 = cases.smooth_field(22, 2, s2, scale=3.0)
    out.update(src2=src2, flow2=flow2,
               warp2_lin=vxm.layers.SpatialTransformer(s2)(t(src2), t(flow2)).numpy(),
               warp2_near=vxm.layers.SpatialTransformer(s2, mode="nearest")(t(cases.label_volume(23, s2)), t(flow2)).numpy(),
               lab2=cases.label_volume(23, s2))
    # VecInt
    vel = cases.smooth_field(31, 3, shape, scale=6.0)
    for n in (0, 1, 4, 7):
        out["vecint_%d" % n] = vxm.layers.VecInt(shape, n)(t(vel)).numpy()
    out["vel"] = vel
    vel2 = cases.smooth_field(32, 2, s2, scale=5.0)
    out.update(vel2=vel2, vecint2_5=vxm.layers.VecInt(s2, 5)(t(vel2)).numpy())
    # ResizeTransform (even and odd sizes; down, up, identity)
    odd = cases.smooth_field(41, 3, (9, 11, 13), scale=2.0)
    out.update(odd=odd,
               resize_down=vxm.layers.ResizeTransform(2, 3)(t(flow)).numpy(),
               resize_up=vxm.layers.ResizeTransform(0.5, 3)(t(flow)).numpy(),
               resize_one=vxm.layers.ResizeTransform(1, 3)(t(flow)).numpy(),
               resize_down_odd=vxm.layers.ResizeTransform(2, 3)(t(odd)).numpy(),
               resize_up_odd=vxm.layers.ResizeTransform(0.5, 3)(t(odd)).numpy(),
               resize2_down=vxm.layers.ResizeTransform(2, 2)(t(flow2)).numpy(),
               resize2_up=vxm.layers.ResizeTransform(0.5, 2)(t(flow2)).numpy())
    save_split("layers", out)

    # ---- losses (values and autograd gradients w.r.t. y_pred) ----------------------------
    out = {}
    lshape = (20, 24, 28)
    I, J = cases.volume_pair(51, lshape, sigma=2.0)
    out.update(I=I, J=J)

    def with_grad(fn, pred):
        p = t(pred).clone().requires_grad_(True)
        v = fn(p)
        v.backward()
        return np.float32(v.item()), p.grad.numpy()

    out["ncc"], out["ncc_grad"] = with_grad(lambda p: NCC().loss(t(I), p), J)
    out["ncc5"], out["ncc5_grad"] = with_grad(lambda p: NCC(win=[5, 5, 5]).loss(t(I), p), J)
    out["mse"], out["mse_grad"] = with_grad(lambda p: vxm.losses.MSE().loss(t(I), p), J)
    fl = np.concatenate([cases.smooth_field(61, 3, (10, 12, 14), scale=3.0),
                         cases.smooth_field(62, 3, (10, 12, 14), scale=1.0)], axis=0)
    out["gflow"] = fl
    out["grad_l2"], out["grad_l2_grad"] = with_grad(lambda p: vxm.losses.Grad("l2", loss_mult=2).loss(None, p), fl)
    out["grad_l1"], out["grad_l1_grad"] = with_grad(lambda p: vxm.losses.Grad("l1").loss(None, p), fl)
    rng = np.random.Generator(np.random.PCG64(71))
    a = (rng.random((2, 5, 10, 12, 14), dtype=np.float32) > 0.6).astype(np.float32)
    b = rng.random((2, 5, 10, 12, 14), dtype=np.float32)
    out.update(dice_true=a, dice_pred=b)
    out["dice"], out["dice_grad"] = with_grad(lambda p: vxm.losses.Dice().loss(t(a), p), b)
    I2, J2 = cases.volume_pair(81, (40, 48), sigma=2.0)
    out.update(I2=I2, J2=J2)
    out["ncc2"], out["ncc2_grad"] = with_grad(lambda p: NCC().loss(t(I2), p), J2)
    np.savez_compressed(os.path.join(GOLD, "losses.npz"), **out)

    # ---- VxmDense: forward outputs + one training step, several ctor variants -------------
    variants = {
        "default3d": dict(inshape=(32, 32, 48)),
        "small3d": dict(inshape=(16, 32, 16), nb_unet_features=SMALL_FEATS),
        "nodiffeo3d": dict(inshape=(16, 16, 16), nb_unet_features=SMALL_FEATS, int_steps=0),
        "bidir_full3d": dict(inshape=(16, 16, 16), nb_unet_features=SMALL_FEATS, bidir=True, int_downsize=1),
        "halfres3d": dict(inshape=(16, 16, 32), nb_unet_features=SMALL_FEATS, unet_half_res=True),
        "intfeat3d": dict(inshape=(16, 16, 16), nb_unet_features=4, nb_unet_levels=3, unet_feat_mult=2,
                          nb_unet_conv_per_level=2),
        "config1_2d": dict(inshape=(64, 64), int_steps=0),
        "diffeo2d": dict(inshape=(32, 48), nb_unet_features=SMALL_FEATS, int_steps=5),
    }
    out = {}
    for name, kw in variants.items():
        model = vxm.networks.VxmDense(**kw)
        cfg = dict(model.config)
        sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2)   # trained-like flow scale
        model.load_state_dict(sd, strict=False)
        shape = kw["inshape"]
        s, g = cases.volume_pair(91, shape, sigma=1.5)
        with torch.no_grad():
            tr = model(t(s), t(g))
            rg = model(t(s), t(g), registration=True)
        for i, y in enumerate(tr):
            out["%s/train%d" % (name, i)] = y.numpy()
        out["%s/reg_flow" % name] = rg[1].numpy()
        # one training step exactly as scripts/torch/train.py:204-220 (NCC for 3-D, MSE for config 1)
        model.train()
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)
        nd = len(shape)
        img = NCC().loss if (nd == 3 and name != "nodiffeo3d") else vxm.losses.MSE().loss
        losses = [img, img] if cfg["bidir"] else [img]
        weights = [0.5, 0.5] if cfg["bidir"] else [1]
        losses += [vxm.losses.Grad("l2", loss_mult=cfg["int_downsize"]).loss]
        weights += [0.01]
        y_true = [t(g), t(s), None] if cfg["bidir"] else [t(g), None]
        y_pred = model(t(s), t(g))
        loss = 0
        for n, fn in enumerate(losses):
            loss = loss + fn(y_true[n], y_pred[n]) * weights[n]
        opt.zero_grad()
        loss.backward()
        out["%s/loss" % name] = np.float32(loss.item())
        for k, p in model.named_parameters():
            if k in ("flow.weight", "flow.bias", "unet_model.encoder.0.0.main.weight",
                     "unet_model.decoder.0.0.main.weight", "unet_model.remaining.0.main.bias"):
                out["%s/grad/%s" % (name, k)] = p.grad.numpy().copy()
        opt.step()
        for k in ("flow.weight", "unet_model.encoder.0.0.main.weight"):
            out["%s/after/%s" % (name, k)] = dict(model.named_parameters())[k].detach().numpy().copy()
    save_split("vxmdense", out)

    # ---- full-size nearest-neighbour label warp: digest only (inputs regenerate exactly) ---
    full = (160, 192, 224)
    lab = cases.label_volume(101, full)
    flow = cases.smooth_field(102, 3, full, scale=8.0)
    moved = vxm.layers.SpatialTransformer(full, mode="nearest")(t(lab), t(flow)).numpy()
    lin = vxm.layers.SpatialTransformer(full)(t(cases.smooth_volume(103, full)), t(flow)).numpy()
    digests = dict(nearest_full_sha256=sha(moved), nearest_full_sum=float(moved.astype(np.float64).sum()),
                   lab_sha256=sha(lab), flow_sha256=sha(flow),
                   linear_full_sum=float(lin.astype(np.float64).sum()),
                   linear_full_abs_sum=float(np.abs(lin).astype(np.float64).sum()))
    # a crop of the real scan / segmentation shipped with the reference (data, not code)
    d = os.path.join(ref_import.REFERENCE_ROOT, "data")
    if os.path.isfile(os.path.join(d, "test_scan.npz")):
        seg = np.load(os.path.join(d, "test_scan.npz"))["seg"].astype(np.float32)
        crop = seg[48:80, 64:112, 80:120][None, None]
        cflow = cases.smooth_field(104, 3, crop.shape[2:], scale=5.0)
        cm = vxm.layers.SpatialTransformer(crop.shape[2:], mode="nearest")(t(crop), t(cflow)).numpy()
        np.savez_compressed(os.path.join(GOLD, "realseg_crop.npz"), seg=crop.astype(np.uint8),
                            flow=cflow, moved=cm.astype(np.uint8))
    import json
    with open(os.path.join(GOLD, "digests.json"), "w") as f:
        json.dump(digests, f, indent=1)
    print("golden written to", GOLD)
    for fn in sorted(os.listdir(GOLD)):
        print("  %-24s %8.1f KB" % (fn, os.path.getsize(os.path.join(GOLD, fn)) / 1024))


if __name__ == "__main__":
    main()
