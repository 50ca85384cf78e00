"""Freeze the UNMODIFIED reference's doubled VoxelMorph U-Net (`--enc 32 64 64 64 --dec 64 64 64 64 64 32 32`, 64-channel
layers and 128-channel concatenations) at a small size into tests/golden/wide.npz: forward outputs, registration flow and
one training step (NCC + Grad, Adam) as scripts/torch/train.py takes it.  tests/test_wide_unet_oracle.py pins
oracle/ref_torch.py to it on the CPU; tests/test_gpu_wide_unet.py checks the bf16x3 engine against it.

TEST INFRASTRUCTURE ONLY: needs the reference tree (VXM_REFERENCE_ROOT, see oracle/ref_import.py).

    VXM_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_wide.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import cases, ref_import, ref_torch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "wide.npz")
KW = dict(inshape=(16, 16, 32), nb_unet_features=[[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]])
GRADS = ("flow.weight", "flow.bias", "unet_model.encoder.0.0.main.weight", "unet_model.encoder.2.0.main.weight",
         "unet_model.decoder.1.0.main.bias", "unet_model.remaining.0.main.bias")


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def main():
    vxm = ref_import.import_reference()
    NCC = ref_import.reference_ncc_class(vxm)
    torch.manual_seed(0)
    model = vxm.networks.VxmDense(**KW)
    cfg = dict(model.config)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2)
    model.load_state_dict(sd, strict=False)
    s, g = cases.volume_pair(91, KW["inshape"], sigma=1.5)
    out = {}
    with torch.no_grad():
        tr = model(t(s), t(g))
        rg = model(t(s), t(g), registration=True)
    for i, y in enumerate(tr):
        out["train%d" % i] = y.numpy()
    out["reg_flow"] = rg[1].numpy()
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    y_pred = model(t(s), t(g))
    loss = NCC().loss(t(g), y_pred[0]) + 0.01 * vxm.losses.Grad("l2", loss_mult=cfg["int_downsize"]).loss(None, y_pred[1])
    opt.zero_grad()
    loss.backward()
    out["loss"] = np.float32(loss.item())
    params = dict(model.named_parameters())
    for k in GRADS:
        out["grad/%s" % k] = params[k].grad.numpy().copy()
    opt.step()
    out["after/flow.weight"] = params["flow.weight"].detach().numpy().copy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
