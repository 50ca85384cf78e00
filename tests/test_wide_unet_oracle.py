"""CPU tests of the wide-U-Net support: the oracle restatement pinned to the unmodified reference's doubled VoxelMorph
(tests/golden/wide.npz, oracle/make_golden_wide.py), the engine selection that stays as it was, and the channel blocks the
tensor-core engine splits wide layers into."""
import numpy as np
import torch

from oracle import cases, ref_torch

from test_oracle import full_cfg

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]
KW = dict(inshape=(16, 16, 32), nb_unet_features=DOUBLED)


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def test_doubled_model_restatement_against_reference(golden):
    g = golden("wide")
    cfg = full_cfg(KW)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2)
    s, tr = cases.volume_pair(91, cfg["inshape"], sigma=1.5)
    with torch.no_grad():
        out = ref_torch.vxm_forward(sd, cfg, t(s), t(tr))
        reg = ref_torch.vxm_forward(sd, cfg, t(s), t(tr), registration=True)
    for i, y in enumerate(out):
        assert np.array_equal(y.numpy(), g["train%d" % i]), i
    assert np.array_equal(reg[1].numpy(), g["reg_flow"])
    # one training step: loss and gradients of the restatement (autograd through the same ops)
    sdc = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    y, flow = ref_torch.vxm_forward(sdc, cfg, t(s), t(tr))
    loss = ref_torch.ncc_loss(t(tr), y) + 0.01 * ref_torch.grad_loss(flow, "l2", 2)
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) <= 1e-6 * abs(float(g["loss"]))
    for k in [k[5:] for k in g if k.startswith("grad/")]:
        ref = t(g["grad/" + k]).double()
        assert float((sdc[k].grad.double() - ref).abs().max() / ref.abs().max()) <= 1e-5, k


def test_tc_default_still_picks_fp32_for_wide_models():
    import voxelmorph_b200 as vxm
    from voxelmorph_b200 import ops
    prev = ops._default_engine
    try:
        ops.set_default_engine("tc")
        for kw in (KW, dict(inshape=(32, 32, 48), nb_unet_features=16, nb_unet_levels=3, unet_feat_mult=2),
                   dict(inshape=(32, 32, 32), nb_unet_features=[[16, 32, 32, 32], [32, 16, 32, 32, 32, 16, 16]])):   # 16 + 32 concat
            assert ops.resolve_engine(vxm.networks.VxmDense(**kw)) == "f32"
        assert ops.resolve_engine(vxm.networks.VxmDense((32, 32, 32))) == "bf16x3"
    finally:
        ops.set_default_engine(prev)


def test_channel_blocks():
    from voxelmorph_b200 import tc
    assert tc.conv_blocks(32, 32, 32, 3) is None                       # today's layers: one launch
    assert tc.conv_blocks(48, 0, 32, 3) is None
    assert tc.conv_blocks(32, 0, 64, 3) is None                        # 32 -> 64 fits one launch
    assert tc.conv_blocks(64, 0, 64, 1) is None                        # 2-D 64 -> 64 too
    # 3-D 64 -> 64: two 32-channel output blocks at channel offsets 0 and 32 of one tensor
    assert tc.conv_blocks(64, 0, 64, 3) == (((2, 0, 64),), ((0, 32, 0, 0), (32, 32, 0, 32)))
    # 64 + 32 -> 64: one K block per source, the 64-channel source last
    assert tc.conv_blocks(64, 32, 64, 3)[0] == ((1, 64, 32), (0, 0, 64))
    assert tc.conv_blocks(64, 64, 64, 1) == (((0, 0, 64), (1, 64, 64)), ((0, 64, 0, 0),))
    # dgrad of a 96 -> 64 concatenation: 64 + 32 outputs into two tensors
    assert tc.conv_blocks(64, 0, 96, 3, 64)[1] == ((0, 32, 0, 0), (32, 32, 0, 32), (64, 32, 1, 0))
    assert tc.conv_blocks(32, 0, 96, 3, 64)[1] == ((0, 64, 0, 0), (64, 32, 1, 0))
