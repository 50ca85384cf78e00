"""Localise non-finite gradients in the bf16 engine: per convolution launch, then per parameter."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
import voxelmorph_b200 as vxm
from voxelmorph_b200 import tc
from oracle import cases, ref_torch
from test_oracle import full_cfg
dev = torch.device("cuda:0")
F16 = [[16, 16, 16, 16], [16, 16, 16, 16, 16, 16, 16]]
kw = dict(inshape=(16, 32, 32), nb_unet_features=F16)
cfg = full_cfg(kw)
sd = ref_torch.init_state_dict(cfg, seed=77, flow_std=2e-2)
s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
S, T = torch.from_numpy(s).to(dev), torch.from_numpy(tr).to(dev)
poison = torch.full((1 << 28,), float("nan"), device=dev); del poison   # NaN-poison the caching allocator

# wrap the conv entry points to check every output for NaN/Inf
def wrap(name):
    orig = getattr(tc, name)
    def f(*a, **k):
        out = orig(*a, **k)
        outs = out if isinstance(out, tuple) else (out,)
        bad = [int((~torch.isfinite(o.float())).sum()) for o in outs if o is not None]
        if any(bad):
            shp = [tuple(x.shape) for x in a[:3] if torch.is_tensor(x)]
            print("   NONFINITE in %s: %s inputs %s kwargs %s" % (name, bad, shp, {kk: (vv if not torch.is_tensor(vv) else tuple(vv.shape)) for kk, vv in k.items()}))
            ins = [int((~torch.isfinite(x.float())).sum()) for x in a[:3] if torch.is_tensor(x)]
            print("      non-finite counts of inputs:", ins)
        return out
    setattr(tc, name, f)
for n in ("conv_fwd_t", "conv_fwd_blocked", "conv_wgrad"):
    wrap(n)

model = vxm.networks.VxmDense(**kw)
model.load_state_dict(sd, strict=False)
model.to(dev).train()
out = model(S, T)
loss = out[-1].square().sum() + out[0].square().sum()
loss.backward()
torch.cuda.synchronize()
nbad = {k: int((~torch.isfinite(p.grad)).sum()) for k, p in model.named_parameters()}
print("nonfinite grads:", {k: v for k, v in nbad.items() if v})
