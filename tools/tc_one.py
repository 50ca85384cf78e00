"""Run one tensor-core conv layer a few times (for a profiler)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from voxelmorph_b200 import tc
dev = torch.device("cuda:0")
name = sys.argv[1] if len(sys.argv) > 1 else "rem1"
cfg = {"rem0": ((160, 192, 224), 32, 16, True, 32), "rem1": ((160, 192, 224), 32, 0, False, 16),
       "rem2": ((160, 192, 224), 16, 0, False, 16)}[name]
shape, Ca, Cb, up, Cout = cfg
D, H, W = shape
ash = (D // 2, H // 2, W // 2) if up else shape
xa = torch.randn((1,) + ash + (Ca,), device=dev).to(torch.bfloat16)
xb = torch.randn((1,) + shape + (Cb,), device=dev).to(torch.bfloat16) if Cb else None
w = torch.randn((Cout, Ca + Cb, 3, 3, 3), device=dev) * 0.05
wpk, cp = tc.pack_weights_t(w, variant="s")
b = torch.zeros(Cout, device=dev)
gz = torch.randn((1,) + shape + (Cout,), device=dev).to(torch.bfloat16)
for _ in range(3):
    tc.conv_fwd_t(xa, xb, wpk, cp, b, Cout, 3, up=up, slope=0.2)
    tc.conv_wgrad(xa, xb, gz, Ca + Cb, Cout, 3, up=up)
torch.cuda.synchronize()
