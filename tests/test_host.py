"""CPU tests of the host side: the C-ABI library loads and exports every symbol include/vxm_b200.h
declares, the module surface / config / state_dict / checkpoint contract (BASELINE config 1 'plumbing'),
loud failure without CUDA, and the data-parallel logic under gloo with world_size 2."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_oracle import VARIANTS, full_cfg


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "vxm_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(vxm_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    import voxelmorph_b200 as vxm
    lib = vxm._lib.load()
    syms = declared_symbols()
    assert len(syms) >= 29
    for s in syms:
        assert hasattr(lib, s), s
        assert s in vxm._lib.SIGNATURES, "no ctypes signature for %s" % s
    assert sorted(vxm._lib.SIGNATURES) == syms
    assert b"sm_90a" in lib.vxm_version()
    # pure host arithmetic entry points work without a GPU
    assert lib.vxm_vecint_workspace_bytes(1, 80, 96, 112, 3, 7) == 80 * 96 * 112 * 3 * 4
    assert lib.vxm_reduce_workspace_bytes() > 0


def test_argument_errors_are_reported_not_thrown():
    import voxelmorph_b200 as vxm
    lib = vxm._lib.load()
    rc = lib.vxm_warp_fwd(None, None, None, 1, 1, 4, 4, 4, 4, 4, 4, 5, 0, 0, None)   # nd = 5
    assert rc == -1 and "nd must be 2 or 3" in vxm._lib.last_error()
    rc = lib.vxm_vecint_fwd(None, None, None, None, 1, 4, 4, 4, 3, -1, 0, None)
    assert rc == -1 and "nsteps should be >= 0" in vxm._lib.last_error()
    rc = lib.vxm_ncc_fwd(None, None, None, None, None, 1, 8, 8, 8, 4, 4, 4, None)     # even window
    assert rc == -3


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_module_surface_matches_reference_contract(name):
    import voxelmorph_b200 as vxm
    from oracle import ref_torch
    kw = VARIANTS[name]
    cfg = full_cfg(kw)
    m = vxm.networks.VxmDense(**kw)
    assert m.config == cfg
    sd_ref = ref_torch.init_state_dict(cfg)
    sd = m.state_dict()
    assert set(sd) == set(sd_ref)                       # reference key names, no .grid buffers
    for k in sd:
        assert tuple(sd[k].shape) == tuple(sd_ref[k].shape), k
    assert (m.resize is None) == (cfg["unet_half_res"] or cfg["int_steps"] == 0 or cfg["int_downsize"] == 1)
    assert (m.integrate is None) == (cfg["int_steps"] == 0)
    assert isinstance(m.transformer, vxm.layers.SpatialTransformer) and hasattr(m.unet_model, "final_nf")
    assert float(m.flow.weight.abs().max()) < 1e-3 and float(m.flow.bias.abs().max()) == 0.0
    assert len(list(m.parameters())) == len(sd_ref)


def test_config1_plumbing_cpu(tmp_path):
    """BASELINE config 1 (2-D 64x64, int_steps=0, MSE): constructor / config / save / load round trip on CPU,
    and a loud failure (no CPU fallback) when the forward is attempted without CUDA."""
    import voxelmorph_b200 as vxm
    m = vxm.networks.VxmDense((64, 64), int_steps=0)
    assert sum(p.numel() for p in m.parameters()) == 109170
    p = str(tmp_path / "c1.pt")
    m.save(p)
    m2 = vxm.networks.VxmDense.load(p, "cpu")
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert torch.equal(a, b), k
    assert m2.config == m.config
    with pytest.raises(vxm._lib.VxmError, match="no CPU fallback"):
        m(torch.rand(1, 1, 64, 64), torch.rand(1, 1, 64, 64))
    with pytest.raises(vxm._lib.VxmError):
        vxm.losses.MSE().loss(torch.rand(1, 1, 64, 64), torch.rand(1, 1, 64, 64))


def test_constructor_errors():
    import voxelmorph_b200 as vxm
    with pytest.raises(NotImplementedError):
        vxm.networks.VxmDense((16, 16, 16), use_probs=True)
    with pytest.raises(ValueError):
        vxm.networks.Unet((16, 16), infeats=2, nb_features=8)                 # int features need nb_levels
    with pytest.raises(ValueError):
        vxm.networks.Unet((16, 16), infeats=2, nb_features=[[4], [4]], nb_levels=2)
    with pytest.raises(AssertionError):
        vxm.layers.VecInt((8, 8), -1)
    with pytest.raises(AssertionError):
        vxm.networks.VxmDense((4, 4, 4, 4))


def test_reference_checkpoint_loads(tmp_path):
    """A checkpoint in the reference's on-disk format (incl. `.grid` buffers) loads into the new model."""
    import voxelmorph_b200 as vxm
    from oracle import ref_torch
    cfg = full_cfg(dict(inshape=(16, 16, 16)))
    sd = ref_torch.init_state_dict(cfg, seed=3)
    sd["transformer.grid"] = torch.zeros(1, 3, 16, 16, 16)
    p = str(tmp_path / "ref.pt")
    torch.save({"config": cfg, "model_state": sd}, p)
    m = vxm.networks.VxmDense.load(p, "cpu")
    assert torch.equal(m.state_dict()["flow.weight"], sd["flow.weight"])


DIST_WORKER = r'''
import os, sys
sys.path.insert(0, os.environ["VXM_ROOT"])
import torch
import torch.distributed as dist
from voxelmorph_b200 import dist as vdist
world, rank, local = vdist.init_from_env(backend="gloo")
assert world == 2
items = vdist.shard_indices(5, world, rank)
assert items == ([0, 2, 4] if rank == 0 else [1, 3])
flat = torch.full((1000,), float(rank + 1))
vdist.broadcast_params(flat, src=0)
assert float(flat[0]) == 1.0
grad = torch.full((1000,), float(rank + 1))
vdist.allreduce_grads(grad)
assert float(grad[0]) == 3.0                      # SUM over ranks; 1/world is applied by the optimizer
m = vdist.max_over_ranks(float(rank), torch.device("cpu"))
assert m == 1.0
dist.barrier()
open(os.path.join(os.environ["VXM_OUT"], "ok_%d" % rank), "w").write("ok")
'''


def test_data_parallel_logic_gloo_world2(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(DIST_WORKER)
    env = dict(os.environ, VXM_ROOT=ROOT, MASTER_ADDR="127.0.0.1", VXM_OUT=str(tmp_path))
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "ok_0").exists() and (tmp_path / "ok_1").exists()


def test_bench_ranks_leave_together_under_torchrun(tmp_path):
    """bench.py's end-of-run rendezvous (store + os._exit, no collective): rank 0 finishes last, every rank exits 0 and
    nothing after `_leave` runs.  World size 3 on CPU with gloo."""
    import socket
    script = tmp_path / "leave.py"
    script.write_text(
        "import sys, time\n"
        "sys.path.insert(0, %r)\n"
        "import torch, torch.distributed as dist\n"
        "import bench\n"
        "dist.init_process_group('gloo')\n"
        "r, w = dist.get_rank(), dist.get_world_size()\n"
        "t = torch.ones(1); dist.all_reduce(t)\n"
        "if r == 0:\n"
        "    time.sleep(1.5)\n"
        "    print('RESULT', float(t), flush=True)\n"
        "bench._leave(w, r)\n"
        "print('NOT REACHED', flush=True)\n" % ROOT)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=240)
    assert p.returncode == 0, p.stderr[-2000:]
    assert "RESULT 3.0" in p.stdout and "NOT REACHED" not in p.stdout
