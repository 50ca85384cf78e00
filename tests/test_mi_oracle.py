"""CPU checks of the MutualInformation spec: the closed-form fp64 oracle (tests/mi_ref.py) against a literal torch-fp64
transcription of neurite's graph differentiated by autograd, and the constructor's defaults and refusals."""
import math

import numpy as np
import pytest

from mi_ref import default_alpha, make_case, mi_closed_form, mi_torch_graph

# (name, volume shape, N, loss kwargs, make_case kwargs)
CASES = [
    ("3d_b2", (7, 9, 11), 2, dict(nb_bins=2), {}),
    ("3d_b16", (7, 9, 11), 1, dict(nb_bins=16), {}),
    ("3d_b23_n3", (5, 7, 9), 3, dict(nb_bins=23), {}),
    ("3d_b64", (9, 7, 5), 2, dict(nb_bins=64), {}),
    ("2d_b16_n3", (13, 17), 3, dict(nb_bins=16), {}),
    ("2d_b23", (19, 11), 1, dict(nb_bins=23), {}),
    ("2d_b64_n2", (15, 21), 2, dict(nb_bins=64), {}),
    ("centres", (5, 9, 8), 2, dict(bin_centers=[0.0, 0.05, 0.15, 0.3, 0.5, 0.75, 1.0]), {}),
    ("centres_alpha_clip", (11, 13), 2, dict(bin_centers=[0.1, 0.2, 0.4, 0.45, 0.7, 0.9], alpha=80.0, min_clip=0.15,
                                              max_clip=0.85), {}),
    ("alpha", (7, 5, 9), 1, dict(nb_bins=16, alpha=60.0), {}),
    ("clip", (7, 5, 9), 2, dict(nb_bins=32, min_clip=0.2, max_clip=0.8), {}),
    ("ties", (9, 11, 7), 2, dict(nb_bins=16), dict(ties=True)),
    ("ties_2d_b23", (21, 19), 1, dict(nb_bins=23), dict(ties=True)),
    ("constant", (13, 17), 2, dict(nb_bins=16), dict(constant=True)),
    ("constant_3d_clip", (5, 6, 7), 1, dict(nb_bins=16, min_clip=0.1, max_clip=0.9), dict(constant=True)),
]


def _case(i, shape, n, extra):
    return make_case(100 + i, shape, n=n, **extra)


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0] for c in CASES])
def test_closed_form_matches_autograd_of_the_graph(idx):
    _, shape, n, kw, extra = CASES[idx]
    x, y = _case(idx, shape, n, extra)
    l1, gx1, gy1 = mi_closed_form(x, y, **kw)
    l2, gx2, gy2 = mi_torch_graph(x, y, **kw)
    V = x[0].size
    # relative to the loss (floored at 1, the scale of MI's summands) and to max|g| (floored at 1/V, the scale of one
    # voxel's share); a constant image's loss and gradients are pure epsilon effects, far below those scales
    assert abs(l1 - l2) <= 1e-12 * max(1.0, abs(l2))
    for g1, g2 in ((gx1, gx2), (gy1, gy2)):
        assert np.all(np.isfinite(g1))
        assert np.abs(g1 - g2).max() <= 1e-12 * max(np.abs(g2).max(), 1.0 / V)


def test_constant_image_gives_no_nan_and_no_gradient():
    x, y = make_case(7, (6, 7, 8), n=1, constant=True)
    loss, gx, gy = mi_closed_form(x, y, nb_bins=16)
    assert math.isfinite(loss) and abs(loss) < 1e-4
    assert np.all(gx == 0) and np.all(np.isfinite(gy))
    # both sides constant
    loss, gx, gy = mi_closed_form(x, x.copy(), nb_bins=16)
    assert math.isfinite(loss) and np.all(gx == 0) and np.all(gy == 0)


def test_oracle_chunking_is_invisible():
    x, y = make_case(9, (10, 12, 14), n=2)
    a = mi_closed_form(x, y, nb_bins=23, chunk=1 << 20)
    b = mi_closed_form(x, y, nb_bins=23, chunk=97)
    assert abs(a[0] - b[0]) <= 1e-13
    for u, v in zip(a[1:], b[1:]):
        assert np.abs(u - v).max() <= 1e-13 * np.abs(u).max()


def test_defaults_and_refusals():
    import voxelmorph_b200 as vxm
    from voxelmorph_b200._lib import VxmError

    mi = vxm.losses.MutualInformation()
    assert mi.nb_bins == 16 and mi.soft_bin_alpha == pytest.approx(450.0, rel=1e-12)
    assert mi.min_clip == -np.inf and mi.max_clip == np.inf and mi.bin_centers is None
    assert vxm.losses.MutualInformation(nb_bins=32).soft_bin_alpha == pytest.approx(1922.0, rel=1e-12)
    c = [0.0, 0.1, 0.3, 0.6]
    m = vxm.losses.MutualInformation(bin_centers=c)
    assert m.nb_bins == 4 and m.soft_bin_alpha == pytest.approx(default_alpha(bin_centers=c), rel=1e-12)
    assert m.soft_bin_alpha == pytest.approx(1.0 / (2.0 * (0.5 * 0.2) ** 2), rel=1e-12)
    assert vxm.losses.MutualInformation(nb_bins=5, soft_bin_alpha=3.0, min_clip=0, max_clip=1).soft_bin_alpha == 3.0
    assert vxm.losses.MutualInformation(nb_bins=2).nb_bins == 2
    assert vxm.losses.MutualInformation(nb_bins=64).nb_bins == 64
    for kw in (dict(bin_centers=[0.0, 1.0], nb_bins=2), dict(nb_bins=1), dict(nb_bins=65), dict(bin_centers=[0.5]),
               dict(bin_centers=np.linspace(0, 1, 65)), dict(bin_centers=[0.0, np.nan, 1.0]),
               dict(bin_centers=[0.0, np.inf]), dict(nb_bins=8, soft_bin_alpha=float("nan")),
               dict(nb_bins=8, soft_bin_alpha=-1.0), dict(bin_centers=[0.5, 0.5, 0.5])):
        with pytest.raises(VxmError):
            vxm.losses.MutualInformation(**kw)


def test_reached_through_the_voxelmorph_package():
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import os; os.environ['VXM_BACKEND'] = 'pytorch'\n"
            "import voxelmorph as vxm, voxelmorph_b200\n"
            "assert vxm.losses.MutualInformation is voxelmorph_b200.losses.MutualInformation\n"
            "assert vxm.losses.MutualInformation().soft_bin_alpha == 450.0\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_refuses_cpu_tensors():
    import torch
    import voxelmorph_b200 as vxm
    from voxelmorph_b200._lib import VxmError

    with pytest.raises(VxmError):
        vxm.losses.MutualInformation().loss(torch.zeros(1, 1, 4, 4), torch.zeros(1, 1, 4, 4))


def test_c_declarations_match_the_bindings():
    import os
    import re
    from voxelmorph_b200 import _lib

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vxm_b200.h")).read()
    for name in ("vxm_mi_workspace_bytes", "vxm_mi_fwd", "vxm_mi_bwd"):
        m = re.search(r"\n(?:int|size_t) %s\(([^;]*)\);" % name, hdr)
        assert m, name
        nargs = len([a for a in m.group(1).split(",") if a.strip() and a.strip() != "void"])
        assert nargs == len(_lib.SIGNATURES[name][1]), name
