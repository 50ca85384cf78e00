"""CPU tests of the surface targets of VxmDenseSemiSupervisedPointCloud: the host helpers of pyutils and
generators.surf_semisupervised, run in float64 mode, must equal the unmodified reference exactly over six yields,
frozen into tests/golden/surf_generators.npz by oracle/make_golden_surf.py on the seeded synthetic blob dataset below."""
import hashlib
import os

import numpy as np
import pytest

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "surf_generators.npz")
STEPS = 6


def _blobs(rng, shape, centres, radii):
    """Label map with one ellipsoid per label (later labels drawn over earlier ones), jittered by up to one voxel."""
    grid = np.stack(np.meshgrid(*[np.arange(s, dtype=float) for s in shape], indexing="ij"), -1)
    seg = np.zeros(shape, np.int32)
    for li, (c, r) in enumerate(zip(centres, radii)):
        c = np.asarray(c, float) + rng.integers(-1, 2, len(shape))
        r = np.asarray(r, float) + rng.uniform(-0.5, 0.5, len(shape))
        seg[(((grid - c) / r) ** 2).sum(-1) <= 1.0] = li + 1
    return seg


LAYOUTS = {
    3: dict(shape=(14, 16, 18), centres=[(5, 5, 6), (9, 10, 11), (5, 11, 12)], radii=[(3, 3, 4), (3, 4, 4), (2, 3, 3)]),
    2: dict(shape=(22, 26), centres=[(7, 8), (14, 17), (6, 18)], radii=[(4, 5), (5, 6), (3, 4)]),
}


def make_dataset(tmp_path, nd, n=4):
    """(files, atlas_vol, atlas_seg): n subjects and an atlas; images are float32 smooth label intensities."""
    lay = LAYOUTS[nd]
    rng = np.random.default_rng(100 + nd)
    files = []
    for i in range(n + 1):
        seg = _blobs(rng, lay["shape"], lay["centres"], lay["radii"])
        vol = (seg * 0.25 + rng.uniform(0, 0.05, seg.shape)).astype(np.float32)
        if i == n:
            return files, vol, seg
        f = os.path.join(str(tmp_path), "surf%d_%02d.npz" % (nd, i))
        np.savez_compressed(f, vol=vol, seg=seg)
        files.append(f)


CASES = {
    "all_labels_3d": dict(nd=3, kw=dict(nb_surface_pts=60)),
    "sampled_labels_3d": dict(nd=3, kw=dict(nb_surface_pts=50, nb_labels_sample=2)),
    "unidir_2d": dict(nd=2, kw=dict(nb_surface_pts=40, surf_bidir=False)),
    "sampled_2d": dict(nd=2, kw=dict(nb_surface_pts=40, nb_labels_sample=1, smooth_seg_std=0.7)),
    "resize_3d": dict(nd=3, kw=dict(nb_surface_pts=30, sdt_vol_resize=0.5)),
    "align_segs_2d": dict(nd=2, kw=dict(nb_surface_pts=20, labels=[2], align_segs=True)),
}


def run_case(mod, tmp_path, case, steps=STEPS, seed=5, **extra):
    files, atlas_vol, atlas_seg = make_dataset(tmp_path, case["nd"])
    np.random.seed(seed)
    gen = mod.surf_semisupervised(files, atlas_vol, atlas_seg, **case["kw"], **extra)
    return [next(gen) for _ in range(steps)]


def flatten(yields):
    """{name: float64 array} of every yielded array, named yield / inputs|outputs / position."""
    out = {}
    for k, (ins, outs) in enumerate(yields):
        for side, arrays in (("in", ins), ("out", outs)):
            for j, a in enumerate(arrays):
                out["%d_%s%d" % (k, side, j)] = np.asarray(a).astype(np.float64)
    return out


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, np.float64).tobytes()).digest(), np.uint8)


def golden_entries(name, yields):
    """What the golden file keeps of one case: every array's shape and sha256 (of its float64 bytes), and the surface
    point arrays in full."""
    out = {}
    for key, a in flatten(yields).items():
        out["%s/%s/shape" % (name, key)] = np.asarray(a.shape, np.int64)
        out["%s/%s/sha256" % (name, key)] = digest(a)
        if a.ndim == 3 and a.shape[-1] in (3, 4) and "_in" in key:
            out["%s/%s/values" % (name, key)] = a
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_surf_semisupervised_equals_reference(tmp_path, name):
    from voxelmorph_b200 import generators
    gold = np.load(GOLDEN)
    yields = run_case(generators, tmp_path, CASES[name], sdt_dtype=np.float64, pts_dtype=np.float64,
                      zeros_dtype=np.float64, cache=generators.VolumeCache())
    got = golden_entries(name, yields)
    want = {k: gold[k] for k in gold.files if k.startswith(name + "/")}
    assert sorted(got) == sorted(want)
    for k in sorted(want):
        if k.endswith("/values"):
            np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    for k in sorted(want):
        assert np.array_equal(got[k], want[k]), k


def test_default_dtypes_are_float32(tmp_path):
    from voxelmorph_b200 import generators
    (ins, outs), = run_case(generators, tmp_path, CASES["all_labels_3d"], steps=1, cache=generators.VolumeCache())
    assert all(a.dtype == np.float32 for a in ins[2:] + outs[2:])
    ref, = run_case(generators, tmp_path, CASES["all_labels_3d"], steps=1, sdt_dtype=np.float64,
                    pts_dtype=np.float64, zeros_dtype=np.float64, cache=generators.VolumeCache())
    for a, b in zip(ins[2:], ref[0][2:]):
        np.testing.assert_array_equal(a, b.astype(np.float32))


def test_helpers_on_worked_cases():
    from voxelmorph_b200 import pyutils
    bw = np.zeros((7, 7), bool)
    bw[1:3, 1:3] = True      # 4 voxels
    bw[4:7, 4:7] = True      # 9 voxels
    assert pyutils.extract_largest_vol(bw).sum() == 9
    sdt = pyutils.signed_dist_trf(bw)
    assert sdt[5, 5] == -2 and sdt[0, 1] == 1 and not np.any(sdt == 0)
    assert list(pyutils.get_surface_pts_per_label(10, [0.26, 0.26, 0.48])) == [3, 3, 4]
