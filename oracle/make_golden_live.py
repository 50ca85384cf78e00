"""Freeze the outputs of the UNMODIFIED reference that the "live" pins compare against (tests/test_oracle_vs_reference.py,
tests/test_generators.py::test_matches_live_reference, tests/test_utils.py::test_against_live_reference) into
tests/golden/reference_live.npz, so that those comparisons run wherever the repository does.

TEST INFRASTRUCTURE ONLY: needs the reference tree (VXM_REFERENCE_ROOT, see oracle/ref_import.py).

    VXM_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_live.py
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import cases, ref_import, ref_torch  # noqa: E402
import test_generators as tg  # noqa: E402
import test_utils as tu  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_live.npz")


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def flatten(item, out):
    """Nested lists / tuples of arrays -> list of arrays (in order) + a structure string."""
    if isinstance(item, (list, tuple)):
        return "[" + ",".join(flatten(x, out) for x in item) + "]"
    out.append(np.asarray(item))
    return "a"


def main():
    vxm = ref_import.import_reference()
    g = {}
    # tests/test_oracle_vs_reference.py::test_layers_live
    shape = (10, 14, 12)
    src = cases.smooth_volume(1, shape)
    flow = cases.smooth_field(2, 3, shape, scale=5.0)
    lab = cases.label_volume(3, shape)
    g["layers/warp_lin"] = vxm.layers.SpatialTransformer(shape)(t(src), t(flow)).numpy()
    g["layers/warp_near"] = vxm.layers.SpatialTransformer(shape, mode="nearest")(t(lab), t(flow)).numpy()
    g["layers/vecint5"] = vxm.layers.VecInt(shape, 5)(t(flow)).numpy()
    for vr in (2, 0.5):
        g["layers/resize_%g" % vr] = vxm.layers.ResizeTransform(vr, 3)(t(flow)).numpy()
    # test_losses_live
    NCC = ref_import.reference_ncc_class(vxm)
    I, J = cases.volume_pair(7, (16, 20, 18))
    g["losses/ncc"] = np.float32(NCC().loss(t(I), t(J)).item())
    f = cases.smooth_field(8, 3, (8, 10, 12), scale=2.0)
    g["losses/grad_l2"] = np.float32(vxm.losses.Grad("l2", loss_mult=2).loss(None, t(f)).item())
    g["losses/mse"] = np.float32(vxm.losses.MSE().loss(t(I), t(J)).item())
    # test_network_live
    kw = dict(inshape=(16, 16, 32), nb_unet_features=[[4, 8, 8, 8], [8, 8, 8, 8, 8, 4, 4]], bidir=True)
    m = vxm.networks.VxmDense(**kw)
    sd = ref_torch.init_state_dict(m.config, seed=5, flow_std=2e-2)
    m.load_state_dict(sd, strict=False)
    s, tg_ = cases.volume_pair(9, kw["inshape"])
    with torch.no_grad():
        outs = m(t(s), t(tg_))
    for i, o in enumerate(outs):
        g["network/out%d" % i] = o.numpy()
    # test_eval_helpers_live and tests/test_utils.py::test_against_live_reference
    nd_mod = sys.modules["pystrum.pynd.ndutils"]
    if not hasattr(nd_mod, "volsize2ndgrid"):
        nd_mod.volsize2ndgrid = lambda volshape: np.meshgrid(*[np.arange(s) for s in volshape], indexing="ij")
    utils = vxm.py.utils
    rng = np.random.RandomState(5)
    a, b = rng.randint(0, 5, size=(9, 10, 11)), rng.randint(0, 6, size=(9, 10, 11))
    g["eval/dice"] = np.asarray(utils.dice(a, b))
    g["eval/dice_labels"] = np.asarray(utils.dice(a, b, labels=[1, 3, 7], include_zero=True))
    for shp in ((7, 9), (6, 7, 8)):
        disp = np.moveaxis(cases.smooth_field(11, len(shp), shp, scale=3.0)[0], 0, -1).astype(np.float64)
        g["eval/jacdet_%dd" % len(shp)] = utils.jacobian_determinant(disp)
    rng = np.random.RandomState(2)
    a, b = rng.randint(0, 5, size=(9, 10, 11)), rng.randint(0, 5, size=(9, 10, 11))
    g["utils/dice"] = np.asarray(utils.dice(a, b))
    for i, d in enumerate(list(tu.fields())[:2]):
        g["utils/jacdet%d" % i] = utils.jacobian_determinant(d)
    # tests/test_generators.py::test_matches_live_reference
    structure = {}
    with tempfile.TemporaryDirectory() as tmp:
        files = tg.make_dataset(tmp)
        for name, case in sorted(tg.CASES.items()):
            arrs = []
            structure[name] = flatten(tg.run_case(vxm.generators, files, case), arrs)
            for i, x in enumerate(arrs):
                g["generators/%s/%d" % (name, i)] = x
    g["generators/structure"] = np.array(json.dumps(structure, sort_keys=True))
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(g), "arrays")


if __name__ == "__main__":
    main()
