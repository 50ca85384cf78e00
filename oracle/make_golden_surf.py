"""Freeze the reference's surface targets (voxelmorph/py/utils.py:308-470, voxelmorph/generators.py:256-418) for
tests/test_surface_generators.py.

TEST INFRASTRUCTURE ONLY (needs the reference tree, see oracle/ref_import.py):
    VXM_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_surf
runs the UNMODIFIED reference surf_semisupervised for every case of tests/test_surface_generators.CASES, six yields on
the seeded synthetic blob dataset of `make_dataset`, and writes tests/golden/surf_generators.npz.  skimage is absent
here: for this recipe only, the stub `skimage.measure` gets `label` (scipy.ndimage.label with the requested
connectivity, components numbered in raster order like skimage's) and `regionprops` (per-label `area`, in label
order)."""
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _shim_measure(measure):
    from scipy import ndimage

    def label(x, connectivity=None):
        x = np.asarray(x)
        lab, _ = ndimage.label(x, structure=ndimage.generate_binary_structure(x.ndim, connectivity or x.ndim))
        return lab

    def regionprops(lab, cache=True):
        areas = np.bincount(np.asarray(lab).ravel())[1:]
        return [types.SimpleNamespace(label=i + 1, area=int(a)) for i, a in enumerate(areas) if a > 0]

    measure.label, measure.regionprops = label, regionprops


def main():
    from oracle import ref_import
    import test_surface_generators as ts
    vxm_ref = ref_import.import_reference()
    _shim_measure(sys.modules["skimage.measure"])
    out = {}
    for name, case in sorted(ts.CASES.items()):
        with tempfile.TemporaryDirectory() as d:
            out.update(ts.golden_entries(name, ts.run_case(vxm_ref.generators, d, case)))
    path = os.path.join(ROOT, "tests", "golden", "surf_generators.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "entries")


if __name__ == "__main__":
    main()
