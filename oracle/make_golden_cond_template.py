"""Freeze the reference's conditional template generator (voxelmorph/generators.py:222-253) and its attribute reader
(voxelmorph/py/utils.py:202-232) for tests/test_cond_template_oracle.py.

TEST INFRASTRUCTURE ONLY (needs the reference tree, see oracle/ref_import.py):
    VXM_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_cond_template
writes tests/golden/cond_template_generator.npz: for every case of test_cond_template_oracle.GEN_CASES, every array of
six consecutive yields of the UNMODIFIED reference generator on the seeded synthetic dataset of
test_cond_template_oracle.make_pheno_dataset (np.random seeded), and the np.random state after them."""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from oracle import ref_import
    import test_cond_template_oracle as tc
    from test_generators import flatten
    vxm_ref = ref_import.import_reference()
    out, structure = {}, {}
    with tempfile.TemporaryDirectory() as d:
        files, csv_path, atlas = tc.make_pheno_dataset(d)
        attributes, kept = vxm_ref.py.utils.load_pheno_csv(csv_path, files)
        for name, kw in sorted(tc.GEN_CASES.items()):
            items, state = tc.run_gen(vxm_ref.generators, kept, atlas, attributes, kw)
            arrs = []
            structure[name] = flatten(items, arrs)
            for i, a in enumerate(arrs):
                out["%s/%d" % (name, i)] = np.asarray(a)
            out["%s/state" % name] = state
    out["structure"] = np.array(json.dumps(structure))
    path = os.path.join(ROOT, "tests", "golden", "cond_template_generator.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
