"""Freeze the behaviour of the reference generators (voxelmorph/generators.py) for tests/test_generators.py.

TEST INFRASTRUCTURE ONLY (needs the reference tree, see oracle/ref_import.py):
    VXM_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_generators
writes tests/golden/generators.json: for every case of tests/test_generators.CASES the shapes and sums of six consecutive
yields of the UNMODIFIED reference generator on the synthetic dataset of `make_dataset` (np.random seeded)."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from oracle import ref_import
    import test_generators as tg
    vxm_ref = ref_import.import_reference()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        files = tg.make_dataset(d)
        for name, case in sorted(tg.CASES.items()):
            out[name] = [tg.summarize(x) for x in tg.run_case(vxm_ref.generators, files, case)]
    path = os.path.join(ROOT, "tests", "golden", "generators.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", path, {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
