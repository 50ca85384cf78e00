"""Host-side feed rate of the scan-to-scan generator (row N1): batches/s a training loop can draw, including the
train.py:200-201 host conversion (`torch.from_numpy(d).float().permute(0, 4, 1, 2, 3)`), for
  reference  : the unmodified voxelmorph.generators.scan_to_scan (needs the reference tree: VXM_REFERENCE_ROOT, see oracle/ref_import.py)
  b200       : voxelmorph_b200.generators.scan_to_scan (decode-once cache, float32, zero-copy batch of one)
  b200+prefetch : the same behind generators.Prefetcher
on N synthetic compressed .npz volumes of the BASELINE shape.  CPU only; prints one JSON line.
Usage: python tools/feed_bench.py [--shape 160 192 224] [--files 4] [--steps 12]"""
import argparse, json, os, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch


def consume(item):
    inputs, y_true = item
    a = [torch.from_numpy(np.asarray(d)).float().permute(0, 4, 1, 2, 3) for d in inputs]
    b = [torch.from_numpy(np.asarray(d)).float().permute(0, 4, 1, 2, 3) for d in y_true]
    return sum(int(t.shape[0]) for t in a + b)


def rate(gen, steps, skip=0):
    for _ in range(skip):
        consume(next(gen))
    t0 = time.perf_counter()
    for _ in range(steps):
        consume(next(gen))
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=3, default=[160, 192, 224])
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--steps", type=int, default=12)
    args = ap.parse_args()
    from voxelmorph_b200 import generators
    from oracle import ref_import
    out = {"shape": args.shape, "files": args.files, "steps": args.steps, "unit": "batches/s (1 pair per batch, host side only)"}
    with tempfile.TemporaryDirectory() as d:
        rng = np.random.RandomState(0)
        files = []
        for i in range(args.files):
            # smooth-ish content so that the deflate ratio resembles a skull-stripped scan (about half zeros)
            v = np.zeros(args.shape, np.float32)
            c = tuple(slice(s // 6, s - s // 6) for s in args.shape)
            v[c] = rng.rand(*[s - 2 * (s // 6) for s in args.shape]).astype(np.float32)
            f = os.path.join(d, "scan%02d.npz" % i)
            np.savez_compressed(f, vol=v)
            files.append(f)
        if ref_import.available():
            ref = ref_import.import_reference()
            np.random.seed(1)
            out["reference"] = rate(ref.generators.scan_to_scan(files, batch_size=1), max(3, args.steps // 3))
        np.random.seed(1)
        cache = generators.VolumeCache()
        gen = generators.scan_to_scan(files, batch_size=1, cache=cache)
        t0 = time.perf_counter()
        for f in files:
            cache.get(f)
        out["b200_first_pass_decode_s"] = time.perf_counter() - t0
        out["b200"] = rate(gen, args.steps * 20, skip=2)
        pf = generators.Prefetcher(generators.scan_to_scan(files, batch_size=1, cache=cache), depth=3)
        out["b200_prefetch"] = rate(pf, args.steps * 20, skip=2)
        pf.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
