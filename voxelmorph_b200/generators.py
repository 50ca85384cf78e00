"""Host-side data feed for the training loop ("next" row N1 of SURVEY.md section 8(f)).

Same generator names, arguments and yield contract as the reference (voxelmorph/generators.py:9-143: `volgen` yields a
tuple of channel-last numpy batches, `scan_to_scan` / `scan_to_atlas` yield `(invols, outvols)` lists), and the same
sequence of draws from `np.random`, so `scripts/torch/train.py:200-201` consumes it unchanged.  What differs is the cost
per step, which bounds the unmodified loop once a GPU step takes milliseconds:

* every file is decoded ONCE (`VolumeCache`): the reference re-opens and re-inflates the `.npz` on every draw
  (py/utils.py:69-129 -> ~0.19 s per 160x192x224 volume);
* volumes are kept as float32, C-contiguous, feature axis included, in page-locked memory when CUDA is present: the
  `.float()` of train.py:200 is a no-op and `.to(device)` is one DMA from pinned memory instead of a pageable staged copy
  preceded by a float64 -> float32 pass;
* a batch of one is a zero-copy view (no `np.concatenate`);
* the all-zero "target flow" that `Grad` ignores (generators.py:96-99) is float32 instead of float64: half the bytes
  for train.py:201 to move, and no cast kernel;
* `Prefetcher` runs any generator one or more batches ahead on a background thread.

Nothing here touches the GPU; it is covered by CPU tests against the reference generators (tests/test_generators.py).
"""
import glob
import os
import queue
import threading
from collections import OrderedDict

import numpy as np

__all__ = ["VolumeCache", "load_volfile", "volgen", "scan_to_scan", "scan_to_atlas", "semisupervised", "template_creation",
           "conditional_template_creation", "hypermorph", "surf_semisupervised", "Prefetcher"]


def _cuda_ready():
    """True once THIS PROCESS already has a CUDA context.  The data feed must never create one itself: the reference's
    train.py draws its first batch (scripts/torch/train.py:113) BEFORE it sets CUDA_VISIBLE_DEVICES (train.py:125), and the CUDA
    runtime reads that variable when it initialises — a feed that page-locks memory at the first draw (or merely asks
    torch.cuda.is_available()) pins every rank of a multi-GPU run to device 0."""
    try:
        import torch
        return torch.cuda.is_initialized()
    except Exception:  # noqa: BLE001
        return False


def _pinned_empty(shape, dtype):
    """Page-locked numpy array when this process already uses CUDA, plain numpy otherwise.  Returns (array, owner)."""
    try:
        if _cuda_ready():
            import torch
            t = torch.empty(tuple(shape), dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True)
            return t.numpy(), t
    except Exception:  # noqa: BLE001 - pinning is an optimisation, never a requirement
        pass
    return np.empty(shape, dtype=dtype), None


def _pad_centered(vol, shape):
    """Zero-pad to `shape`, content centred with floor((target - size) / 2) leading zeros (py/utils.py:235-247)."""
    if vol.shape == tuple(shape):
        return vol
    if len(shape) != vol.ndim or any(p < v for p, v in zip(shape, vol.shape)):
        raise ValueError("pad_shape %r cannot hold a volume of shape %r" % (tuple(shape), vol.shape))
    out = np.zeros(shape, dtype=vol.dtype)
    lead = [int((p - v) / 2) for p, v in zip(shape, vol.shape)]
    out[tuple(slice(o, o + n) for o, n in zip(lead, vol.shape))] = vol
    return out


def _decode(src, np_var):
    """File name or preloaded array -> numpy array (py/utils.py:92-117).  Preloaded arrays are passed through."""
    if isinstance(src, os.PathLike):
        src = os.fspath(src)
    if not isinstance(src, str):
        return np.asarray(src)
    if not os.path.isfile(src):
        raise ValueError("'%s' is not a file." % src)
    if src.endswith((".nii", ".nii.gz", ".mgz")):
        try:
            import nibabel as nib
        except ImportError as e:
            raise ValueError("loading %s needs nibabel, which is not installed" % src) from e
        return np.squeeze(nib.load(src).dataobj)
    if src.endswith(".npy"):
        return np.load(src)
    if src.endswith(".npz"):
        with np.load(src) as z:
            keys = list(z.keys())
            return z[keys[0]] if len(keys) == 1 else z[np_var]
    raise ValueError("unknown filetype for %s" % src)


def _resize_nearest(vol, factor):
    """Nearest-neighbour zoom of every axis but the trailing feature axis (py/utils.py:250-262, scipy zoom order 0)."""
    if factor == 1:
        return vol
    from scipy import ndimage
    return ndimage.zoom(vol, [factor] * (vol.ndim - 1) + [1], order=0)


class VolumeCache:
    """Decode-once store: (source, np_var, pad_shape, resize_factor, add_feat_axis) -> ready-to-batch array.

    Floating-point volumes are stored as float32 (what train.py:200 converts to anyway); integer volumes (label maps)
    keep their dtype.  `max_bytes` bounds the cache (least recently used entries are dropped); `pin=None` page-locks the
    volumes once the process has a CUDA context (never creating one: see _cuda_ready).
    """

    def __init__(self, max_bytes=None, pin=None):
        self.max_bytes = max_bytes
        self.pin = pin
        self._items = OrderedDict()
        self._owners = {}
        self._bytes = 0
        self._lock = threading.Lock()
        self.hits = self.misses = 0

    def get(self, src, np_var="vol", pad_shape=None, resize_factor=1, add_feat_axis=True):
        if not isinstance(src, (str, os.PathLike)):
            # preloaded arrays are never cached (an id()-keyed entry could outlive its array and be served to a later
            # array that reuses the address, or go stale when the array is modified in place): like the reference
            # (py/utils.py:95-99) they are passed through, with the same padding / axis handling
            vol = np.asarray(src)
            if pad_shape:
                vol = _pad_centered(vol, pad_shape)
            if add_feat_axis:
                vol = vol[..., np.newaxis]
            return _resize_nearest(vol, resize_factor)
        key = (os.fspath(src), np_var, None if pad_shape is None else tuple(pad_shape), resize_factor, bool(add_feat_axis))
        with self._lock:
            hit = self._items.get(key)
            if hit is not None:
                self._items.move_to_end(key)
                self.hits += 1
                if (self.pin is not False and key not in self._owners and hit.dtype == np.float32 and _cuda_ready()):
                    # decoded before the process had a CUDA context (see _cuda_ready): page-lock it now, once
                    buf, owner = _pinned_empty(hit.shape, hit.dtype)
                    if owner is not None:
                        np.copyto(buf, hit)
                        buf.setflags(write=False)
                        self._items[key] = buf
                        self._owners[key] = owner
                        hit = buf
                return hit
        vol = _decode(src, np_var)
        if pad_shape:
            vol = _pad_centered(vol, pad_shape)
        if add_feat_axis:
            vol = vol[..., np.newaxis]
        vol = _resize_nearest(vol, resize_factor)
        dtype = np.float32 if np.issubdtype(vol.dtype, np.floating) else vol.dtype
        owner = None
        if self.pin is not False and dtype == np.float32:
            buf, owner = _pinned_empty(vol.shape, dtype)
            np.copyto(buf, vol, casting="same_kind")
            vol = buf
        else:
            vol = np.ascontiguousarray(vol, dtype=dtype)
        vol.setflags(write=False)
        with self._lock:
            self.misses += 1
            self._items[key] = vol
            if owner is not None:
                self._owners[key] = owner
            self._bytes += vol.nbytes
            while self.max_bytes is not None and self._bytes > self.max_bytes and len(self._items) > 1:
                k, v = self._items.popitem(last=False)
                self._owners.pop(k, None)
                self._bytes -= v.nbytes
        return vol

    def __len__(self):
        return len(self._items)


def _default_cache_bytes():
    """Bound of the process-wide cache: VXM_B200_CACHE_GB, else a quarter of the host's RAM, at most 16 GiB
    (page-locking more than that can destabilise the host)."""
    env = os.environ.get("VXM_B200_CACHE_GB")
    if env:
        return int(float(env) * (1 << 30))
    try:
        ram = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES")
    except (ValueError, OSError, AttributeError):
        ram = 32 << 30
    return int(min(16 << 30, ram // 4))


_default_cache = VolumeCache(max_bytes=_default_cache_bytes())


def load_volfile(filename, np_var="vol", add_batch_axis=False, add_feat_axis=False, pad_shape=None, resize_factor=1, cache=None):
    """Reference-compatible loader (py/utils.py:69-129 without `ret_affine`) that decodes each file once."""
    vol = (_default_cache if cache is None else cache).get(filename, np_var, pad_shape, resize_factor, add_feat_axis)
    return vol[np.newaxis, ...] if add_batch_axis else vol


def _expand_names(vol_names):
    if isinstance(vol_names, str):
        if os.path.isdir(vol_names):
            vol_names = os.path.join(vol_names, "*")
        vol_names = glob.glob(vol_names)
    return vol_names


def _batch(items):
    """Stack volumes along a new leading axis; one volume is returned as a view."""
    if len(items) == 1:
        return items[0][np.newaxis, ...]
    out, owner = _pinned_empty((len(items),) + items[0].shape, items[0].dtype) if items[0].dtype == np.float32 else \
        (np.empty((len(items),) + items[0].shape, items[0].dtype), None)
    for i, v in enumerate(items):
        out[i] = v
    if owner is not None:
        out = _Owned(out, owner)
    return out


class _Owned(np.ndarray):
    """ndarray view that keeps the page-locked torch storage it aliases alive."""

    def __new__(cls, arr, owner):
        obj = arr.view(cls)
        obj._owner = owner
        return obj

    def __array_finalize__(self, obj):
        self._owner = getattr(obj, "_owner", None)


def volgen(vol_names, batch_size=1, segs=None, np_var="vol", pad_shape=None, resize_factor=1, add_feat_axis=True, cache=None):
    """Random volume batches; arguments and yields as reference generators.py:9-68 (`cache`: a VolumeCache to share)."""
    vol_names = _expand_names(vol_names)
    if isinstance(segs, list) and len(segs) != len(vol_names):
        raise ValueError("Number of image files must match number of seg files.")
    cache = _default_cache if cache is None else cache
    opts = dict(pad_shape=pad_shape, resize_factor=resize_factor, add_feat_axis=add_feat_axis)
    while True:
        indices = np.random.randint(len(vol_names), size=batch_size)   # same draw as generators.py:50
        vols = [_batch([cache.get(vol_names[i], np_var, **opts) for i in indices])]
        if segs is True:        # npz files carrying a 'seg' variable next to 'vol'
            vols.append(_batch([cache.get(vol_names[i], "seg", **opts) for i in indices]))
        elif isinstance(segs, list):
            vols.append(_batch([cache.get(segs[i], np_var, **opts) for i in indices]))
        yield tuple(vols)


def _zero_flow(batch_size, vol_shape, dtype):
    z = np.zeros((batch_size,) + tuple(vol_shape) + (len(vol_shape),), dtype=dtype)
    z.setflags(write=False)
    return z


def scan_to_scan(vol_names, bidir=False, batch_size=1, prob_same=0, no_warp=False, zeros_dtype=np.float32, **kwargs):
    """Scan-to-scan pairs; arguments, yields and random draws as reference generators.py:71-107."""
    zeros = None
    gen = volgen(vol_names, batch_size=batch_size, **kwargs)
    while True:
        scan1 = next(gen)[0]
        scan2 = next(gen)[0]
        if prob_same > 0 and np.random.rand() < prob_same:
            if np.random.rand() > 0.5:
                scan1 = scan2
            else:
                scan2 = scan1
        if not no_warp and zeros is None:
            zeros = _zero_flow(batch_size, scan1.shape[1:-1], zeros_dtype)
        invols = [scan1, scan2]
        outvols = [scan2, scan1] if bidir else [scan2]
        if not no_warp:
            outvols.append(zeros)
        yield (invols, outvols)


def scan_to_atlas(vol_names, atlas, bidir=False, batch_size=1, no_warp=False, segs=None, zeros_dtype=np.float32, **kwargs):
    """Scan-to-atlas pairs; arguments and yields as reference generators.py:110-143 (`atlas`: (1, *vol, 1) array)."""
    atlas = np.asarray(atlas)
    zeros = _zero_flow(batch_size, atlas.shape[1:-1], zeros_dtype)
    atlas = np.repeat(atlas.astype(np.float32, copy=False), batch_size, axis=0)
    gen = volgen(vol_names, batch_size=batch_size, segs=segs, **kwargs)
    while True:
        res = next(gen)
        scan = res[0]
        invols = [scan, atlas]
        if not segs:
            outvols = [atlas, scan] if bidir else [atlas]
        else:
            outvols = [res[1], scan] if bidir else [res[1]]
        if not no_warp:
            outvols.append(zeros)
        yield (invols, outvols)


def template_creation(vol_names, bidir=False, batch_size=1, zeros_dtype=np.float32, **kwargs):
    """Unconditional template creation; arguments, yields and random draws as reference generators.py:197-219:
    ([scan], [scan, zeros, zeros(, zeros)]), zeros of shape (1, *vol, nd) (the mean stream's and the flow's targets,
    float32 like scan_to_atlas's)."""
    zeros = None
    gen = volgen(vol_names, batch_size=batch_size, **kwargs)
    while True:
        scan = next(gen)[0]
        if zeros is None:
            zeros = _zero_flow(1, scan.shape[1:-1], zeros_dtype)
        invols = [scan]
        outvols = [scan, zeros, zeros, zeros] if bidir else [scan, zeros, zeros]
        yield (invols, outvols)


def conditional_template_creation(vol_names, atlas, attributes, batch_size=1, np_var='vol', pad_shape=None,
                                  add_feat_axis=True, zeros_dtype=np.float32, cache=None):
    """Conditional template creation; arguments, yields and random draws as reference generators.py:222-253:
    ([pheno, atlas, vols], [vols, zeros, zeros, zeros]) with pheno (batch_size, P) the rows of `attributes` (a dict keyed
    by the entries of `vol_names`, e.g. pyutils.load_pheno_csv's) for the drawn volumes, atlas (1, *vol, C) repeated over
    the batch, zeros (batch_size, *vol, nd).  Volumes come through the decode-once cache; every array is float32."""
    atlas = np.asarray(atlas)
    zeros = _zero_flow(batch_size, atlas.shape[1:-1], zeros_dtype)
    atlas = np.repeat(atlas.astype(np.float32, copy=False), batch_size, axis=0)
    cache = _default_cache if cache is None else cache
    opts = dict(pad_shape=pad_shape, add_feat_axis=add_feat_axis)
    while True:
        indices = np.random.randint(len(vol_names), size=batch_size)   # same draw as generators.py:241
        pheno = np.stack([attributes[vol_names[i]] for i in indices], axis=0).astype(np.float32)
        vols = _batch([cache.get(vol_names[i], np_var, **opts) for i in indices])
        yield ([pheno, atlas, vols], [vols, zeros, zeros, zeros])


def semisupervised(vol_names, seg_names, labels, atlas_file=None, downsize=2, prob_dtype=np.float32, zeros_dtype=np.float32, cache=None):
    """Semi-supervised pairs ("next" row N2; reference generators.py:146-194): yields
    ([src_vol, trg_vol, src_prob_seg], [trg_vol, zeros, trg_prob_seg]) with the label maps turned into one-hot
    probability maps over `labels` and sub-sampled by `downsize` per axis.  Batch size is 1, 3-D only, like the
    reference; the draws from np.random follow its order (one volgen draw for the source, one for the target unless an
    atlas file supplies it).  The one-hot is built on the sub-sampled label map in one comparison against the label
    vector (float32 instead of float64: a 30-label map at 80x96x112 is 103 MB rather than 206 MB per segmentation)."""
    labels = np.asarray(labels)
    cache = _default_cache if cache is None else cache
    gen = volgen(vol_names, segs=seg_names, np_var="vol", cache=cache)

    def prob_seg(seg):
        if seg.shape[0] != 1 or seg.ndim != 5:
            raise ValueError("semisupervised: segmentations must be (1, D, H, W, 1) label maps (batch size 1, 3-D)")
        sub = seg[0, ::downsize, ::downsize, ::downsize, 0]
        return (sub[..., np.newaxis] == labels).astype(prob_dtype)[np.newaxis]

    trg_vol = trg_seg = None
    if atlas_file:
        trg_vol = cache.get(atlas_file, "vol", add_feat_axis=True)[np.newaxis]
        trg_seg = prob_seg(cache.get(atlas_file, "seg", add_feat_axis=True)[np.newaxis])
    zeros = None
    while True:
        src_vol, src_lab = next(gen)
        src_seg = prob_seg(src_lab)
        if not atlas_file:
            trg_vol, trg_lab = next(gen)
            trg_seg = prob_seg(trg_lab)
        if zeros is None:
            zeros = _zero_flow(1, src_vol.shape[1:-1], zeros_dtype)
        yield ([src_vol, trg_vol, src_seg], [trg_vol, zeros, trg_seg])


def surf_semisupervised(vol_names, atlas_vol, atlas_seg, nb_surface_pts, labels=None, batch_size=1, surf_bidir=True,
                        surface_pts_upsample_factor=2, smooth_seg_std=1, nb_labels_sample=None, sdt_vol_resize=1,
                        align_segs=False, add_feat_axis=True, sdt_dtype=np.float32, pts_dtype=np.float32,
                        zeros_dtype=np.float32, cache=None):
    """Scan-to-atlas batches with surface targets for VxmDenseSemiSupervisedPointCloud (reference
    generators.py:256-418): arguments, yield contract and np.random draws as the reference's.  Yields

        ([subj, atlas, subj_sdt, atlas_sdt, subj_surf, atlas_surf], [atlas, subj, zero_flow, zeros, zeros])

    or, without `surf_bidir`, ([subj, atlas, subj_sdt, atlas_surf], [atlas, subj, zero_flow, zeros]); arrays are
    channel-last: SDTs (B, *sdt_shape, nb_labels_sample), surfaces (B, nb_surface_pts, nd + 1) with the label slot in
    the last column, zeros (B, nb_surface_pts, 1).  Per label the segmentation is cleaned (pyutils.clean_seg), its
    signed distance transform taken and points drawn on its surface; with nb_labels_sample below the label count a
    random subset of labels is drawn per batch.  Batch size 1 only, like the reference.

    The reference yields float64; `sdt_dtype`, `pts_dtype` and `zeros_dtype` (float32 by default) choose the output
    types, the computation stays float64 (38 labels at 160x192x224 are 2.1 GB of SDTs per batch in float32).  The
    reference's quirk is kept: the atlas SDT stacked for a sampled label is that of its position in the sample, not of
    the label itself (generators.py:384)."""
    from . import pyutils
    assert nb_surface_pts > 0, 'number of surface point should be greater than 0'
    vol_shape = atlas_seg.shape
    nd = len(vol_shape)
    sdt_shape = [int(f * sdt_vol_resize) for f in vol_shape]
    if labels is not None:
        atlas_seg = pyutils.filter_labels(atlas_seg, labels)
    else:
        labels = np.sort(np.unique(atlas_seg))[1:]
    nb_labels = len(labels)
    if nb_labels_sample is None:
        nb_labels_sample = nb_labels
    sample = nb_labels_sample != nb_labels

    atlas_vol_bs = np.repeat(atlas_vol[np.newaxis, ..., np.newaxis], batch_size, axis=0)
    atlas_seg_bs = np.repeat(atlas_seg[np.newaxis, ..., np.newaxis], batch_size, axis=0)

    def surf_pts(sdt, n):
        return pyutils.sdt_to_surface_pts(sdt, n, surface_pts_upsample_factor=surface_pts_upsample_factor,
                                          thr=(1 / surface_pts_upsample_factor + 1e-5))

    zero_flow = np.zeros((batch_size, *vol_shape, nd), dtype=zeros_dtype)
    zero_values = np.zeros((batch_size, nb_surface_pts, 1), dtype=zeros_dtype)

    atlas_sdt = []
    nb_edges = np.zeros(nb_labels)
    for li, label in enumerate(labels):
        atlas_sdt.append(pyutils.vol_to_sdt(pyutils.clean_seg(atlas_seg == label, smooth_seg_std), sdt=True,
                                            sdt_vol_resize=sdt_vol_resize))
        nb_edges[li] = np.sum(np.abs(atlas_sdt[li]) < 1.01)
    edge_ratios = nb_edges / np.sum(nb_edges)

    def slot(counts, li):
        return slice(int(np.sum(counts[:li])), int(np.sum(counts[:li + 1])))

    atlas_surf = np.zeros((batch_size, nb_surface_pts, nd + 1), dtype=pts_dtype)
    if not sample:
        counts = pyutils.get_surface_pts_per_label(nb_surface_pts, edge_ratios)
        for li in range(nb_labels):
            s = slot(counts, li)
            atlas_surf[:, s, :-1] = surf_pts(atlas_sdt[li], counts[li])[np.newaxis]
            atlas_surf[:, s, -1] = li

    gen = volgen(vol_names, segs=True, batch_size=batch_size, add_feat_axis=add_feat_axis, cache=cache)
    assert batch_size == 1, 'only batch size 1 supported for now'

    while True:
        X_img, X_lab = next(gen)
        X_seg = pyutils.filter_labels(X_lab, labels)
        sel = range(nb_labels)
        if sample:
            sel = np.sort(np.random.choice(range(nb_labels), size=nb_labels_sample, replace=False))
            counts = pyutils.get_surface_pts_per_label(nb_surface_pts, [edge_ratios[li] for li in sel])
            atlas_surf = np.zeros((batch_size, nb_surface_pts, nd + 1), dtype=pts_dtype)
        subj_sdt = np.zeros((batch_size, *sdt_shape, nb_labels_sample), dtype=sdt_dtype)
        atl_sdt = np.zeros((batch_size, *sdt_shape, nb_labels_sample), dtype=sdt_dtype)
        subj_surf = np.zeros((batch_size, nb_surface_pts, nd + 1), dtype=pts_dtype)

        for li, sli in enumerate(sel):
            s = slot(counts, li)
            if sample:
                atlas_surf[:, s, :-1] = surf_pts(atlas_sdt[sli], counts[li])[np.newaxis]
                atlas_surf[:, s, -1] = sli
            label_bw = pyutils.clean_seg_batch(X_seg == labels[sli], smooth_seg_std)
            sdt = pyutils.vol_to_sdt_batch(label_bw, sdt=True, sdt_vol_resize=sdt_vol_resize)[..., 0]
            subj_sdt[..., li] = sdt
            if surf_bidir:
                atl_sdt[..., li] = atlas_sdt[li][np.newaxis]
                subj_surf[:, s, :-1] = np.stack([surf_pts(f, counts[li]) for f in sdt], 0)
                subj_surf[:, s, -1] = li

        X_ret, atlas_ret = X_img, atlas_vol_bs
        if align_segs:
            assert nb_labels == 1, 'align_seg generator is only implemented for single label'
            X_ret = X_seg == labels[0]
            atlas_ret = atlas_seg_bs == labels[0]

        if surf_bidir:
            yield ([X_ret, atlas_ret, subj_sdt, atl_sdt, subj_surf, atlas_surf],
                   [atlas_ret, X_ret, zero_flow, zero_values, zero_values])
        else:
            yield ([X_ret, atlas_ret, subj_sdt, atlas_surf], [atlas_ret, X_ret, zero_flow, zero_values])


class Prefetcher:
    """Iterate `gen` on a background thread, `depth` items ahead (decode / batch assembly overlaps the GPU step).

    The random draws still happen in generator order, on the worker thread.  Exceptions raised by the generator are
    re-raised by `next()`; `close()` stops the worker.
    """

    _END = object()

    def __init__(self, gen, depth=2):
        self._q = queue.Queue(maxsize=max(1, depth))
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._run, args=(gen,), daemon=True)
        self._thread.start()

    def _run(self, gen):
        try:
            for item in gen:
                while not self._stop.is_set():
                    try:
                        self._q.put(item, timeout=0.1)
                        break
                    except queue.Full:
                        continue
                if self._stop.is_set():
                    return
            self._q.put(self._END)
        except BaseException as e:  # noqa: BLE001 - handed to the consumer
            self._q.put(e)

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if item is self._END:
            raise StopIteration
        if isinstance(item, BaseException):
            raise item
        return item

    def close(self):
        self._stop.set()


def hypermorph(base_generator, oversample_rate=0.2):
    """HyperMorph's hyperparameter extension of any generator (reference scripts/tf/train_hypermorph.py:107-121): yields
    ((*inputs, hyp), outputs) for every (inputs, outputs) of `base_generator`, hyp of shape (1, 1) float32.  lambda is
    drawn as the script's random_hyperparam draws it — np.random.rand() < oversample_rate picks np.random.choice([0, 1]),
    otherwise np.random.rand() — before next(base_generator).  The draw is made once per batch, not once per batch entry
    as in the script: HyperVxmDense takes one lambda per step, shared by the batch.  At batch size 1 (the script's
    default) the sequence of np.random draws is the script's."""
    while True:
        lam = np.random.choice([0, 1]) if np.random.rand() < oversample_rate else np.random.rand()
        hyp = np.full((1, 1), lam, dtype=np.float32)
        inputs, outputs = next(base_generator)
        yield (tuple(inputs) + (hyp,), outputs)
