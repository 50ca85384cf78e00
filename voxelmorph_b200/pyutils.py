"""Host-side helpers with the surface of the reference's `voxelmorph.py.utils` (voxelmorph/py/utils.py) — the part of
it the torch scripts and the data feed touch: file lists, volume I/O, padding / resizing, label filtering, plus the
evaluation helpers of `voxelmorph_b200.utils`.  Pure numpy host code around the hot path (SURVEY.md section 8(b1));
written for this repo, not transcribed: loaders are a suffix-dispatch table, NIfTI support is resolved lazily so the
package imports (and `.npz` / `.npy` I/O works) on hosts without nibabel.
"""
import csv
import glob
import os

import numpy as np

from .utils import count_folds, dice, jacobian_determinant  # noqa: F401  (re-exported: py/utils.py:265-287, :473-516)

__all__ = ["default_unet_features", "get_backend", "read_file_list", "read_pair_list", "load_volfile", "save_volfile",
           "load_labels", "load_pheno_csv", "pad", "resize", "dice", "filter_labels", "affine_shift_to_matrix",
           "jacobian_determinant", "count_folds", "extract_largest_vol", "clean_seg", "clean_seg_batch", "dist_trf",
           "signed_dist_trf", "vol_to_sdt", "vol_to_sdt_batch", "get_surface_pts_per_label", "edge_to_surface_pts",
           "sdt_to_surface_pts"]


def default_unet_features():
    """Encoder / decoder widths of the default U-Net (py/utils.py:16-21)."""
    return [[16, 32, 32, 32], [32, 32, 32, 32, 32, 16, 16]]


def get_backend():
    """'pytorch' when VXM_BACKEND says so, 'tensorflow' otherwise (py/utils.py:24-29).  Only the pytorch backend
    exists in this build; `voxelmorph/__init__.py` refuses the other one."""
    return "pytorch" if os.environ.get("VXM_BACKEND") == "pytorch" else "tensorflow"


def _decorate(names, prefix, suffix):
    pre, suf = prefix or "", suffix or ""
    return [pre + n + suf for n in names]


def read_file_list(filename, prefix=None, suffix=None):
    """Non-empty lines of a text file, each optionally wrapped in prefix / suffix (py/utils.py:32-48)."""
    with open(filename, "r") as fh:
        names = [ln.strip() for ln in fh]
    return _decorate([n for n in names if n], prefix, suffix)


def read_pair_list(filename, delim=None, prefix=None, suffix=None):
    """Lines split into file pairs (py/utils.py:51-66)."""
    return [_decorate(line.split(delim), prefix, suffix) for line in read_file_list(filename)]


# ---- volume I/O ------------------------------------------------------------------------------------------------------
def _nib():
    try:
        import nibabel
    except ImportError as e:  # pragma: no cover - depends on the host
        raise ImportError("NIfTI / MGZ files need nibabel, which is not installed on this host; use .npz or .npy") from e
    return nibabel


def _read_nifti(path, np_var):
    img = _nib().load(path)
    return np.squeeze(img.dataobj), img.affine


def _read_npy(path, np_var):
    return np.load(path), None


def _read_npz(path, np_var):
    with np.load(path) as z:
        keys = list(z.keys())
        return (z[keys[0]] if len(keys) == 1 else z[np_var]), None


_READERS = ((".nii.gz", _read_nifti), (".nii", _read_nifti), (".mgz", _read_nifti), (".npy", _read_npy), (".npz", _read_npz))


def load_volfile(filename, np_var="vol", add_batch_axis=False, add_feat_axis=False, pad_shape=None, resize_factor=1,
                 ret_affine=False):
    """Load a nii / nii.gz / mgz / npz / npy volume; anything that is not a path is taken as the preloaded volume itself
    (or a (volume, affine) pair when `ret_affine`).  Same arguments and result as py/utils.py:69-129."""
    if isinstance(filename, os.PathLike):
        filename = os.fspath(filename)
    affine = None
    if isinstance(filename, str):
        if not os.path.isfile(filename):
            raise ValueError("'%s' is not a file." % filename)
        for suffix, reader in _READERS:
            if filename.endswith(suffix):
                vol, affine = reader(filename, np_var)
                break
        else:
            raise ValueError("unknown filetype for %s" % filename)
    elif ret_affine:
        vol, affine = filename
    else:
        vol = filename
    if pad_shape:
        vol, _ = pad(vol, pad_shape)
    if add_feat_axis:
        vol = vol[..., np.newaxis]
    if resize_factor != 1:
        vol = resize(vol, resize_factor)
    if add_batch_axis:
        vol = vol[np.newaxis, ...]
    return (vol, affine) if ret_affine else vol


def _lia_affine(shape3):
    """Default vox-to-RAS matrix of a volume without one: LIA orientation, centred (py/utils.py:146-153)."""
    m = np.array([[-1.0, 0, 0, 0], [0, 0, 1.0, 0], [0, -1.0, 0, 0], [0, 0, 0, 1.0]])
    centre = np.append(np.asarray(shape3, dtype=float) / 2.0, 1.0)
    m[:3, 3] = -(m @ centre)[:3]
    return m


def save_volfile(array, filename, affine=None):
    """Write nii / nii.gz (nibabel) or npz (key 'vol'); py/utils.py:132-158."""
    if isinstance(filename, os.PathLike):
        filename = os.fspath(filename)
    if filename.endswith((".nii", ".nii.gz")):
        nib = _nib()
        if affine is None and array.ndim >= 3:
            affine = _lia_affine(array.shape[:3])
        nib.save(nib.Nifti1Image(array, affine), filename)
    elif filename.endswith(".npz"):
        np.savez_compressed(filename, vol=array)
    else:
        raise ValueError("unknown filetype for %s" % filename)


def load_labels(arg, ext=(".nii.gz", ".nii", ".mgz", ".npy", ".npz")):
    """Label maps from folders / glob patterns -> (sorted unique labels, list of maps); py/utils.py:161-199."""
    patterns = [arg] if not isinstance(arg, (tuple, list)) else list(arg)
    files = []
    for pat in map(str, patterns):
        files.extend(glob.glob(os.path.join(pat, "*") if os.path.isdir(pat) else pat))
    files = [f for f in files if f.endswith(tuple(ext))]
    if not files:
        raise ValueError('no labels found for argument "%s"' % files)
    maps, shape = [], None
    for f in files:
        lab = np.squeeze(load_volfile(f))
        shape = lab.shape if shape is None else shape
        if not np.issubdtype(lab.dtype, np.integer):
            raise ValueError('file "%s" has non-integral data type' % f)
        if lab.shape != shape:
            raise ValueError('shape %s of file "%s" is not %s' % (lab.shape, f, shape))
        maps.append(lab)
    return np.unique(maps), maps


def load_pheno_csv(filename, training_files=None):
    """CSV of `basename,attr1,attr2,...` rows -> ({key: float array}, usable training files); py/utils.py:202-232."""
    table = {}
    with open(filename) as fh:
        rows = csv.reader(fh, delimiter=",")
        next(rows)  # header
        for row in rows:
            table[row[0]] = np.array([float(x) for x in row[1:]])
    if training_files is None:
        return table, list(table.keys())
    kept = [f for f in training_files if os.path.basename(f) in table]
    for f in kept:
        table[f] = table[os.path.basename(f)]
    return table, kept


def pad(array, shape):
    """Zero-pad to `shape` with the content centred; returns (padded, slices that crop it back); py/utils.py:235-247."""
    shape = tuple(shape)
    if array.shape == shape:
        return array, ...
    lead = [int((p - v) / 2) for p, v in zip(shape, array.shape)]
    window = tuple(slice(o, o + n) for o, n in zip(lead, array.shape))
    out = np.zeros(shape, dtype=array.dtype)
    out[window] = array
    return out, window


def resize(array, factor, batch_axis=False):
    """Nearest-neighbour zoom of the spatial axes of an array that carries a trailing feature axis (and a leading batch
    axis when `batch_axis`); py/utils.py:250-262."""
    if factor == 1:
        return array
    from scipy import ndimage
    zoom = [factor] * array.ndim
    zoom[-1] = 1
    if batch_axis:
        zoom[0] = 1
    return ndimage.zoom(array, zoom, order=0)


def filter_labels(atlas_vol, labels):
    """Keep the listed labels of a segmentation, zero elsewhere (py/utils.py:354-361)."""
    seg = np.asarray(atlas_vol)
    return np.where(np.isin(seg, np.asarray(labels)), seg, np.zeros((), dtype=seg.dtype))


def affine_shift_to_matrix(trf, resize=None, unshift_shape=None):
    """(12,) affine shift over the identity -> 4x4 matrix, optionally rescaled and un-centred (py/utils.py:290-305; 3-D)."""
    m = np.eye(4)
    m[:3, :] += np.asarray(trf, dtype=float).reshape(3, 4)
    if resize is not None:
        m[:3, 3] *= resize
    if unshift_shape is not None:
        to_centre = np.eye(4)
        to_centre[:3, 3] = (np.asarray(unshift_shape, dtype=float) - 1) / 2
        m = to_centre @ m @ np.linalg.inv(to_centre)
    return m


# ---- surface targets of VxmDenseSemiSupervisedPointCloud (py/utils.py:308-470), on scipy.ndimage alone ----

def extract_largest_vol(bw, connectivity=1):
    """The largest connected component of a binary image (py/utils.py:308-318).  Components are labelled in raster
    order with `connectivity` (1: faces), as skimage's measure.label numbers them; ties in size go to the component
    np.argsort(areas)[::-1] puts first."""
    from scipy import ndimage
    bw = np.asarray(bw).astype(int)
    lab, n = ndimage.label(bw, structure=ndimage.generate_binary_structure(bw.ndim, connectivity))
    areas = np.bincount(lab.ravel(), minlength=n + 1)[1:]
    return lab == np.argsort(areas)[::-1][0] + 1


def clean_seg(x, std=1):
    """Clean a binary segmentation (py/utils.py:321-337): keep the largest island, fill the holes, blur with a
    Gaussian of sigma `std` and threshold the blur so that the volume is kept.  Returns float64 0 / 1."""
    from scipy import ndimage
    bw = extract_largest_vol(x)
    bw = 1 - extract_largest_vol(1 - bw)
    blur = ndimage.gaussian_filter(bw.astype(float), std)
    k = int(np.ceil(bw.sum()))
    flat = blur.ravel()
    thr = np.partition(flat, flat.size - 1 - k)[flat.size - 1 - k]     # the (k+1)-th largest value
    clean = blur > thr
    assert np.isclose(bw.sum(), clean.sum(), atol=5), 'cleaning segmentation failed'
    return clean.astype(float)


def clean_seg_batch(X_label, std=1):
    """clean_seg of every (*vol, 1) item of a batch (py/utils.py:340-351); float64 (B, *vol, 1)."""
    X_label = np.asarray(X_label)
    out = np.zeros(X_label.shape)
    for i, x in enumerate(X_label):
        out[i, ..., 0] = clean_seg(x[..., 0], std)
    return out


def dist_trf(bwvol):
    """Euclidean distance of every voxel to the nearest True voxel (py/utils.py:364-369)."""
    from scipy import ndimage
    return ndimage.distance_transform_edt(np.logical_not(bwvol))


def signed_dist_trf(bwvol):
    """Signed distance to the surface of a binary image, positive outside and negative inside; no voxel is 0
    (py/utils.py:372-391)."""
    outside = np.logical_not(bwvol)
    return dist_trf(bwvol) * outside - dist_trf(outside) * bwvol


def vol_to_sdt(X_label, sdt=True, sdt_vol_resize=1):
    """Signed distance transform of a binary volume, zoomed by `sdt_vol_resize` (linear, 'reflect'); its absolute
    value unless `sdt` (py/utils.py:394-410)."""
    from scipy import ndimage
    X_dt = signed_dist_trf(X_label)
    if sdt_vol_resize != 1:
        factors = list(sdt_vol_resize) if isinstance(sdt_vol_resize, (list, tuple)) else [sdt_vol_resize] * X_dt.ndim
        if any(f != 1 for f in factors):
            X_dt = ndimage.zoom(X_dt, factors, order=1, mode='reflect')
    return X_dt if sdt else np.abs(X_dt)


def vol_to_sdt_batch(X_label, sdt=True, sdt_vol_resize=1):
    """vol_to_sdt of every item of a (B, *vol, 1) batch (py/utils.py:413-424)."""
    assert X_label.shape[-1] == 1, 'implemented assuming size is [batch_size, *vol_shape, 1]'
    return np.stack([vol_to_sdt(x[..., 0], sdt=sdt, sdt_vol_resize=sdt_vol_resize) for x in X_label], 0)[..., np.newaxis]


def get_surface_pts_per_label(total_nb_surface_pts, layer_edge_ratios):
    """Split a point budget over labels in proportion to their edge counts, the last label taking the remainder
    (py/utils.py:427-434)."""
    n = np.round(np.array(layer_edge_ratios) * total_nb_surface_pts).astype('int')
    n[-1] = total_nb_surface_pts - int(np.sum(n[:-1]))
    return n


def edge_to_surface_pts(X_edges, nb_surface_pts=None):
    """Coordinates (P, nd) of the True voxels, or `nb_surface_pts` of them drawn with replacement
    (np.random.choice, py/utils.py:437-449)."""
    pts = np.stack(np.where(X_edges), 0).transpose()
    if nb_surface_pts is not None:
        pts = pts[np.random.choice(pts.shape[0], size=nb_surface_pts), :]
    return pts


def sdt_to_surface_pts(X_sdt, nb_surface_pts, surface_pts_upsample_factor=2, thr=0.50001, resize_fn=None):
    """Surface points of a signed distance transform (py/utils.py:452-470): the SDT is upsampled (linear zoom,
    'reflect', or `resize_fn`), voxels with |sdt| < thr are the surface, `nb_surface_pts` of them are drawn and
    mapped back to the SDT's grid, coordinates scaled by (S - 1) / (S_up - 1) per axis."""
    from scipy import ndimage
    if resize_fn is None:
        up = ndimage.zoom(X_sdt, [surface_pts_upsample_factor] * X_sdt.ndim, order=1, mode='reflect')
    else:
        up = resize_fn(X_sdt)
        assert np.array_equal(np.array(X_sdt.shape) * surface_pts_upsample_factor, up.shape), 'resizing failed'
    edges = np.abs(up) < thr
    pts = edge_to_surface_pts(edges, nb_surface_pts=nb_surface_pts)
    return np.stack([pts[..., d] * (X_sdt.shape[d] - 1) / (edges.shape[d] - 1) for d in range(X_sdt.ndim)], -1)
