"""Host restatement of experiments/pet_ct_tnm_classification/preprocessing.py for the PET-CT preprocessing tests.

  - resample: ITK's ResampleImageFilter with the identity transform and LinearInterpolateImageFunction, restated in numpy fp64 voxel by
    voxel (every voxel independently; ITK's scan-line path accumulates the continuous index incrementally instead).  Output index ->
    physical point -> input continuous index with the matrices direction diag(spacing) and diag(1 / spacing) direction^T, each row summed in
    axis order; outside [-0.5, size - 0.5) on some axis -> 0; base = max(0, floor(c)); lerps a + (b - a) d along x, then y, then z (the
    base sample where d <= 0 or base + 1 is past the end); CastPixelWithBoundsChecking to the output type.
  - clear_border: skimage.segmentation.clear_border restated on scipy.ndimage.label with the full 2-D structure.
  - everything else on numpy / scipy as the reference writes it: get_z_crops, the segment merge, the crop and the normalisation.

Grids are dicts {'size': (x, y, z), 'origin', 'spacing', 'direction' (9, row-major)}; arrays are (z, y, x)."""
import numpy as np
from scipy import ndimage

BACKGROUND_CATEGORIES = ['M1b_brain', 'N_inflammation', 'T_benign', 'T_other']
NEW_SPACING = (0.976562, 0.976562, 3.27)
_RANGE = {np.dtype(np.uint8): (0.0, 255.0), np.dtype(np.int16): (-32768.0, 32767.0),
          np.dtype(np.float32): (-float(np.finfo(np.float32).max), float(np.finfo(np.float32).max)),
          np.dtype(np.float64): (-np.inf, np.inf)}      # float64: the interpolated value before the cast


def grid(size, origin, spacing, direction=(1, 0, 0, 0, 1, 0, 0, 0, 1)):
    return {'size': tuple(int(s) for s in size), 'origin': tuple(float(o) for o in origin), 'spacing': tuple(float(s) for s in spacing),
            'direction': tuple(float(d) for d in direction)}


def continuous_index(in_grid, out_grid, zs):
    """[3] fp64 arrays (x, y, z) of the input continuous index of every output voxel of the z slices zs, each (len(zs), Y, X)"""
    X, Y, _ = out_grid['size']
    k, j, i = np.meshgrid(np.asarray(zs, np.float64), np.arange(Y, dtype=np.float64), np.arange(X, dtype=np.float64), indexing='ij')
    idx = (i, j, k)
    do, so, oo = out_grid['direction'], out_grid['spacing'], out_grid['origin']
    di, si, oi = in_grid['direction'], in_grid['spacing'], in_grid['origin']
    v = []
    for r in range(3):
        p = np.full(i.shape, oo[r])
        for c in range(3):
            p = p + (do[3 * r + c] * so[c]) * idx[c]
        v.append(p - oi[r])
    out = []
    for r in range(3):
        c = np.zeros(i.shape)
        for q in range(3):
            c = c + (di[3 * q + r] / si[r]) * v[q]
        out.append(c)
    return out


def resample(src, in_grid, out_grid, out_dtype, chunk=16):
    """src (z, y, x) on in_grid -> out_dtype (z, y, x) on out_grid"""
    out_dtype = np.dtype(out_dtype)
    X, Y, Z = out_grid['size']
    size = in_grid['size']
    out = np.empty((Z, Y, X), out_dtype)
    lo, hi = _RANGE[out_dtype]
    for z0 in range(0, Z, chunk):
        ci = continuous_index(in_grid, out_grid, range(z0, min(Z, z0 + chunk)))
        inside = np.ones(ci[0].shape, bool)
        b0, b1, d = [], [], []
        for r in range(3):
            inside &= (ci[r] >= -0.5) & (ci[r] < size[r] - 0.5)
            b = np.maximum(np.floor(np.where(inside, ci[r], 0.0)), 0.0)
            dd = ci[r] - b
            step = (dd > 0) & (b + 1 <= size[r] - 1)
            b = b.astype(np.int64)
            b0.append(np.where(inside, b, 0))
            b1.append(np.where(inside & step, b + 1, np.where(inside, b, 0)))
            d.append(np.where(step, dd, 0.0))
        s = lambda bx, by, bz: src[bz, by, bx].astype(np.float64)
        lerp = lambda a, b, t: a + (b - a) * t
        vx = [[lerp(s(b0[0], by, bz), s(b1[0], by, bz), d[0]) for by in (b0[1], b1[1])] for bz in (b0[2], b1[2])]
        vxy = [lerp(vx[q][0], vx[q][1], d[1]) for q in range(2)]
        val = np.where(inside, lerp(vxy[0], vxy[1], d[2]), 0.0)
        out[z0:z0 + len(val)] = np.clip(val, lo, hi).astype(out_dtype)
    return out


def image_grid(shape_zyx, spacing, origin, direction):
    return grid(tuple(shape_zyx)[::-1], origin, spacing, direction)


def new_ct_grid(ct_grid):
    """the reference's target grid when the CT's x spacing is below 0.95 or its z spacing below 3, else None"""
    sp = ct_grid['spacing']
    if not (sp[0] < 0.95 or sp[2] < 3):
        return None
    size = [int(ct_grid['size'][a] * sp[a] / NEW_SPACING[a]) for a in range(3)]
    return grid(size, ct_grid['origin'], NEW_SPACING, ct_grid['direction'])


def clear_border(img):
    """skimage.segmentation.clear_border of a 2-D bool image: its 8-connected components that touch the one-pixel border removed"""
    labels, _ = ndimage.label(img, structure=np.ones((3, 3), int))
    border = np.zeros(img.shape, bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    out = img.copy()
    out[np.isin(labels, np.unique(labels[border])) & (labels > 0)] = False
    return out


def body_components(ct):
    """(slice_first [Z + 1], stats [n, 3] int64 (count, sum of rows, sum of columns)) of the per-slice 4-connected components of
    clear_border(ct < -600), numbered in C order over the volume"""
    first, stats = [0], []
    for z in range(ct.shape[0]):
        lab, n = ndimage.label(clear_border(ct[z] < -600))
        r, c = np.nonzero(lab)
        ids = lab[r, c] - 1
        stats.append(np.stack([np.bincount(ids, minlength=n), np.bincount(ids, r, minlength=n).astype(np.int64),
                               np.bincount(ids, c, minlength=n).astype(np.int64)], axis=1).astype(np.int64).reshape(n, 3))
        first.append(first[-1] + n)
    return np.array(first, np.int64), (np.concatenate(stats) if stats else np.zeros((0, 3), np.int64))


def zcrop_flags(first, stats, Y, X, min_pix, n_comps, rad_crit):
    """[Z] bool: the slices get_z_crops appends for these parameters, from the component statistics"""
    cy, cx = Y / 2, X / 2
    out = np.zeros(len(first) - 1, bool)
    for z in range(len(out)):
        s = stats[first[z]:first[z + 1]]
        s = s[s[:, 0] > min_pix]
        n = s[:, 0].astype(np.float64)
        d = (s[:, 1] / n - cy) ** 2 + (s[:, 2] / n - cx) ** 2
        out[z] = int((d < rad_crit).sum()) >= n_comps
    return out


def get_z_crops(x, ix, min_pix=1500, n_comps=2, rad_crit=20000):
    """the reference's get_z_crops with clear_border restated (same criteria, recursion and failures)"""
    final_slices = []
    for six in range(x.shape[0]):
        tx = np.copy(x[six]) < -600
        img_center = np.array(tx.shape) / 2
        tx = clear_border(tx)
        clusters, n_cands = ndimage.label(tx)
        count = np.unique(clusters, return_counts=True)
        keep_comps = np.array([ii for ii in np.argwhere((count[1] > min_pix)) if ii > 0]).astype(int)
        if len(keep_comps) > n_comps - 1:
            coms = ndimage.center_of_mass(tx, clusters, index=keep_comps)
            keep_com = [i for i, ii in enumerate(coms[0]) if ((ii[0] - img_center[0]) ** 2 + (ii[1] - img_center[1]) ** 2 < rad_crit)]
            keep_comps = keep_comps[keep_com]
            if len(keep_comps) > n_comps - 1:
                final_slices.append(six)
    z_min = np.min(final_slices) - 7
    z_max = np.max(final_slices) + 7
    dist = z_max - z_min
    if dist >= 151:
        z_min, z_max = get_z_crops(x, ix, min_pix=min_pix + 500, rad_crit=rad_crit - 500)
    if dist <= 43:
        z_min, z_max = get_z_crops(x, ix, n_comps=1, min_pix=min_pix - 100, rad_crit=rad_crit + 100)
    return z_min, z_max


def merge_segments(readdata, labels):
    """(n_seg, x, y, z) -> binary uint8 (z, y, x): 1 where a segment whose name is not a background category is == 1"""
    seg = np.zeros(readdata.shape[1:], np.uint8)
    for k in range(readdata.shape[0]):
        if labels[k] not in BACKGROUND_CATEGORIES:
            seg[readdata[k] == 1] = 1
    return np.ascontiguousarray(np.transpose(seg, (2, 1, 0)))


def seg_geometry(readdata, header):
    """(readdata as (n_seg, x, y, z), spacing, origin, labels) as pp_patient derives them from a pynrrd header"""
    if readdata.ndim == 3:
        readdata = readdata[None]
        spacing = np.diagonal(np.asarray(header['space directions'], float))
    else:
        spacing = np.diagonal(np.asarray(header['space directions'], float)[1:, :])
    origin = np.asarray(header['space origin'], float) * np.sign(spacing)
    labels = [header[k].split('=')[-1] for k in header.keys() if '_Name' in k]
    return readdata, np.abs(spacing), origin, labels


def normalize(x, p):
    """the reference's normalisation of the cropped CT (fp64) and PET (its own dtype); -> float32 (2, z, y, x)"""
    x = np.clip(x, -1200, 600)
    x = (1200 + x) / (600 + 1200)
    x = (x - np.mean(x)) / np.std(x)
    p = (p - np.mean(p)) / np.std(p)
    return np.concatenate((x[None], p[None])).astype(np.float32)


def normalize_device(x, p):
    """the device's normalisation restated: fp64 statistics of the same values (numpy's pairwise sums in place of the device's trees; the
    two differ in the last bits), the PET's rounded to fp32 before a float32 apply"""
    c = (1200 + np.clip(x.astype(np.int64), -1200, 600)) / 1800.0
    mc = c.mean()
    sc = np.sqrt(np.mean((c - mc) ** 2))
    p64 = p.astype(np.float64)
    mp = p64.mean()
    sp = np.sqrt(np.mean((p64 - mp) ** 2))
    pc = ((c - mc) / sc).astype(np.float32)
    pp = (p.astype(np.float32) - np.float32(mp)) / np.float32(sp)
    return np.concatenate((pc[None], pp[None].astype(np.float32)))


def pp_patient(ct, ct_geom, pet, pet_geom, readdata, header, ix=0):
    """(img float32 (2, z, y, x), rois uint8, class_target, fg_slices, (z_min, z_max)) of one patient; *_geom = (spacing, origin, direction)"""
    readdata, s_spacing, s_origin, labels = seg_geometry(readdata, header)
    seg = merge_segments(readdata, labels)
    s_grid = image_grid(seg.shape, s_spacing, s_origin, (1, 0, 0, 0, 1, 0, 0, 0, 1))
    x_grid = image_grid(ct.shape, *ct_geom)
    new = new_ct_grid(x_grid)
    if new is not None:
        ct = resample(ct, x_grid, new, ct.dtype)
        x_grid = new
    pi = resample(pet, image_grid(pet.shape, *pet_geom), x_grid, pet.dtype)
    si = resample(seg, s_grid, x_grid, np.uint8)
    zmin, zmax = get_z_crops(ct, ix)
    x, p, s = ct[zmin:zmax], pi[zmin:zmax], si[zmin:zmax]
    img = normalize(x, p)
    remaining = np.unique(s)
    class_target = [ii for k, ii in enumerate(labels) if k + 1 in remaining]
    s = (s > 0).astype(np.uint8)
    fg_slices = [ii for ii in np.unique(np.argwhere(s != 0)[:, 0])]
    return img, s, class_target, fg_slices, (zmin, zmax)
