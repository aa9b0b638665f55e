"""numpy / scipy restatement of the LIDC preprocessing of the reference's experiments/lidc_exp/preprocessing.py.

`resize` restates skimage.transform.resize of scikit-image 0.16.2 for the reference's call (order=1, mode='edge', clip=True, anti_aliasing
left at its default True), written from that version's documented behaviour on scipy.ndimage:
  - factors = in_shape / out_shape; gaussian_filter(image, max(0, (factors - 1) / 2), mode='nearest') (scipy skips sigma <= 1e-15);
  - n-D branch: map_coordinates(order=1, mode='nearest') at factors[i] * (j + 0.5) - 0.5;
  - 2-D warp branch, taken when the last output extent equals the input's: the affine map estimated from three corner points, each
    channel of the last axis warped bilinearly with edge mode (here through map_coordinates at the affine's coordinates);
  - clip to the filtered image's [min, max].
`pp_patient` restates one patient on arrays already read and grouped, with the device's normalisation statistics (fp64 mean and
population std) or, with stats='numpy', numpy's float32 np.mean / np.std as the reference computes them."""
import math

import numpy as np
from scipy import ndimage as ndi

CLIP_LO, CLIP_HI = -1200, 600


def target_shape(shape, src_spacing, target_spacing):
    """the resampled extent per (z, y, x) axis: spacings are (x, y, z), the source spacing rounded to 3 decimals"""
    src_zyx = np.round(src_spacing, 3)[::-1]
    tgt_zyx = tuple(target_spacing)[::-1]
    out = [int(n * s / t) for n, s, t in zip(shape, src_zyx, tgt_zyx)]
    if min(out) <= 0:
        raise AssertionError("AssertionError:", shape, src_spacing, target_spacing)
    return out


def resize(image, output_shape, branch='auto'):
    """skimage.transform.resize(image, output_shape, order=1, mode='edge', clip=True) of scikit-image 0.16.2 (fp64 in, fp64 out).
    branch: 'auto' as skimage chooses, 'nd' or 'warp' to force one interpolation branch."""
    image = np.asarray(image, dtype=np.float64)
    output_shape = tuple(int(s) for s in output_shape)
    factors = np.asarray(image.shape, dtype=float) / np.asarray(output_shape, dtype=float)
    image = ndi.gaussian_filter(image, np.maximum(0, (factors - 1) / 2), mode='nearest')
    if branch == 'auto':
        branch = 'warp' if len(output_shape) == 2 or (len(output_shape) == 3 and output_shape[2] == image.shape[2]) else 'nd'
    if branch == 'warp':
        out = _warp_2d(image, output_shape, factors)
    else:
        axes = [factors[i] * (np.arange(d) + 0.5) - 0.5 for i, d in enumerate(output_shape)]
        coords = np.array(np.meshgrid(*axes, sparse=False, indexing='ij'))
        out = ndi.map_coordinates(image, coords, order=1, mode='nearest')
    np.clip(out, image.min(), image.max(), out=out)
    return out


def gaussian_weights(sigma):
    """scipy's 1-D gaussian kernel of gaussian_filter (truncate 4): exp(-x^2 / (2 sigma^2)) over [-r, r], r = int(4 sigma + 0.5),
    normalised by its sum; [1.0] for sigma <= 1e-15 (scipy skips the axis)"""
    if sigma <= 1e-15:
        return np.ones(1)
    r = int(4.0 * float(sigma) + 0.5)
    x = np.arange(-r, r + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def resize_points(image, output_shape, points):
    """resize(image, output_shape) of the n-D branch evaluated at the output voxels points [P, 3] only, in fp64 (the blur summed over
    each sample's clamped neighbourhood); for spot checks of volumes too large for the full restatement"""
    image = np.asarray(image)
    factors = np.asarray(image.shape, dtype=float) / np.asarray(output_shape, dtype=float)
    per_axis = []
    for a in range(3):
        n = image.shape[a]
        w = gaussian_weights(max(0.0, (factors[a] - 1) / 2))
        r = len(w) // 2
        c = np.clip(factors[a] * (points[:, a] + 0.5) - 0.5, 0, n - 1)
        i0 = np.floor(c).astype(np.int64)
        t = c - i0
        corners = [(i0, 1.0 - t), (np.minimum(i0 + 1, n - 1), t)]
        idx = np.concatenate([np.clip(ic[:, None] + np.arange(-r, r + 1)[None, :], 0, n - 1) for ic, _ in corners], axis=1)
        wt = np.concatenate([wc[:, None] * w[None, :] for _, wc in corners], axis=1)
        per_axis.append((idx, wt))
    (iz, wz), (iy, wy), (ix, wx) = per_axis
    out = np.zeros(len(points))
    for a in range(iz.shape[1]):
        for b in range(iy.shape[1]):
            v = image[iz[:, a, None], iy[:, b, None], ix].astype(np.float64)
            out += wz[:, a] * wy[:, b] * (v * wx).sum(axis=1)
    return out


def _warp_2d(image, output_shape, factors):
    """the 2-D warp branch: AffineTransform.estimate from the corners (0, 0), (0, rows - 1), (cols - 1, rows - 1) of the output grid
    (x, y order) to their source positions, shear and perspective zeroed, then bilinear with edge mode per channel of the last axis"""
    rows, cols = output_shape[0], output_shape[1]
    if rows == 1 and cols == 1:
        m = np.array([[1.0, 0.0, image.shape[1] / 2.0 - 0.5], [0.0, 1.0, image.shape[0] / 2.0 - 0.5], [0, 0, 1]])
    else:
        src = np.array([[1, 1], [1, rows], [cols, rows]], dtype=float) - 1
        dst = np.zeros(src.shape)
        dst[:, 0] = factors[1] * (src[:, 0] + 0.5) - 0.5
        dst[:, 1] = factors[0] * (src[:, 1] + 0.5) - 0.5
        m = _estimate_affine(src, dst)
        m[2] = (0, 0, 1)
        m[0, 1] = 0
        m[1, 0] = 0
    cc, rr = np.meshgrid(np.arange(cols, dtype=float), np.arange(rows, dtype=float))
    xs = m[0, 0] * cc + m[0, 1] * rr + m[0, 2]
    ys = m[1, 0] * cc + m[1, 1] * rr + m[1, 2]
    if image.ndim == 2:
        return ndi.map_coordinates(image, [ys, xs], order=1, mode='nearest')
    return np.stack([ndi.map_coordinates(image[..., c], [ys, xs], order=1, mode='nearest') for c in range(image.shape[2])], axis=-1)


def _estimate_affine(src, dst):
    """skimage's AffineTransform.estimate: the total-least-squares solution of the homogeneous system through its SVD"""
    n = src.shape[0]
    xs, ys = src[:, 0], src[:, 1]
    xd, yd = dst[:, 0], dst[:, 1]
    a = np.zeros((2 * n, 7))
    a[:n, 0], a[:n, 1], a[:n, 2], a[:n, 6] = xs, ys, 1, xd
    a[n:, 3], a[n:, 4], a[n:, 5], a[n:, 6] = xs, ys, 1, yd
    _, _, v = np.linalg.svd(a)
    h = -v[-1, :-1] / v[-1, -1]
    return np.array([[h[0], h[1], h[2]], [h[3], h[4], h[5]], [0, 0, 1]])


def resample_array(src_imgs, src_spacing, target_spacing, branch='auto'):
    """resample_array of the reference: resize to target_shape in fp64, then float32"""
    shape = target_shape(src_imgs.shape, src_spacing, target_spacing)
    return resize(src_imgs.astype(float), shape, branch=branch).astype(np.float32)


def device_stats(x):
    """the device's statistics of the clipped float32 CT, exactly: fp64 mean and population std (math.fsum)"""
    v = x.astype(np.float64).ravel()
    mean = math.fsum(v) / v.size
    d = v - mean
    return mean, math.sqrt(math.fsum(d * d) / v.size)


def normalize(x, stats='device'):
    """clip to [-1200, 600] and normalise as the reference does.  stats='device': fl32(fl32(x - fl32(mean)) / fp16(fl32(std))) with the
    fp64 statistics; stats='numpy': numpy's own float32 np.mean / np.std.  Returns (y, mean, std16) with mean as used (float32)."""
    x = np.clip(x, CLIP_LO, CLIP_HI).astype(np.float32)
    if stats == 'device':
        mean, std = device_stats(x)
        mean32 = np.float32(mean)
        std16 = np.float32(std).astype(np.float16)
    else:
        mean32 = np.mean(x)
        std16 = np.std(x).astype(np.float16)
    return (x - mean32) / std16, mean32, std16


def vote(raters):
    """the mean over max(4, n) raters in float32 (sequential sum in list order, one division), values below 0.5 zeroed"""
    acc = raters[0].copy()
    for r in raters[1:]:
        acc += r
    v = acc / np.float32(max(4, len(raters)))
    v[v < 0.5] = 0
    return v


def pp_patient(ct, ct_spacing, rois, target_spacing, stats='device'):
    """one patient.  ct: array (z, y, x); rois: per ROI in processing order, (file names, [(rater array, spacing_xyz)], malignancy label).
    Returns dict(img, rois, class_target, fg_slices, suppressed = [file name lists of the suppressed ROIs], mean, std16)."""
    img, mean, std16 = normalize(resample_array(ct, ct_spacing, target_spacing), stats)
    labels = np.zeros(img.shape, np.uint8)
    mal, suppressed = [], []
    for names, raters, label in rois:
        res = []
        for arr, sp in raters:
            r = resample_array(arr.astype(np.uint8), sp, target_spacing)
            assert r.shape == img.shape
            res.append(r)
        v = vote(res)
        if v.sum() > 0:
            mal.append(label)
            labels[v >= 0.5] = len(mal)
        else:
            suppressed.append(list(names))
    fg = [z for z in np.unique(np.argwhere(labels != 0)[:, 0])]
    assert len(mal) + 1 == len(np.unique(labels))
    return dict(img=img, rois=labels, class_target=np.array(mal), fg_slices=fg, suppressed=suppressed, mean=mean, std16=std16)
