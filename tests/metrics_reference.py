"""SSIM and PSNR of waternet_b200/metrics.py restated in float64 numpy: separable Gaussian windows over reflect-indexed
planes, the crop, the per-image means and the list rules of training.batch_quality.  The ground truth of the native
metrics (wn_quality)."""
import numpy as np

RAD = 5


def gaussian():
    x = np.arange(2 * RAD + 1, dtype=np.float64) - RAD
    g = np.exp(-(x ** 2) / (2 * 1.5 ** 2))
    return g / g.sum()


def _reflect(n):
    """Indices of the reflect padding of 5 of a side of n (n >= 6)."""
    i = np.arange(-RAD, n + RAD)
    i = np.where(i < 0, -i, i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def blur(x):
    """The 11 x 11 Gaussian window over the reflect-padded last two axes, as two 11-tap passes."""
    g = gaussian()
    h, w = x.shape[-2:]
    xp = x[..., _reflect(h), :][..., _reflect(w)]
    rows = sum(g[k] * xp[..., :, k:k + w] for k in range(2 * RAD + 1))
    return sum(g[k] * rows[..., k:k + h, :] for k in range(2 * RAD + 1))


def image_ssims(p, t):
    """Per-image SSIM of a (N,3,H,W) group: one data range over the whole group.  The variances and the covariance
    are taken of values centred on the group's mid-range (they are shift-invariant), so that a constant pair gives
    0 / 0 = NaN as in exact arithmetic."""
    p, t = np.asarray(p, np.float64), np.asarray(t, np.float64)
    dr = max(p.max() - p.min(), t.max() - t.min())
    c1, c2 = (0.01 * dr) ** 2, (0.03 * dr) ** 2
    mid = 0.5 * (min(p.min(), t.min()) + max(p.max(), t.max()))
    pc, tc = p - mid, t - mid
    mpc, mtc = blur(pc), blur(tc)
    mp, mt = mpc + mid, mtc + mid
    vp, vt, cov = blur(pc * pc) - mpc ** 2, blur(tc * tc) - mtc ** 2, blur(pc * tc) - mpc * mtc
    with np.errstate(invalid="ignore", divide="ignore"):
        s = ((2 * mp * mt + c1) * (2 * cov + c2)) / ((mp ** 2 + mt ** 2 + c1) * (vp + vt + c2))
    if s.shape[-1] > 2 * RAD and s.shape[-2] > 2 * RAD:
        s = s[..., RAD:-RAD, RAD:-RAD]
    return s.reshape(s.shape[0], -1).mean(-1)


def quality(out, ref):
    """(SSIM, PSNR) of batch_quality: a (N,3,H,W) batch, or two lists of (N_i,3,H_i,W_i) items (the mean of the items'
    SSIMs, the PSNR of the squared error pooled over every element)."""
    items = list(zip(out, ref)) if isinstance(out, (list, tuple)) else [(out, ref)]
    s = np.mean([image_ssims(o, r).mean() for o, r in items])
    sq = sum(np.sum((np.asarray(o, np.float64) - np.asarray(r, np.float64)) ** 2) for o, r in items)
    n = sum(np.asarray(o).size for o, _ in items)
    with np.errstate(divide="ignore"):
        return float(s), float(10 * np.log10(n / sq))


def inputs(kind, shape, seed=0):
    """(out, ref) fp32 arrays of ``shape``: "noise" (uniform), "smooth" (low-frequency waves), "flat" (0.5 plus
    noise of 1e-3: nearly constant)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        a = rng.random(shape)
        b = np.clip(a + 0.1 * rng.standard_normal(shape), 0, 1)
    elif kind == "smooth":
        n, c, h, w = shape
        y, x = np.meshgrid(np.arange(h) / max(h, 1), np.arange(w) / max(w, 1), indexing="ij")
        ph = rng.random((n, c, 1, 1)) * 6.28
        a = 0.5 + 0.4 * np.sin(3 * x + 2 * y + ph)
        b = 0.5 + 0.35 * np.sin(3 * x + 2.2 * y + ph + 0.3)
    elif kind == "flat":
        a = 0.5 + 1e-3 * rng.random(shape)
        b = 0.5 + 1e-3 * rng.random(shape)
    else:
        raise ValueError(kind)
    return a.astype(np.float32), b.astype(np.float32)
