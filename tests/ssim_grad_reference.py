"""d(1 - SSIM)/d(out) restated in float64 numpy: the ground truth of the native SSIM gradient (wn_ssim_grad,
metrics.ssim_loss).  Built on tests/metrics_reference.py (its window, reflect indexing and centring), it is the
adjoint of metrics.ssim term by term: the per-pixel derivatives by mu_out, E[out^2] and E[out ref], their transposed
window folded back through the reflect padding, and the data-range term at the tied extremes (torch's rules for max,
min and maximum).  The keyword switches each break one of those rules; the CPU tests show the GPU bar rejects them.

The bar of the GPU tests (DESIGN.md 4.17), element by element:

    |G - R| <= 4 max(E_torch32, F),   F = 32 u M,   u = 2^-24,

with R this restatement, E_torch32 the worst element error of torch fp32 autograd on the same input, and M the
largest sum of the three terms' magnitudes |w*A| + 2 |out| |w*B| + |ref| |w*C| (centred values): the fp32 kernel
rounds each term a few dozen times at most, so F bounds what it can lose where torch happens to be exact.
"""
import numpy as np

from metrics_reference import RAD, _reflect, blur, gaussian

U = 2.0 ** -24
FLOOR_ULPS = 32
FACTOR = 4


def _adjoint_axis(a, axis, fold=True):
    """The adjoint of one 11-tap pass of ``blur`` along ``axis`` (output side n -> source side n): the transposed
    window onto the padded positions, then each padded position added to its reflected source (``fold``) or, without
    it, the padded positions dropped."""
    g = gaussian()
    a = np.moveaxis(a, axis, -1)
    n = a.shape[-1]
    padded = np.zeros(a.shape[:-1] + (n + 2 * RAD,))
    for k in range(2 * RAD + 1):
        padded[..., k:k + n] += g[k] * a
    src = padded[..., RAD:RAD + n].copy()
    if fold:
        idx = _reflect(n)
        for j in list(range(RAD)) + list(range(n + RAD, n + 2 * RAD)):
            src[..., idx[j]] += padded[..., j]
    return np.moveaxis(src, -1, axis)


def blur_t(a, fold=True):
    """The adjoint of ``blur`` on the last two axes."""
    return _adjoint_axis(_adjoint_axis(a, -1, fold), -2, fold)


def _group_grad(p, t, scale, split_ties=True, range_term=True, fold=True, crop=True, terms=False):
    """d/dp of scale * sum_i SSIM_i for a (N,3,H,W) group with one data range (SSIM_i: image i's mean over its counted
    pixels).  ``terms``: also the per-element sum of the three terms' magnitudes."""
    p, t = np.asarray(p, np.float64), np.asarray(t, np.float64)
    ro, rr = p.max() - p.min(), t.max() - t.min()
    dr = max(ro, rr)
    c1, c2 = (0.01 * dr) ** 2, (0.03 * dr) ** 2
    mid = 0.5 * (min(p.min(), t.min()) + max(p.max(), t.max()))
    pc, tc = p - mid, t - mid
    mpc, mtc = blur(pc), blur(tc)
    up, ut = mpc + mid, mtc + mid
    vp, vt, cov = blur(pc * pc) - mpc ** 2, blur(tc * tc) - mtc ** 2, blur(pc * tc) - mpc * mtc
    a1, b1 = 2 * up * ut + c1, 2 * cov + c2
    a2, b2 = up ** 2 + ut ** 2 + c1, vp + vt + c2
    with np.errstate(invalid="ignore", divide="ignore"):
        s = (a1 * b1) / (a2 * b2)
        h, w = p.shape[-2:]
        mask = np.zeros((h, w))
        if crop and h > 2 * RAD and w > 2 * RAD:
            mask[RAD:-RAD, RAD:-RAD] = 1
        else:
            mask[:] = 1
        wpx = scale * mask / (p.shape[1] * mask.sum())  # per image: its planes times their counted pixels
        da = wpx * s * (2 * ut / a1 - 2 * up / a2 - 2 * mtc / b1 + 2 * mpc / b2)
        db = -wpx * s / b2
        dc = 2 * wpx * s / b1
        ta, tb, tcc = blur_t(da, fold), blur_t(db, fold), blur_t(dc, fold)
        grad = ta + 2 * pc * tb + tc * tcc
        if range_term:
            d_range = np.sum(wpx * (s * (1 / a1 - 1 / a2) * 2e-4 * dr + s * (1 / b1 - 1 / b2) * 18e-4 * dr))
            share = 1.0 if ro > rr else (0.5 if ro == rr else 0.0)
            at_max, at_min = p == p.max(), p == p.min()
            grad = grad + share * d_range * (at_max / (at_max.sum() if split_ties else 1))
            grad = grad - share * d_range * (at_min / (at_min.sum() if split_ties else 1))
    if terms:
        return grad, np.abs(ta) + 2 * np.abs(pc * tb) + np.abs(tc * tcc)
    return grad


def grad(out, ref, pool_items=False, terms=False, **mutations):
    """d(1 - S)/d(out): S = ssim(out, ref) of a (N,3,H,W) batch (the mean over images, one data range), or for two
    lists the mean over items of each item's ssim (batch_quality).  Returns an array, or a list for lists; with
    ``terms`` also the largest magnitude sum M of the bar.  ``pool_items``: one data range and one mean over all
    images of a list (a mutation)."""
    if not isinstance(out, (list, tuple)):
        g, m = _group_grad(out, ref, -1.0 / len(out), terms=True, **mutations)
        return (g, m.max()) if terms else g
    if pool_items:
        n = sum(len(o) for o in out)
        sizes = {o.shape[1:] for o in out}
        assert len(sizes) == 1, "pooling needs one size"
        g, m = _group_grad(np.concatenate(out), np.concatenate(ref), -1.0 / n, terms=True, **mutations)
        gs = np.split(g, np.cumsum([len(o) for o in out])[:-1])
        return (gs, m.max()) if terms else gs
    res = [_group_grad(o, r, -1.0 / len(out) / len(o), terms=True, **mutations) for o, r in zip(out, ref)]
    gs = [g for g, _ in res]
    return (gs, max(m.max() for _, m in res)) if terms else gs


def floor(m):
    """F of the bar for the largest magnitude sum ``m``."""
    return FLOOR_ULPS * U * m


def bar_violations(got, want, torch32, m):
    """Elements of ``got`` outside the bar around ``want``, given torch fp32's gradient ``torch32``; lists are taken
    whole (one worst error over all items).  Returns (count, worst error, allowed)."""
    if isinstance(got, (list, tuple)):
        got, want, torch32 = (np.concatenate([np.ravel(a) for a in x]) for x in (got, want, torch32))
    got, want, torch32 = (np.asarray(a, np.float64) for a in (got, want, torch32))
    allowed = FACTOR * max(np.max(np.abs(torch32 - want)), floor(m))
    err = np.abs(got - want)
    return int(np.sum(~(err <= allowed))), float(np.max(err)), float(allowed)
