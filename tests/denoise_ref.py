"""numpy restatement of the denoiser (csrc/device/denoise.h, include/lrk.h's lrk_denoise / lrk_download_gbuffer) for the CPU and GPU
tests: fp32 throughout, one rounded operation at a time in the device's order, so that only exp differs (exp rounded from fp64 against expf)."""
from __future__ import annotations

import numpy as np

f = np.float32
SIGMA_L, SIGMA_Z, NORMAL_SQUARINGS, ITERATIONS, ALBEDO_BIAS = f(4.0), f(0.05), 7, 5, f(0.01)
K5 = [f(1 / 16), f(1 / 4), f(3 / 8), f(1 / 4), f(1 / 16)]
B3 = [f(0.25), f(0.5), f(0.25)]


def lum(r, g, b):
    return f(0.2126) * r + f(0.7152) * g + f(0.0722) * b


def guides(albedo_sum, normal_sum, hits):
    """albedo_sum [..., 4] = (sum albedo, S), normal_sum [..., 4] = (sum n, sum t), hits [...] = H -> albedo_cov, normal_depth."""
    s = albedo_sum[..., 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        ac = np.concatenate([albedo_sum[..., :3] / s[..., None], (hits / s)[..., None]], axis=-1)
        n = normal_sum
        nn = n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1] + n[..., 2] * n[..., 2]
        inv = f(1) / np.sqrt(nn)
        nrm = np.where((nn != 0)[..., None], n[..., :3] * inv[..., None], f(0))
        z = np.where(hits > 0, n[..., 3] / hits, f(0))
    nd = np.concatenate([nrm, z[..., None]], axis=-1)
    empty = (s == 0)[..., None]
    return np.where(empty, f(0), ac).astype(f), np.where(empty, f(0), nd).astype(f)


def normal_weight(np_, cov_p, nq, cov_q):
    hp, hq = cov_p != 0, cov_q != 0
    c = np.maximum(f(0), np_[..., 0] * nq[..., 0] + np_[..., 1] * nq[..., 1] + np_[..., 2] * nq[..., 2])
    for _ in range(NORMAL_SQUARINGS):
        c = c * c
    return np.where(~hp & ~hq, f(1), np.where(hp != hq, f(0), c)).astype(f)


def _exp(x):
    """exp of fp32 arguments, rounded once to fp32 (closer to the device's expf than numpy's own fp32 exp)."""
    return np.exp(x.astype(np.float64)).astype(f)


def _shift(a, dy, dx):
    """a[y + dy, x + dx] where that is inside the image (zeros elsewhere) and the mask of where it is."""
    h, w = a.shape[:2]
    out = np.zeros_like(a)
    valid = np.zeros((h, w), bool)
    y0, y1, x0, x1 = max(0, -dy), min(h, h - dy), max(0, -dx), min(w, w - dx)
    if y0 < y1 and x0 < x1:
        out[y0:y1, x0:x1] = a[y0 + dy:y1 + dy, x0 + dx:x1 + dx]
        valid[y0:y1, x0:x1] = True
    return out, valid


def atrous(cur, ac, nd, step):
    """One à-trous step over the whole image: cur [H, W, 4] = (I.rgb, var)."""
    var = cur[..., 3]
    g = np.zeros(var.shape, f)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            vq, valid = _shift(var, dy, dx)
            with np.errstate(invalid="ignore"):
                g = np.where(valid, g + (B3[dy + 1] * B3[dx + 1]) * vq, g)
    g = np.sqrt(g)
    lp = lum(cur[..., 0], cur[..., 1], cur[..., 2])
    cov_p = ac[..., 3]
    sw, sr, sg, sb, sv = (np.zeros(var.shape, f) for _ in range(5))
    for dy in range(-2, 3):
        for dx in range(-2, 3):
            iq, valid = _shift(cur, step * dy, step * dx)
            nq, _ = _shift(nd, step * dy, step * dx)
            acq, _ = _shift(ac, step * dy, step * dx)
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                if dx == 0 and dy == 0:
                    wt = np.ones(var.shape, f)
                else:
                    wl = _exp(-np.abs(lp - lum(iq[..., 0], iq[..., 1], iq[..., 2])) / (SIGMA_L * g + f(1e-6)))
                    wn = normal_weight(nd, cov_p, nq, acq[..., 3])
                    wz = _exp(-np.abs(nd[..., 3] - nq[..., 3]) / (SIGMA_Z * f(step) * np.maximum(nd[..., 3], nq[..., 3]) + f(1e-6)))
                    wt = wl * wn * wz
                hw = (K5[dy + 2] * K5[dx + 2]) * wt
                take = valid & (hw != 0)
                sw = np.where(take, sw + hw, sw)
                sr = np.where(take, sr + hw * iq[..., 0], sr)
                sg = np.where(take, sg + hw * iq[..., 1], sg)
                sb = np.where(take, sb + hw * iq[..., 2], sb)
                hw2 = hw * hw
                sv = np.where(take & (hw2 != 0), sv + hw2 * iq[..., 3], sv)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.stack([sr / sw, sg / sw, sb / sw, sv / (sw * sw)], axis=-1).astype(f)


def denoise(color, ac, nd, v):
    """color [H, W, >=3]: the normalised film; ac / nd: the guides; v [H, W]: the variance (inf below two samples).
    Returns the denoised [H, W, 4] with alpha 1."""
    d = ac[..., :3] + ALBEDO_BIAS
    ld = lum(d[..., 0], d[..., 1], d[..., 2])
    with np.errstate(over="ignore"):
        cur = np.concatenate([color[..., :3] / d, (v / (ld * ld))[..., None]], axis=-1).astype(f)
    for it in range(ITERATIONS):
        cur = atrous(cur, ac, nd, 1 << it)
    out = np.ones(color.shape[:2] + (4,), f)
    out[..., :3] = d * cur[..., :3]
    return out
