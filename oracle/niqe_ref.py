"""NumPy restatement of the reference's NIQE (Deraining/basicsr/metrics/niqe.py: niqe, compute_feature, estimate_aggd_param) in the
precision the library computes it: test infrastructure only.  It takes the float32 planes (the plane cut to whole 96 x 96 blocks,
and its half) and the r(gamma) table as inputs, so it can be fed the reference's planes (tests/golden/niqe_ref.npz) or the GPU's own.

MSCN values: each 7 x 7 convolution (edges 'nearest') summed in float64 and rounded once to float32, then float32 arithmetic, as
scipy.ndimage stores them.  Distribution statistics: float64 sums of the float32 values and products.  Gamma functions: math.gamma.
Score: np.linalg.solve in float64; NaN with fewer than two NaN-free rows.  Also: the library's half plane (half_plane), and the
golden cases' seeded inputs (case_image), which are made from integer arithmetic so that every machine rebuilds the same bytes."""
import math

import numpy as np

BLOCK = 96
NTABLE = 9801
SHIFTS = ((0, 1), (1, 0), (1, 1), (1, -1))


def gam(i):
    """np.arange(0.2, 10.001, 0.001)[i]: numpy fills start + i * ((start + step) - start)"""
    return 0.2 + np.asarray(i, dtype=np.float64) * ((0.2 + 0.001) - 0.2)


def table():
    """r(gamma) of estimate_aggd_param over the 9801 entries, with math.gamma"""
    out = []
    for g in gam(np.arange(NTABLE)):
        rec = 1.0 / g
        g2 = math.gamma(rec * 2)
        out.append((g2 * g2) / (math.gamma(rec) * math.gamma(rec * 3)))
    return np.array(out)


def half_plane(plane):
    """the library's half plane of a float32 plane: fl32(((q00 + q01) + (q10 + q11)) * 0.25) * 255 with q = plane / 255, float32"""
    q = np.asarray(plane, dtype=np.float32) / np.float32(255)
    m = ((q[0::2, 0::2] + q[0::2, 1::2]) + (q[1::2, 0::2] + q[1::2, 1::2])) * np.float32(0.25)
    return m * np.float32(255)


def _mix(n):
    """splitmix64 of uint64 n (wrapping arithmetic)"""
    z = n + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _tri(t, period):
    """triangle wave of integer t: 0 .. period, period 2 * period"""
    return np.abs(t % (2 * period) - period)


def case_image(seed, h, w, c, dtype, flat=False):
    """the seeded input of a golden case, (h, w, c) BGR, or (h, w) for c = 0, from integer arithmetic only (so every machine makes
    the same bits): smooth ramps per channel, a texture whose strength varies over the image, and noise of about 6 grey levels.
    dtype: 'uint8' / 'uint16' / 'float32' (multiples of 1/8) / 'float64' (multiples of 1/64) in [0, 255] (uint16: [0, 65535]).
    flat: a flat square, a clipped (saturated) region and a brightened band, as uint8."""
    with np.errstate(over="ignore"):
        y, x = np.mgrid[0:h, 0:w].astype(np.int64)
        out = []
        for ch in range(max(c, 1)):
            r = _mix(np.arange(8, dtype=np.uint64) + np.uint64(1000 * seed + 17 * ch)) % np.uint64(97)
            p = [int(v) + 40 for v in r]
            base = 40 * 64 + 30 * _tri(y * p[0] // 16 + x * p[1] // 16 + p[2] * 9, 64 * 64) // 64 \
                + 20 * _tri(x * p[3] // 8 - y * p[4] // 8, 48 * 64) // 48
            n = _mix((np.uint64(seed) << np.uint64(40)) + (np.uint64(ch) << np.uint64(36)) + (y * w + x).astype(np.uint64))
            noise = (n % np.uint64(769)).astype(np.int64) + ((n >> np.uint64(20)) % np.uint64(769)).astype(np.int64) - 768
            texture = _tri(x * 7 + y * 3, 40) * _tri(y * p[5] // 32 + x, 96) // 60 * ((n >> np.uint64(40)) % np.uint64(9)).astype(np.int64)
            out.append(np.clip(base + noise + texture * 8, 0, 255 * 64))
    v = np.stack(out, axis=-1)  # integers in [0, 255 * 64]
    if flat:
        v[:110, :110] = 128 * 64
        v[100:, 150:] = 255 * 64
        v[:96, 200:] = np.minimum(v[:96, 200:] + 120 * 64, 255 * 64)
    img = {"uint8": lambda: ((v + 32) // 64).astype(np.uint8), "uint16": lambda: (v * 65535 // (255 * 64)).astype(np.uint16),
           "float32": lambda: ((v // 8) / 8).astype(np.float32), "float64": lambda: v / 64.0}[dtype]()
    return img[..., 0] if c == 0 else img


def mscn(img, window):
    """(H, W) float32 -> the float32 MSCN map (img - mu) / (sigma + 1)"""
    img = np.asarray(img, dtype=np.float32)
    H, W = img.shape
    p = np.pad(img, 3, mode="edge")
    p2 = np.square(p)
    mu = np.zeros((H, W))
    sq = np.zeros((H, W))
    for i in range(7):
        for j in range(7):  # convolution: tap (i, j) meets pixel (y + 3 - i, x + 3 - j)
            mu += window[i, j] * p[6 - i:6 - i + H, 6 - j:6 - j + W].astype(np.float64)
            sq += window[i, j] * p2[6 - i:6 - i + H, 6 - j:6 - j + W].astype(np.float64)
    muf, sqf = mu.astype(np.float32), sq.astype(np.float32)
    sigma = np.sqrt(np.abs(sqf - muf * muf))
    return (img - muf) / (sigma + np.float32(1))


def aggd(x, tab):
    """estimate_aggd_param of the float32 values x -> (alpha index, alpha, beta_l, beta_r), statistics in float64"""
    u = np.asarray(x, dtype=np.float32).reshape(-1).astype(np.float64)
    neg, pos = u[u < 0], u[u > 0]
    nan = float("nan")
    left = math.sqrt(np.sum(neg * neg) / len(neg)) if len(neg) else nan
    right = math.sqrt(np.sum(pos * pos) / len(pos)) if len(pos) else nan
    gh = left / right if right else nan
    m1, m2 = np.sum(np.abs(u)) / u.size, np.sum(u * u) / u.size
    rhat = m1 * m1 / m2 if m2 else nan
    rn = (rhat * (gh * gh * gh + 1) * (gh + 1)) / ((gh * gh + 1) * (gh * gh + 1))
    idx = 0 if math.isnan(rn) else int(np.argmin((tab - rn) ** 2))
    alpha = float(gam(idx))
    r = math.sqrt(math.gamma(1 / alpha) / math.gamma(3 / alpha))
    return idx, alpha, left * r, right * r


def block_features(block, tab):
    """compute_feature of one float32 MSCN block -> 18 float64 features"""
    _, a, bl, br = aggd(block, tab)
    feat = [a, (bl + br) / 2]
    for s in SHIFTS:
        _, a, bl, br = aggd(block * np.roll(block, s, axis=(0, 1)), tab)
        feat += [a, (br - bl) * (math.gamma(2 / a) / math.gamma(1 / a)), bl, br]
    return feat


def features(plane, half, window, tab):
    """(H, W) plane cut to whole blocks and its (H / 2, W / 2) half, float32 -> (blocks, 36) float64 distparam, row w * nbh + h"""
    nbh, nbw = plane.shape[0] // BLOCK, plane.shape[1] // BLOCK
    out = []
    for scale, img in ((1, plane), (2, half)):
        n = mscn(img, window)
        bs = BLOCK // scale
        out.append([block_features(n[h * bs:(h + 1) * bs, w * bs:(w + 1) * bs], tab) for w in range(nbw) for h in range(nbh)])
    return np.concatenate([np.array(f).reshape(nbh * nbw, 18) for f in out], axis=1)


def score(feats, mu_pris, cov_pris):
    """the NIQE score of (blocks, 36) features; NaN with fewer than two NaN-free rows"""
    ok = ~np.isnan(feats).any(axis=1)
    if ok.sum() < 2:
        return float("nan")
    with np.errstate(all="ignore"):
        mu = np.nanmean(feats, axis=0)
    d = np.reshape(mu_pris, -1) - mu
    m = (cov_pris + np.cov(feats[ok], rowvar=False)) / 2
    return float(math.sqrt(d @ np.linalg.solve(m, d)))
