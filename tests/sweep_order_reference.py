"""The sweep's Morton order (srl_fast.cu: k_sweep_keys, k_sweep_order_cluster) restated in numpy.

Every keypoint's LiDAR-frame 1 m cell, per axis c = fmin(fmax(floor(x) + 128, 0), 255): numpy's fmax / fmin drop a NaN
operand as CUDA's do, so NaN lands in cell 0, +inf in 255 and -inf in 0.  The 24-bit key interleaves the cells' bits, x
at bit 3i, y at 3i + 1, z at 3i + 2; the order is the stable sort of the keys (np.argsort(kind="stable")), entry s = the
keypoint at sorted position s.

The cluster kernel's geometry is restated too, for a cluster of 16 CTAs of 32 warps: every warp owns `per` consecutive
keys (a multiple of 32, at most 8 x 32), warp g the range [g per, (g + 1) per) clipped to n, a CTA its 32 warps' ranges.
The case builders use it to say which boundary a case sits on.
"""
import numpy as np

N_CTA = 16
WARPS = 32
ROUNDS = 8
KEYS_PER_CTA = WARPS * ROUNDS * 32     # 8192
CAPACITY = N_CTA * KEYS_PER_CTA        # 131072: longer sweeps are sorted by CUB


def cells(xyz):
    """(n, 3) float64 -> (n, 3) uint32 cells in [0, 255]."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore"):
        c = np.fmin(np.fmax(np.floor(xyz) + 128.0, 0.0), 255.0)
    return c.astype(np.uint32)


def spread8(c):
    """Bit i of c to bit 3i."""
    c = np.asarray(c, np.uint32) & np.uint32(0xFF)
    out = np.zeros_like(c)
    for i in range(8):
        out |= ((c >> np.uint32(i)) & np.uint32(1)) << np.uint32(3 * i)
    return out


def morton(c):
    """(n, 3) cells -> (n,) 24-bit keys."""
    c = np.asarray(c, np.uint32).reshape(-1, 3)
    return spread8(c[:, 0]) | (spread8(c[:, 1]) << np.uint32(1)) | (spread8(c[:, 2]) << np.uint32(2))


def keys(xyz):
    return morton(cells(xyz))


def order(xyz):
    """The sweep order: (n,) uint32."""
    return np.argsort(keys(xyz), kind="stable").astype(np.uint32)


def unmorton(k):
    """(n,) 24-bit keys -> (n, 3) cells: the inverse of morton."""
    k = np.asarray(k, np.uint32)
    c = np.zeros((k.size, 3), np.uint32)
    for i in range(8):
        for a in range(3):
            c[:, a] |= ((k >> np.uint32(3 * i + a)) & np.uint32(1)) << np.uint32(i)
    return c


def points_for_keys(k, rng, frac=None):
    """Points whose keys are k: cell - 128 + a fraction in [0, 1) per axis (seeded, or `frac` as given)."""
    c = unmorton(k).astype(np.float64) - 128.0
    if frac is None:
        frac = rng.uniform(0.0, 1.0, c.shape)
    xyz = c + frac
    # cell - 128 + frac rounds up to the next integer when frac is within half an ulp of 1: keep it inside the cell
    over = np.floor(xyz) > c
    xyz[over] = np.nextafter(c[over] + 1.0, -np.inf)
    return xyz


def digit(k, p):
    """The 8-bit digit radix pass p sorts by."""
    return (np.asarray(k, np.uint32) >> np.uint32(8 * p)) & np.uint32(0xFF)


def pass_inputs(k):
    """The key sequence each of the 3 radix passes reads: the keys, then stably sorted by digit 0, then by digits 0 and 1."""
    k = np.asarray(k, np.uint32)
    seq = [k]
    for p in range(2):
        seq.append(seq[-1][np.argsort(digit(seq[-1], p), kind="stable")])
    return seq


def geometry(n, n_cta=N_CTA):
    """The cluster kernel's split of n keys: dict(per, begin, end (per warp, cluster order), cta_n (per CTA))."""
    n_warps = n_cta * WARPS
    per = ((n + n_warps - 1) // n_warps + 31) // 32 * 32
    g = np.arange(n_warps, dtype=np.int64)
    begin = np.minimum(n, g * per)
    end = np.minimum(n, begin + per)
    c = np.arange(n_cta, dtype=np.int64)
    cta_n = np.minimum(n, (c + 1) * WARPS * per) - np.minimum(n, c * WARPS * per)
    return dict(per=per, begin=begin, end=end, cta_n=cta_n)
