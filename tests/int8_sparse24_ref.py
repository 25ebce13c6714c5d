"""numpy restatement of the 2:4 sparser's mask (sb200_sparse24_mask) and of the 2:4 weight format
(sb200_int8_sparse24_pack, include/sparsebit_b200.h section 5a), down to the metadata word order the sparse wgmma reads.

Mask: every row of w.reshape(rows, -1), in aligned groups of 4 from k = 0, keeps its two largest |w|; ties go to the
lower index, NaN ranks above every number, +-0 rank as 0, a tail group of r < 4 keeps min(2, r).

Pack: d = w_q - w_zero (0 for k >= K, and for a row whose w_scale is NaN); a group keeps i0 < i1, its nonzero positions
then its lowest zero positions up to two."""
import numpy as np

PAD_WORD = 0x44444444


def mask24(w):
    """bool mask shaped like ``w`` (2-D or more; rows along axis 0)."""
    w = np.asarray(w, np.float32)
    rows = w.reshape(w.shape[0], -1)
    n, k = rows.shape
    out = np.zeros((n, k), bool)
    key = np.where(np.isnan(rows), np.inf, np.abs(rows)).astype(np.float64)
    nan = np.isnan(rows)
    for g0 in range(0, k, 4):
        r = min(4, k - g0)
        for i in range(r):
            beaten = np.zeros(n, np.int64)
            for j in range(r):
                if j == i:
                    continue
                a, b = g0 + j, g0 + i
                above = np.where(nan[:, a] | nan[:, b], nan[:, a] & ~nan[:, b], key[:, a] > key[:, b])
                below = np.where(nan[:, a] | nan[:, b], nan[:, b] & ~nan[:, a], key[:, b] > key[:, a])
                beaten += above | ((j < i) & ~below)
            out[:, g0 + i] = beaten < 2
    return out.reshape(w.shape)


def k64(k):
    return (k + 63) // 64 * 64


def centred(w_q, w_zero, w_scale, k):
    """d [N, K64] int64: the centred grid, zero past K and on NaN-scale rows."""
    n = w_q.shape[0]
    d = np.zeros((n, k64(k)), np.int64)
    d[:, :k] = w_q[:, :k].astype(np.int64) - np.asarray(w_zero, np.int64).reshape(-1, 1)
    d[np.isnan(np.asarray(w_scale, np.float32))] = 0
    return d


def kept(d):
    """(i0, i1, bad) per group: [N, G] each."""
    n = d.shape[0]
    g = d.reshape(n, -1, 4)
    nz = g != 0
    order = np.argsort(~nz, axis=2, kind="stable")  # nonzeros first, each part in index order
    i0, i1 = np.minimum(order[..., 0], order[..., 1]), np.maximum(order[..., 0], order[..., 1])
    bad = (nz.sum(2) > 2) | ((g < -128) | (g > 127)).any(2)
    return i0, i1, bad


def thread_feature(t):
    """The feature (within a 64-feature half-tile) and the K half of consumer thread t's metadata word."""
    return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * (t & 1), (t >> 1) & 1


def pack(w_q, w_zero, w_scale, k):
    """(vals int8 [N, K64 / 2], meta uint32 [ceil(N / 128), K64 / 64, 2, 128], dsum int32 [N], bad int32 [N])."""
    d = centred(w_q, w_zero, w_scale, k)
    n, kk = d.shape
    i0, i1, bad = kept(d)
    g = d.reshape(n, -1, 4)
    v0 = np.take_along_axis(g, i0[..., None], 2)[..., 0]
    v1 = np.take_along_axis(g, i1[..., None], 2)[..., 0]
    vals = np.stack([v0, v1], 2).reshape(n, kk // 2).astype(np.int8)
    nib = (i0 | (i1 << 2)).astype(np.uint64)  # [N, G]
    tiles, steps = (n + 127) // 128, kk // 64
    meta = np.full((tiles, steps, 2, 128), PAD_WORD, np.uint64)
    for b in range(tiles):
        for h in range(2):
            for t in range(128):
                f, half = thread_feature(t)
                row = 128 * b + 64 * h + f
                if row >= n:
                    continue
                for s in range(steps):
                    j0 = 16 * s + 8 * half
                    meta[b, s, h, t] = int(sum(int(nib[row, j0 + q]) << (4 * q) for q in range(8)))
    return vals, meta.astype(np.uint32), d.sum(1).astype(np.int32), bad.sum(1).astype(np.int32)


def unpack(vals, meta, n, k):
    """The dense centred grid [N, K64] that (vals, meta) stand for."""
    kk = k64(k)
    d = np.zeros((n, kk), np.int64)
    meta = np.asarray(meta).view(np.uint32)
    for b in range(meta.shape[0]):
        for h in range(2):
            for t in range(128):
                f, half = thread_feature(t)
                row = 128 * b + 64 * h + f
                if row >= n:
                    continue
                for s in range(meta.shape[1]):
                    word = int(meta[b, s, h, t])
                    for q in range(8):
                        j = 16 * s + 8 * half + q
                        nibble = (word >> (4 * q)) & 15
                        d[row, 4 * j + (nibble & 3)] += int(vals[row, 2 * j])
                        d[row, 4 * j + (nibble >> 2)] += int(vals[row, 2 * j + 1])
    return d
