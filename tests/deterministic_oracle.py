"""Host restatement of the deterministic render backward's reduction (include/glic_b200.h, glic_backward_deterministic).

A Gaussian's contributions v_0 .. v_{n-1}, in ascending tile order, are added as:
  chunk c = v_{32c} .. v_{32c+31} left-folded from its first element (s_c = ((v_{32c} + v_{32c+1}) + ...)),
  result = the left fold of the chunk sums in chunk order ((s_0 + s_1) + s_2) + ...
Every add is one float32 add, rounded to nearest (numpy float32 arithmetic)."""
import numpy as np

CHUNK = 32


def fold(values):
    """The documented association over one Gaussian's contributions: values [n, ...] float32 (n >= 1) -> [...] float32."""
    v = np.asarray(values, dtype=np.float32)
    total = None
    for c0 in range(0, v.shape[0], CHUNK):
        s = v[c0].copy()
        for j in range(c0 + 1, min(c0 + CHUNK, v.shape[0])):
            s = s + v[j]
        total = s if total is None else total + s
    return total


def fold_entries(gid, values):
    """fold() for every run of equal gids of an ordered entry list at once.  gid [n] (runs contiguous), values [n, 9] float32.
    Returns (gids [m], sums [m, 9] float32, counts [m], abs_sums [m, 9] float64 = sum |v|)."""
    gid = np.asarray(gid, dtype=np.int64)
    v = np.asarray(values, dtype=np.float32)
    n = gid.shape[0]
    if n == 0:
        return gid, np.zeros((0, 9), np.float32), np.zeros(0, np.int64), np.zeros((0, 9))
    head = np.ones(n, bool)
    head[1:] = gid[1:] != gid[:-1]
    seg_start = np.flatnonzero(head)
    seg = np.cumsum(head) - 1
    pos = np.arange(n) - seg_start[seg]
    chunk, within = pos // CHUNK, pos % CHUNK
    # chunks numbered globally in entry order: a chunk starts where within == 0
    chunk_id = np.cumsum(within == 0) - 1
    n_chunks = int(chunk_id[-1]) + 1
    csum = np.zeros((n_chunks, v.shape[1]), np.float32)
    for j in range(CHUNK):                             # left fold inside every chunk, all chunks at once
        sel = within == j
        if not sel.any():
            break
        csum[chunk_id[sel]] = v[sel] if j == 0 else csum[chunk_id[sel]] + v[sel]
    first = within == 0
    c_seg, c_idx = seg[first], chunk[first]
    m = seg_start.shape[0]
    tot = np.zeros((m, v.shape[1]), np.float32)
    for c in range(int(c_idx.max()) + 1):              # left fold of the chunk sums, all Gaussians at once
        sel = c_idx == c
        tot[c_seg[sel]] = csum[sel] if c == 0 else tot[c_seg[sel]] + csum[sel]
    counts = np.bincount(seg, minlength=m)
    abs_sums = np.zeros((m, v.shape[1]))
    np.add.at(abs_sums, seg, np.abs(v.astype(np.float64)))
    return gid[seg_start], tot, counts, abs_sums


def scatter(P, gids, sums):
    """The four 2-D gradient arrays (dL_dmeans2D [P,3], dL_dconic [P,4], dL_dopacity [P,1], dL_dcolors [P,3]) the reduction
    writes, zero where a row has no contribution."""
    out = dict(dL_dmeans2D=np.zeros((P, 3), np.float32), dL_dconic=np.zeros((P, 4), np.float32),
               dL_dopacity=np.zeros((P, 1), np.float32), dL_dcolors=np.zeros((P, 3), np.float32))
    out["dL_dmeans2D"][gids, 0:2] = sums[:, 0:2]
    out["dL_dconic"][gids, 0] = sums[:, 2]
    out["dL_dconic"][gids, 1] = sums[:, 3]
    out["dL_dconic"][gids, 3] = sums[:, 4]
    out["dL_dcolors"][gids] = sums[:, 5:8]
    out["dL_dopacity"][gids, 0] = sums[:, 8]
    return out


def gamma(k, u=2.0 ** -24):
    """gamma_k = k u / (1 - k u): the bound on the relative error of k float32 adds"""
    k = np.asarray(k, dtype=np.float64)
    return k * u / (1.0 - k * u)
