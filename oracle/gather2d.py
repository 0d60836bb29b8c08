"""float64 restatement of the gather-form input gradient of a many-to-one submanifold table (csrc/gather2d.cu).

Rule 3 of oracle/rulebook.py: a non-centre tap of row o reads the LOWEST row at pixel p(o) + delta_k, the centre tap is the
row itself.  So the scatter-form gradient din[nbr[k, o]] += dout[o] W_k^T equals, per row i,
    din[i] = W_c^T dout[i] + [i is the lowest row at p(i)] sum_{k != c} W_k^T S[p(i) - delta_k],
with S[p] the sum of dout over the rows at pixel p (ascending row order), read through the mirrored table
nbr[K - 1 - k, i] (= the lowest row at p(i) - delta_k for odd, centred kernels)."""
import numpy as np

from . import rulebook as orb


def representatives(indices, spatial_shape):
    """rep[i] = the lowest row at row i's coordinate."""
    uniq, winner = orb._lookup_table(indices, spatial_shape)
    lin = orb.linearize(np.asarray(indices, dtype=np.int64), spatial_shape)
    return winner[np.searchsorted(uniq, lin)].astype(np.int64)


def scatter_dgrad(dout, w, nbr):
    """din[nbr[k, o]] += dout[o] @ w[:, k, :]  (w: [C_out, K, C_in]), float64."""
    dout, w = np.asarray(dout, np.float64), np.asarray(w, np.float64)
    K, n = nbr.shape
    din = np.zeros((n, w.shape[2]))
    for k in range(K):
        o = np.nonzero(nbr[k] >= 0)[0]
        np.add.at(din, nbr[k, o], dout[o] @ w[:, k, :])
    return din


def group_sums(dout, rep):
    """S stored at each group's representative row: S[r] = sum of dout[o] over rep[o] == r, ascending o."""
    s = np.zeros_like(np.asarray(dout, np.float64))
    np.add.at(s, rep, np.asarray(dout, np.float64))       # (np.add.at is unbuffered: rows are added in index order)
    return s


def gather_dgrad(dout, w, nbr, rep, s=None):
    """The gather form (s: the group sums, default group_sums(dout, rep))."""
    dout, w = np.asarray(dout, np.float64), np.asarray(w, np.float64)
    K, n = nbr.shape
    c = K // 2
    if s is None:
        s = group_sums(dout, rep)
    din = dout @ w[:, c, :]
    is_rep = rep == np.arange(n)
    for k in range(K):
        if k == c:
            continue
        j = nbr[K - 1 - k]
        i = np.nonzero(is_rep & (j >= 0))[0]
        din[i] += s[j[i]] @ w[:, k, :]
    return din
