"""Host mirror of the AHC initialisation (SURVEY.md 8f.3, VBx/vbhmm.py:131-152).

The O(T^2) work (cosine similarities, the two-Gaussian threshold calibration, the average-linkage clustering) runs
on the device behind `vbx_ahc` (csrc/vbx_ahc.cu).  What is left for the host is what the reference does with the
linkage matrix: cut it at the calibrated threshold (VBx/vbhmm.py:142-146, scipy's `fcluster(..., 'distance')`) and
number the flat clusters.  `flat_clusters` reproduces scipy's numbering, so the speaker columns of the initial gamma
come out in the reference's order.
"""
import ctypes

import numpy as np
import torch



def flat_clusters(Z, t):
    """fcluster(Z, t, criterion='distance') for a monotone linkage Z [T-1,4] (scipy layout); returns labels 1..K [T].

    scipy's numbering: walk down from the root; the first node on a path whose height is <= t becomes a flat cluster
    and takes the next number.  At every node the non-leaf children are explored first (left, then right), and only
    then are its leaf children (left, then right) labelled - with the enclosing cluster's number, or as new
    singletons."""
    Z = np.asarray(Z, dtype=np.float64)
    n = Z.shape[0] + 1
    labels = np.zeros(n, dtype=np.int32)
    if n == 1:
        labels[0] = 1
        return labels
    left = Z[:, 0].astype(np.int64).tolist()
    right = Z[:, 1].astype(np.int64).tolist()
    height = np.maximum.accumulate(Z[:, 2]).tolist()   # max height inside the subtree (UPGMA heights are sorted)
    visited = [False] * (n - 1)
    k = 0
    leader = -1
    path = [n - 2]                                     # merge rows on the current root-to-node path
    while path:
        r = path[-1]
        lc, rc = left[r], right[r]
        if leader == -1 and height[r] <= t:
            leader = r
            k += 1
        if lc >= n and not visited[lc - n]:
            visited[lc - n] = True
            path.append(lc - n)
            continue
        if rc >= n and not visited[rc - n]:
            visited[rc - n] = True
            path.append(rc - n)
            continue
        for c in (lc, rc):
            if c < n:
                if leader == -1:
                    k += 1
                labels[c] = k
        if leader == r:
            leader = -1
        path.pop()
    return labels


def ahc_batch(vb, x, threshold=-0.015, workspace=None):
    """AHC labels for every recording of the planned batch `vb` (VbxBatch).  x: [N,dim] float32 or float64 CUDA tensor
    of transformed x-vectors (the output of VBx/vbhmm.py:129).  Returns (labels, thr, Z): a list of int arrays
    (0-based cluster ids, VBx/vbhmm.py:145-146), the calibrated thresholds [B] and the linkage matrices (list)."""
    th, Zs = linkage_batch(vb, x, workspace)
    return cut(Zs, th, vb.lengths, threshold), th, Zs


def linkage_batch(vb, x, workspace=None):
    """The device half of ahc_batch: vbx_ahc on every recording of `vb`, its outputs copied to the host.  Returns (the
    calibrated thresholds [B], the linkage matrices (list)); cut() turns them into labels."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.is_contiguous() and x.dim() == 2 and x.shape[0] == vb.N
            and x.dtype in (torch.float32, torch.float64)):
        raise ValueError('x: expected a contiguous float32/float64 CUDA tensor of shape [N, dim]')
    need = ctypes.c_size_t()
    vb._check(vb.lib.vbx_ahc_workspace_bytes(vb._h, ctypes.byref(need)))
    if workspace is None:
        workspace = torch.empty(int(need.value), dtype=torch.uint8, device=vb.device)
    Z = torch.empty((vb.N, 4), dtype=torch.float64, device=vb.device)
    thr = torch.empty(vb.B, dtype=torch.float64, device=vb.device)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    vb._check(vb.lib.vbx_ahc(vb._h, ptr(x), int(x.dtype == torch.float64), int(x.shape[1]), ptr(workspace),
                             workspace.numel(), ptr(Z), ptr(thr), vb._stream()))
    Zh, th = Z.cpu().numpy(), thr.cpu().numpy()       # 32 B per x-vector leave the device
    Zs = [Zh[int(vb.offsets[b]):int(vb.offsets[b + 1]) - 1] if vb.offsets[b + 1] > vb.offsets[b] else Zh[0:0]
          for b in range(vb.B)]
    return th, Zs


def cut(Zs, th, lengths, threshold):
    """VBx/vbhmm.py:144-146 for every recording: the 0-based flat clusters of linkage Zs[b] at the calibrated threshold
    th[b] shifted by `threshold`.  Host work only, so a threshold sweep repeats this and nothing else."""
    labels = []
    for b, T in enumerate(lengths):
        if T == 0:
            labels.append(np.zeros(0, dtype=np.int64))
        elif T == 1:
            labels.append(np.zeros(1, dtype=np.int64))
        elif not np.isfinite(Zs[b]).all():
            # a NaN or infinite x-vector: its distances are NaN, so the linkage stops before it (its last rows are
            # NaN) and the calibrated threshold is NaN as well; like any NaN cut, every x-vector stays on its own
            labels.append(np.arange(T, dtype=np.int64))
        else:
            # a degenerate calibration (NaN threshold, e.g. two x-vectors) leaves every x-vector on its own, exactly
            # what the reference's fcluster call does with a NaN cut
            labels.append(flat_clusters(Zs[b], -(th[b] + threshold)).astype(np.int64) - 1)
    return labels


def cut_count(Zs, lengths, counts):
    """scipy's fcluster(Z, k, criterion='maxclust') for every recording, k = counts[b]: the 0-based flat clusters of
    linkage Zs[b] cut at the lowest merge height that leaves at most k clusters, numbered like flat_clusters.  Merges at
    a tied height all happen together, so ties can leave fewer than k clusters, exactly as in scipy; k >= T leaves every
    x-vector on its own.  A linkage with non-finite heights leaves every x-vector on its own, as cut() does."""
    labels = []
    for b, T in enumerate(lengths):
        T, k = int(T), int(counts[b])
        if k < 1:
            raise ValueError(f'cluster count must be >= 1, got {k}')
        Z = np.asarray(Zs[b], dtype=np.float64)
        if T <= 1:
            labels.append(np.zeros(T, dtype=np.int64))
        elif k >= T or not np.isfinite(Z).all():
            labels.append(np.arange(T, dtype=np.int64))      # scipy numbers singletons in x-vector order
        else:
            # the clusters left at height t are T minus the merges whose subtree height is <= t
            height = np.sort(np.maximum.accumulate(Z[:, 2]))
            labels.append(flat_clusters(Z, height[T - k - 1]).astype(np.int64) - 1)
    return labels
