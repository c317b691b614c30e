"""k-reciprocal re-ranking (Zhong et al., CVPR 2017) with the call contract of the reference's
ibl/utils/rerank.py:32-100 -- `re_ranking(q_g_dist, q_q_dist, g_g_dist, k1, k2, lambda_value)` -> re-ranked
query x gallery distances -- used by Evaluator.evaluate(rerank=True) (ibl/evaluators.py:194-199).

The reference walks the N = m + n rows in Python (np.where / np.intersect1d / np.unique per row, an inverted
index for the Jaccard term).  Two implementations follow it:

  * Host inputs (numpy arrays or CPU tensors, `device=None`), a CUDA device present and max(k1 + 1, k2) <= 128:
    the inputs are copied to the current CUDA device and re-ranked there by Engine.rerank_dense (ibl_rerank_dense,
    rerank.cu): dense neighbour lists, then the sparse stage of the evaluator's re-ranking, then the full [m,n]
    output, in the reference's arithmetic and summation order.  Workspace O(N * k1): no [N,N] temporary.  This is
    the call of the SFRS sampler refresh (examples/netvlad_img_sfrs.py:84).  The result comes back to the host.
  * CUDA-tensor inputs, an explicit `device=`, no CUDA device, or wider neighbour lists: the dense torch
    restatement below, on the inputs' (or the given) device.  It builds several [N,N] temporaries; the tests use
    it as an independent oracle for the device paths.

The torch restatement states the algorithm as dense set algebra:

  * neighbour lists      R   = the k1+1 nearest columns of each row of the row-max-normalised squared distances
  * k-reciprocal sets    Kr  [N,N] bool:  Kr[i,j]  <=>  j in R[i] and i in R[j]              (rerank.py:53-57)
  * half-size sets       Kc  the same with round(k1/2)+1 neighbours                           (rerank.py:60-64)
  * expansion            E   = Kr | ((Kr & [ |Kc[c] n Kr[i]| > 2/3 |Kc[c]| ]) @ Kc)   -- two 0/1 matrix products
                                                                                               (rerank.py:58-68)
  * encoding             V   = row-normalised exp(-dist) on E, optional mean over the k2 nearest rows
                                                                                               (rerank.py:69-77)
  * Jaccard              1 - t/(2-t),  t[i,r] = sum_j min(V[i,j], V[r,j]), evaluated over the non-zero columns
                         of each query row only                                                (rerank.py:78-92)

Both are pinned against the unmodified reference function on seeded inputs (tests/golden/rerank.npz,
tests/golden/rerank_sfrs.npz)."""
import numpy as np
import torch

__all__ = ["re_ranking"]


def _half(k1):
    return int(np.around(k1 / 2.0))          # banker's rounding, as the reference (rerank.py:61)


def _reciprocal_sets(rank_lists, width):
    """bool [N,N]: S[i,j] <=> j among the first `width` neighbours of i AND i among the first `width` of j."""
    N = rank_lists.shape[0]
    fwd = rank_lists[:, :width]                                   # [N,w]
    back = rank_lists[fwd][:, :, :width]                          # [N,w,w]: neighbours of each neighbour
    me = torch.arange(N, device=rank_lists.device).view(N, 1, 1)
    mutual = (back == me).any(dim=2)                              # [N,w]
    S = torch.zeros(N, N, dtype=torch.bool, device=rank_lists.device)
    rows = torch.arange(N, device=rank_lists.device).view(N, 1).expand_as(fwd)
    S[rows[mutual], fwd[mutual]] = True
    return S


def _on_host(a):
    return isinstance(a, np.ndarray) or (isinstance(a, torch.Tensor) and a.device.type == "cpu")


def re_ranking(q_g_dist, q_q_dist, g_g_dist, k1=20, k2=6, lambda_value=0.3, device=None):
    as_numpy = isinstance(q_g_dist, np.ndarray)
    m, n = q_g_dist.shape
    N = m + n
    if N < k1 + 1:
        raise ValueError("re_ranking needs at least k1 + 1 images")
    if (device is None and all(_on_host(a) for a in (q_g_dist, q_q_dist, g_g_dist)) and torch.cuda.is_available()
            and m >= 1 and n >= 1 and max(k1 + 1, k2) <= min(128, N)):
        # host arrays, as the SFRS sampler refresh passes them: the sparse device path (Engine.rerank_dense)
        from ..engine import Engine
        dev = torch.cuda.current_device()
        qg, qq, gg = (torch.as_tensor(a).to(dev).float().contiguous() for a in (q_g_dist, q_q_dist, g_g_dist))
        final = Engine.get(dev).rerank_dense(qg, qq, gg, k1, k2, lambda_value).cpu()
        return final.numpy() if as_numpy else final
    t = (lambda a: torch.as_tensor(a)) if device is None else (lambda a: torch.as_tensor(a).to(device))
    final = _re_ranking_torch(t(q_g_dist).float(), t(q_q_dist).float(), t(g_g_dist).float(), k1, k2, lambda_value)
    return final.cpu().numpy() if as_numpy else final


def _re_ranking_torch(qg, qq, gg, k1, k2, lambda_value):
    """The dense set-algebra restatement on qg's device -> final [m,n] there."""
    m, n = qg.shape
    N = m + n
    dist = torch.cat([torch.cat([qq, qg], dim=1), torch.cat([qg.t(), gg], dim=1)], dim=0)
    dist = dist.pow(2)
    dist = (dist / dist.max(dim=0, keepdim=True).values).t().contiguous()    # rerank.py:42-43
    width = k1 + 1
    # stable ascending order of the k1+1 smallest entries per row (the reference argsorts whole rows)
    rank_lists = torch.sort(dist, dim=1, stable=True).indices[:, : max(width, k2)]

    Kr = _reciprocal_sets(rank_lists, width)
    Kc = _reciprocal_sets(rank_lists, _half(k1) + 1)
    Krf, Kcf = Kr.float(), Kc.float()
    inter = Krf @ Kcf.t()                                          # |Kc[c] n Kr[i]|, exact small integers
    size = Kcf.sum(dim=1)
    take = Kr & (inter.double() > (2.0 / 3.0) * size.double().view(1, N))
    E = Kr | ((take.float() @ Kcf) > 0)

    w = torch.where(E, torch.exp(-dist), torch.zeros((), device=dist.device))
    V = w / w.sum(dim=1, keepdim=True)
    if k2 != 1:
        V = V[rank_lists[:, :k2]].mean(dim=1)                      # rerank.py:73-76

    od = dist[:m]
    jac = torch.empty(m, N, device=dist.device)
    Vt = V.t().contiguous()
    step = 64
    for i0 in range(0, m, step):
        rows = V[i0:min(i0 + step, m)]                             # [b,N] query rows only
        nz = rows != 0
        width_nz = int(nz.sum(dim=1).max().item())
        # columns of the non-zeros of each query row, padded with column 0 and weight 0
        order = torch.argsort(nz.to(torch.uint8), dim=1, descending=True, stable=True)[:, :width_nz]
        vals = torch.gather(rows, 1, order)                        # [b,w] (zeros on the padding)
        cols = Vt[order]                                           # [b,w,N]: V[:, j] for each listed column j
        tmin = torch.minimum(cols, vals.unsqueeze(2)).sum(dim=1)   # [b,N]
        jac[i0:i0 + rows.shape[0]] = 1.0 - tmin / (2.0 - tmin)
    final = jac * (1 - lambda_value) + od * lambda_value
    return final[:, m:]
