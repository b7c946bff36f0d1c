"""Float64 oracle of the k-NN query and of the appearance-feature similarity regulariser
(internal/metrics/appearance_feature_similarity_regularization_metrics.py, ``SimilarityRegularizationMixin.get_similarity_metric``).

``knn(queries, points, K)``: brute force, ties broken by the point index (a stable sort), in chunks of queries; returns (dists,
idx, gap) with gap the relative distance between the K-th and (K+1)-th squared distances per query (inf when N == K).  A query with
gap <= AMBIGUOUS may legitimately get another K-th neighbour from an fp32 search.
``similarity_metric(features, idx, dists, decay, lam, kind, dtype)``: the reference's formula restated in torch (gather, the
[S,K,K] similarities, the column weights, the triangular mask, the mean, times lambda), in ``dtype``; float64 is the oracle, float32
the reference's own arithmetic (e32 = its distance from the oracle).  Returns (loss, mean) with autograd to ``features``.
"""
import torch

AMBIGUOUS = 8 * 2.0 ** -23


def knn(queries, points, K, chunk=512):
    q = queries.to(torch.float64)
    p = points.to(torch.float64)
    n = p.shape[0]
    kk = min(K + 1, n)
    dists, idx, gap = [], [], []
    for a in range(0, q.shape[0], chunk):
        d = ((q[a:a + chunk, None, :] - p[None, :, :]) ** 2).sum(-1)
        sd, si = torch.sort(d, dim=1, stable=True)
        dists.append(sd[:, :K])
        idx.append(si[:, :K])
        if kk > K:
            gap.append((sd[:, K] - sd[:, K - 1]) / sd[:, K].clamp_min(1e-300))
        else:
            gap.append(torch.full((sd.shape[0],), float("inf"), dtype=torch.float64, device=sd.device))
    return torch.cat(dists), torch.cat(idx), torch.cat(gap)


def similarity_metric(features, idx, dists, decay, lam, kind, dtype=torch.float64, absolute=False):
    f = features.to(dtype)
    w = torch.exp(-decay * dists.to(dtype))                                        # [S,K]
    g = f[idx]                                                                     # [S,K,D]
    if kind == "cosine":
        nf = torch.nn.functional.normalize(g, dim=-1)
        sim = (nf[:, :, None, :] * nf[:, None, :, :]).sum(dim=-1)
    elif kind == "euclidean":
        sim = -torch.norm(g[:, :, None, :] - g[:, None, :, :], dim=-1)
    else:
        raise ValueError(kind)
    raw = -sim.abs() if absolute else -sim            # absolute: the mean of |r| w, the size of the terms the mean cancels
    weighted = raw * w[:, None, :]
    k = idx.shape[1]
    triu = torch.triu(torch.ones((k, k), dtype=torch.bool, device=f.device), diagonal=1)
    mean = weighted[:, triu].mean()
    return mean * lam, mean


def similarity_grad(features, idx, dists, decay, lam, kind, dtype=torch.float64, max_bytes=1 << 30):
    """(loss, mean, d loss / d features) of similarity_metric in dtype.  Large S runs in chunks of samples whose [s,K,K,D]
    intermediates fit in max_bytes; the chunk means are combined with their sample counts (S is the whole mean's count)."""
    s, k = idx.shape
    d = features.shape[1]
    chunk = max(1, max_bytes // (k * k * d * torch.finfo(dtype).bits // 8 * 4))
    f = features.detach().to(dtype).requires_grad_(True)
    mean_tot = torch.zeros((), dtype=dtype, device=features.device)
    grad = torch.zeros_like(f)
    for a in range(0, s, chunk):
        _, mean = similarity_metric(f, idx[a:a + chunk], dists[a:a + chunk], decay, 1.0, kind, dtype)
        part = mean * (idx[a:a + chunk].shape[0] / s)
        (g,) = torch.autograd.grad(part * lam, f)
        grad += g
        mean_tot += part.detach()
    return mean_tot * lam, mean_tot, grad
