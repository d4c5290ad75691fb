"""Gallery-vs-query ranking on device: one similarity GEMM + a sort-free CMC / AP kernel.

Replaces the per-query Python loop of ``tools/evaluate.py:88-142`` (one ``torch.mm`` + ``.cpu()`` + ``np.argsort`` +
numpy set ops per query) with two kernel launches and a single device->host copy of the final numbers.
"""
from __future__ import annotations

from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import native
from .gemm import gemm


def similarity(query: torch.Tensor, gallery: torch.Tensor, precise: bool = True) -> torch.Tensor:
    """``S[q, g] = <query_q, gallery_g>`` in fp32. With ``precise`` the bf16 tensor-core GEMM is run on a
    hi/lo split of both operands (3 passes) which recovers ~fp32 accuracy for L2-normalised features."""
    if not query.is_cuda:
        return query.float() @ gallery.float().t()
    q, g = query.float().contiguous(), gallery.float().contiguous()
    k = q.shape[1]
    if k % 8:  # TMA needs 16-byte row strides
        pad = 8 - k % 8
        q = torch.nn.functional.pad(q, (0, pad))
        g = torch.nn.functional.pad(g, (0, pad))
    q_hi, g_hi = q.to(torch.bfloat16), g.to(torch.bfloat16)
    s = gemm(q_hi, g_hi, out_dtype=torch.float32)
    if precise:
        q_lo = (q - q_hi.float()).to(torch.bfloat16)
        g_lo = (g - g_hi.float()).to(torch.bfloat16)
        s += gemm(q_lo, g_hi, out_dtype=torch.float32)
        s += gemm(q_hi, g_lo, out_dtype=torch.float32)
    return s


def rank_metrics_reference(sim: torch.Tensor, q_labels: torch.Tensor, g_labels: torch.Tensor
                           ) -> Tuple[np.ndarray, float]:
    """Straightforward (sorting) CPU implementation with the semantics of ``tools/evaluate.py``."""
    sim = sim.detach().cpu().float().numpy()
    ql = q_labels.cpu().numpy()
    gl = g_labels.cpu().numpy()
    nq, ng = sim.shape
    total_cmc = np.zeros(ng, dtype=np.float64)
    total_ap = 0.0
    for i in range(nq):
        order = np.argsort(sim[i], kind="stable")[::-1]
        hits = np.flatnonzero(gl[order] == ql[i])
        if hits.size == 0:
            continue
        total_cmc[hits[0]:] += 1
        ap = 0.0
        for j, loc in enumerate(hits):
            precision = (j + 1) / (loc + 1)
            old = j / loc if loc != 0 else 1.0
            ap += (old + precision) / 2 / hits.size
        total_ap += ap
    return total_cmc / nq, total_ap / nq


def rank_metrics(sim: torch.Tensor, q_labels: torch.Tensor, g_labels: torch.Tensor) -> Tuple[np.ndarray, float]:
    """CMC curve (length G, float64) and mAP from a similarity matrix. Queries with no match are skipped but still
    count in the denominator (``tools/evaluate.py:137-142``)."""
    if not native.on_device(sim, "flpr_rank_eval"):
        return rank_metrics_reference(sim, q_labels, g_labels)
    nq, ng = sim.shape
    lib = native.kernels()
    sim = sim.float().contiguous()
    ql = q_labels.to(sim.device).long().contiguous()
    gl = g_labels.to(sim.device).long().contiguous()
    ap = torch.empty(nq, dtype=torch.float32, device=sim.device)
    first = torch.empty(nq, dtype=torch.int32, device=sim.device)
    rc = lib.flpr_rank_eval(native.ptr(sim), native.ptr(ql), native.ptr(gl), native.ptr(ap), native.ptr(first), nq, ng,
                            sim.stride(0), native.stream_of(sim.device))
    native.check(rc, "flpr_rank_eval")
    native.count_launch()
    valid = first >= 0
    hist = torch.bincount(first[valid].long(), minlength=ng).double()
    cmc = torch.cumsum(hist, 0) / nq
    m_ap = ap.double().sum() / nq
    out = torch.cat([cmc, m_ap.view(1)]).cpu().numpy()  # single D2H
    return out[:-1], float(out[-1])


def rank_metrics_with_cameras(sim: torch.Tensor, q_labels: torch.Tensor, g_labels: torch.Tensor,
                              q_cameras: torch.Tensor, g_cameras: torch.Tensor) -> Tuple[np.ndarray, float]:
    """CMC / mAP with the reference's junk rule (``tools/evaluate.py:12-33,60-67``): gallery items of the query's
    identity *seen by the query's camera*, and mis-detections (label ``-1``), are removed from the ranking; the hits
    are the same identity under another camera. Tensor ops on ``sim``'s device (counts instead of a sort per query):

        position(hit) = #{non-junk g : S[q, g] > s_hit},   index among hits = #{hits h : s_h > s_hit}
    """
    dev = sim.device
    ql, gl = q_labels.to(dev).long().view(-1, 1), g_labels.to(dev).long().view(1, -1)
    qc, gc = q_cameras.to(dev).long().view(-1, 1), g_cameras.to(dev).long().view(1, -1)
    nq, ng = sim.shape
    same_id, same_cam = gl == ql, gc == qc
    junk = (same_id & same_cam) | (gl == -1)
    hit = same_id & ~same_cam
    neg = torch.finfo(torch.float32).min
    s = sim.float()
    keep = torch.where(junk, torch.full_like(s, neg), s)                 # junk can never outrank anything
    s_sorted, _ = torch.sort(keep, dim=1)
    h_sorted, _ = torch.sort(torch.where(hit, s, torch.full_like(s, neg)), dim=1)
    loc = (ng - torch.searchsorted(s_sorted, s.contiguous(), right=True)).double()      # [Q, G], valid where hit
    j = (ng - torch.searchsorted(h_sorted, s.contiguous(), right=True)).double()
    n_hits = hit.sum(1).double()
    precision = (j + 1) / (loc + 1)
    old = torch.where(loc > 0, j / loc.clamp(min=1), torch.ones_like(loc))
    ap = torch.where(hit, (old + precision) / 2, torch.zeros_like(loc)).sum(1) / n_hits.clamp(min=1)
    has = n_hits > 0
    first = torch.where(hit, loc, torch.full_like(loc, float(ng))).min(1).values.long()
    hist = torch.bincount(first[has], minlength=ng)[:ng].double()
    # the reference's per-query curve keeps the full gallery length even after junk removal (evaluate.py:53,72)
    cmc = torch.cumsum(hist, 0) / nq
    out = torch.cat([cmc, ((ap * has).sum() / nq).view(1)]).cpu().numpy()
    return out[:-1], float(out[-1])


def evaluate(query_features: torch.Tensor, query_labels: torch.Tensor, gallery_features: torch.Tensor,
             gallery_labels: torch.Tensor, query_camera_labels: torch.Tensor | None = None,
             gallery_camera_labels: torch.Tensor | None = None, device: str | torch.device | None = None,
             precise: bool = True, re_ranking: Optional[Dict] = None) -> Tuple[np.ndarray, float]:
    """Drop-in for ``tools.evaluate.evaluate`` (same positional order). Camera labels are optional - the reference's
    runtime never passes them - and switch on its same-camera / mis-detection junk rule.

    ``re_ranking``: ``None`` (plain ranking) or a dict of :func:`re_ranking`'s ``k1`` / ``k2`` / ``lambda_value``
    (missing keys take the defaults); the queries are then ranked by the negated re-ranked distance."""
    if device is not None:
        query_features = query_features.to(device)
        gallery_features = gallery_features.to(device)
    rr = re_ranking_params(re_ranking)
    if rr is not None:
        sim = -_re_ranking(query_features, gallery_features, **rr)
    else:
        sim = similarity(query_features, gallery_features, precise=precise)
    if query_camera_labels is not None and gallery_camera_labels is not None:
        return rank_metrics_with_cameras(sim, query_labels, gallery_labels, query_camera_labels,
                                         gallery_camera_labels)
    return rank_metrics(sim, query_labels, gallery_labels)


# ------------------------------------------------------------------------------------------------- gallery-sharded
def evaluate_sharded(query_features: torch.Tensor, query_labels: torch.Tensor, gallery_shard: torch.Tensor,
                     gallery_shard_labels: torch.Tensor, group=None, precise: bool = True
                     ) -> Tuple[np.ndarray, float]:
    """Exact CMC / mAP when the **gallery is sharded over the ranks** of ``group`` (SURVEY §5.7: the dimension that
    scales in this workload is the gallery, the analogue of sequence parallelism is to give every rank a slice of it).

    Every rank scores its shard against all queries. A hit's position in the global ranking is the number of gallery
    items that score higher, and that count is a *sum over shards* - so instead of gathering the ``Q x G`` similarity
    matrix (or merging sorted lists) the ranks exchange only the similarities of the hits (``Q x P``, ``P`` = matches per
    query and shard) and all-reduce two small count tensors:

        above[r, q, p]     = #{g in shard_r : S[q, g] > s_p}            -> position of hit p in the full ranking
        hits_above[r, q, p] = #{g in shard_r : S[q, g] > s_p, g a hit}  -> index of hit p among the hits

    from which AP (the reference's trapezoid form, ``tools/evaluate.py:75-82``) and the first-hit position (CMC) follow
    locally and identically on every rank. Returns what :func:`evaluate` returns on the concatenated gallery.
    Without an initialised process group (or ``world == 1``) this *is* :func:`evaluate`.
    """
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return evaluate(query_features, query_labels, gallery_shard, gallery_shard_labels, precise=precise)
    world = dist.get_world_size(group)
    dev = query_features.device
    sim = similarity(query_features, gallery_shard, precise=precise)                   # [Q, Gr]
    ql = query_labels.to(dev).long()
    gl = gallery_shard_labels.to(dev).long()
    nq, ngr = sim.shape
    match = gl.view(1, -1) == ql.view(-1, 1)                                           # [Q, Gr]
    # ---- exchange the hit similarities (padded to the largest per-shard hit count) -----------------------------------
    sizes = torch.tensor([int(match.sum(1).max()) if ngr else 0, ngr], device=dev, dtype=torch.long)
    size_list = [torch.empty_like(sizes) for _ in range(world)]
    dist.all_gather(size_list, sizes, group=group)
    pmax = max(int(s[0]) for s in size_list)
    ng_total = sum(int(s[1]) for s in size_list)
    if pmax == 0:
        return np.zeros(ng_total, dtype=np.float64), 0.0
    neg = torch.finfo(torch.float32).min
    # hits first (stable), then padding
    order = torch.argsort((~match).to(torch.int8), dim=1, stable=True)[:, :pmax] if ngr else \
        torch.zeros(nq, 0, dtype=torch.long, device=dev)
    mine = torch.full((nq, pmax), neg, dtype=torch.float32, device=dev)
    valid = torch.zeros(nq, pmax, dtype=torch.bool, device=dev)
    if ngr:
        k = order.shape[1]
        valid[:, :k] = match.gather(1, order)
        mine[:, :k] = torch.where(valid[:, :k], sim.gather(1, order), torch.full_like(mine[:, :k], neg))
    hit_list = [torch.empty_like(mine) for _ in range(world)]
    val_list = [torch.empty(nq, pmax, dtype=torch.uint8, device=dev) for _ in range(world)]
    dist.all_gather(hit_list, mine.contiguous(), group=group)
    dist.all_gather(val_list, valid.to(torch.uint8).contiguous(), group=group)
    hits = torch.stack(hit_list, 1).reshape(nq, world * pmax)                           # [Q, W*P]
    hvalid = torch.stack(val_list, 1).reshape(nq, world * pmax).bool()
    # ---- local counts: sorted shard rows + searchsorted ---------------------------------------------------------------
    if ngr:
        s_sorted, _ = torch.sort(sim, dim=1)                                            # ascending
        above = ngr - torch.searchsorted(s_sorted, hits.contiguous(), right=True)       # strictly greater
        pos_only = torch.where(match, sim, torch.full_like(sim, neg))
        p_sorted, _ = torch.sort(pos_only, dim=1)
        hits_above = ngr - torch.searchsorted(p_sorted, hits.contiguous(), right=True)
    else:
        above = torch.zeros_like(hits, dtype=torch.long)
        hits_above = torch.zeros_like(hits, dtype=torch.long)
    counts = torch.stack([above, hits_above]).to(torch.int64)
    dist.all_reduce(counts, group=group)
    loc, j = counts[0].double(), counts[1].double()                                     # 0-based rank / hit index
    # ---- AP and first hit ----------------------------------------------------------------------------------------------
    n_hits = hvalid.sum(1).double()
    precision = (j + 1) / (loc + 1)
    old = torch.where(loc > 0, j / loc.clamp(min=1), torch.ones_like(loc))
    ap = (torch.where(hvalid, (old + precision) / 2, torch.zeros_like(loc)).sum(1) / n_hits.clamp(min=1))
    has = n_hits > 0
    first = torch.where(hvalid, loc, torch.full_like(loc, float(ng_total))).min(1).values.long()
    hist = torch.bincount(first[has], minlength=ng_total)[:ng_total].double()
    cmc = torch.cumsum(hist, 0) / nq
    m_ap = (ap * has).sum() / nq
    out = torch.cat([cmc, m_ap.view(1)]).cpu().numpy()
    return out[:-1], float(out[-1])


# ------------------------------------------------------------------------------------------------- k-reciprocal re-ranking
RE_RANKING_DEFAULTS = {"k1": 20, "k2": 6, "lambda_value": 0.3}


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def check_re_ranking_params(k1, k2, lambda_value) -> Tuple[int, int, float]:
    """``1 <= k1 <= 63`` (a row's ``k1 + 1`` neighbours fit two per lane of one warp), ``1 <= k2 <= k1 + 1``,
    ``0 <= lambda_value <= 1``; anything else raises ``ValueError``."""
    if not _is_int(k1) or not 1 <= k1 <= 63:
        raise ValueError(f"re-ranking k1 must be an integer in [1, 63], got {k1!r}")
    if not _is_int(k2) or not 1 <= k2 <= k1 + 1:
        raise ValueError(f"re-ranking k2 must be an integer in [1, k1 + 1 = {k1 + 1}], got {k2!r}")
    if isinstance(lambda_value, bool) or not isinstance(lambda_value, (int, float, np.floating)) \
            or not 0.0 <= float(lambda_value) <= 1.0:
        raise ValueError(f"re-ranking lambda_value must be a number in [0, 1], got {lambda_value!r}")
    return int(k1), int(k2), float(lambda_value)


def re_ranking_params(spec) -> Optional[Dict]:
    """``engine_opts.re_ranking`` / ``evaluate(re_ranking=...)`` -> ``None`` (off) or a full, checked parameter dict.
    ``False`` / ``None``: off; ``True``: the defaults; a dict: its keys over the defaults."""
    if spec is None or spec is False:
        return None
    if spec is True:
        spec = {}
    if not isinstance(spec, dict):
        raise ValueError(f"re_ranking must be false, true or a dict of k1 / k2 / lambda_value, got {spec!r}")
    unknown = set(spec) - set(RE_RANKING_DEFAULTS)
    if unknown:
        raise ValueError(f"unknown re_ranking parameters {sorted(unknown)} (known: k1, k2, lambda_value)")
    p = dict(RE_RANKING_DEFAULTS, **spec)
    k1, k2, lam = check_re_ranking_params(p["k1"], p["k2"], p["lambda_value"])
    return {"k1": k1, "k2": k2, "lambda_value": lam}


def _expansion_h(k1: int) -> int:
    return int(round(k1 / 2)) + 1          # Python's round: half to even


# ---- float64 reference (the test oracle; also what CPU tensors run) ------------------------------------------------------
def re_ranking_distance_reference(query: torch.Tensor, gallery: torch.Tensor) -> torch.Tensor:
    """Step 1 in float64 on the inputs' device: squared euclidean distances of ``X = cat(query, gallery)``, clamped at 0,
    zero diagonal, every row divided by its maximum (an all-zero row stays zero)."""
    x = torch.cat([query, gallery]).double()
    sq = (x * x).sum(1)
    d = (sq.view(-1, 1) + sq.view(1, -1) - 2.0 * (x @ x.t())).clamp_min(0.0)
    d.fill_diagonal_(0.0)
    mx = d.max(1, keepdim=True).values
    return torch.where(mx > 0, d / torch.where(mx > 0, mx, torch.ones_like(mx)), d)


def re_ranking_topk_reference(D: torch.Tensor, k1: int, rows=None, chunk: int = 1024) -> torch.Tensor:
    """Step 2: ``R[i, :K]``, ``K = min(k1 + 1, N)``: stable ascending sort of ``D[i]`` (ties to the lower index).
    ``rows``: only these rows (int64 ``[len(rows), K]``), else all. Runs on ``D``'s device, chunked."""
    n = D.shape[0]
    k = min(k1 + 1, n)
    rows = torch.arange(n, device=D.device) if rows is None else torch.as_tensor(rows, device=D.device).long()
    out = []
    for s in range(0, len(rows), chunk):
        blk = D[rows[s:s + chunk]].double()
        out.append(torch.sort(blk, dim=1, stable=True).indices[:, :k])
    return torch.cat(out) if out else torch.zeros(0, k, dtype=torch.long, device=D.device)


def re_ranking_encode_reference(d_row, R: np.ndarray, i: int, k1: int):
    """Steps 3-5 for row ``i`` alone: ``(K(i), E(i), weights)``. ``d_row``: ``D[i, :]``; ``R``: the full initial ranking
    (int numpy ``[N, K]``). ``K(i)`` is in ``R[i]``'s order, ``E(i)`` ascending, ``weights`` float64 over ``E(i)``."""
    R = np.asarray(R)
    K = R.shape[1]
    h = min(_expansion_h(k1), K)
    F = R[i, :K]
    Ki = F[(R[F, :K] == i).any(1)]
    E = [int(v) for v in Ki]
    for c in Ki:
        fw = R[c, :h]
        Kc = fw[(R[fw, :h] == c).any(1)]
        inter = int(np.isin(Kc, Ki).sum())
        if 3 * inter > 2 * len(Kc):                     # |Kc n K(i)| > (2/3) |Kc|
            E.extend(int(v) for v in Kc)
    E = np.array(sorted(set(E)), dtype=np.int64)
    d = torch.as_tensor(d_row).double().cpu().numpy()
    w = np.exp(-d[E])
    if len(E):
        w = w / w.sum()
    return [int(v) for v in Ki], E, w


def re_ranking_reference(query: torch.Tensor, gallery: torch.Tensor, k1: int = 20, k2: int = 6,
                         lambda_value: float = 0.3, distance: Optional[torch.Tensor] = None, details: bool = False):
    """k-reciprocal re-ranking, a plain float64 transcription of the eight steps (DESIGN §3). Returns the ``[Q, G]``
    float64 distance on the inputs' device; ``distance``: start from this ``D`` (step 1 skipped). ``details``: also a
    dict of the intermediates ``D, R, K, E, V, Vq`` (dense ``V`` / ``Vq``, lists of index arrays ``K`` / ``E``)."""
    k1, k2, lambda_value = check_re_ranking_params(k1, k2, lambda_value)
    nq = query.shape[0]
    D = re_ranking_distance_reference(query, gallery) if distance is None else distance.double()
    dev = D.device
    n = D.shape[0]
    R = re_ranking_topk_reference(D, k1).cpu().numpy()
    Dc = D.cpu().numpy()
    V = np.zeros((n, n), dtype=np.float64)
    Ks, Es = [], []
    for i in range(n):
        Ki, Ei, w = re_ranking_encode_reference(Dc[i], R, i, k1)
        V[i, Ei] = w
        Ks.append(Ki)
        Es.append(Ei)
    Vt = torch.from_numpy(V).to(dev)
    if k2 != 1:                                            # local query expansion: mean over R[i, :k2] (clamped)
        kk = min(k2, R.shape[1])
        Rt = torch.from_numpy(R[:, :kk]).to(dev)
        Vq = torch.zeros_like(Vt)
        for r in range(kk):
            Vq += Vt[Rt[:, r]]
        Vq /= kk
    else:
        Vq = Vt
    final = torch.empty(nq, n - nq, dtype=torch.float64, device=dev)
    Vg = Vq[nq:]
    for i in range(nq):
        nz = torch.nonzero(Vq[i]).flatten()
        m = torch.minimum(Vq[i, nz].view(1, -1), Vg[:, nz]).sum(1)
        final[i] = 1.0 - m / (2.0 - m)
    final = (1.0 - lambda_value) * final + lambda_value * D[:nq, nq:]
    if details:
        return final, {"D": D, "R": R, "K": Ks, "E": Es, "V": V, "Vq": Vq.cpu().numpy()}
    return final


# ---- native stages -------------------------------------------------------------------------------------------------------
class SparseRows(NamedTuple):
    """Fixed-capacity sparse rows: row ``i`` holds ``nnz[i]`` entries ``cols[i, :nnz[i]]`` (ascending) / ``vals``."""
    cols: torch.Tensor     # int32 [N, cap]
    vals: torch.Tensor     # fp32  [N, cap]
    nnz: torch.Tensor      # int32 [N]

    def dense(self, n: int) -> torch.Tensor:
        out = torch.zeros(self.cols.shape[0], n, dtype=torch.float64, device=self.cols.device)
        cap = self.cols.shape[1]
        mask = torch.arange(cap, device=self.cols.device).view(1, -1) < self.nnz.view(-1, 1).long()
        r = torch.arange(self.cols.shape[0], device=self.cols.device).view(-1, 1).expand(-1, cap)
        out[r[mask], self.cols.long()[mask]] = self.vals.double()[mask]
        return out


def _rr_call(name: str, *args) -> None:
    lib = native.kernels()
    native.check(getattr(lib, name)(*args), name)
    native.count_launch()


def rr_distance(S: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """Step 1 on the kernels: ``S = x x^T`` (fp32 ``[N, N]``, contiguous) becomes ``D`` in place; ``x``: the features."""
    x = x.float().contiguous()
    n = x.shape[0]
    sqn = torch.empty(n, dtype=torch.float32, device=x.device)
    st = native.stream_of(x.device)
    _rr_call("flpr_rr_sqnorm", native.ptr(x), native.ptr(sqn), n, x.shape[1], x.stride(0), st)
    _rr_call("flpr_rr_distance", native.ptr(S), native.ptr(sqn), n, S.stride(0), st)
    return S


def rr_topk(D: torch.Tensor, k1: int) -> torch.Tensor:
    """Step 2: int32 ``[N, min(k1 + 1, N)]``."""
    n = D.shape[0]
    k = min(k1 + 1, n)
    R = torch.empty(n, k, dtype=torch.int32, device=D.device)
    _rr_call("flpr_rr_topk", native.ptr(D), native.ptr(R), n, k, D.stride(0), native.stream_of(D.device))
    return R


def rr_encode(D: torch.Tensor, R: torch.Tensor, k1: int) -> SparseRows:
    """Steps 3-5: the weighted k-reciprocal expansion of every row (capacity ``K (h + 1)``)."""
    n, k = R.shape
    hh = min(_expansion_h(k1), k)
    cap = k * (hh + 1)
    cols = torch.zeros(n, cap, dtype=torch.int32, device=D.device)
    vals = torch.zeros(n, cap, dtype=torch.float32, device=D.device)
    nnz = torch.empty(n, dtype=torch.int32, device=D.device)
    _rr_call("flpr_rr_encode", native.ptr(D), native.ptr(R), native.ptr(cols), native.ptr(vals), native.ptr(nnz), n, k,
             hh, cap, D.stride(0), native.stream_of(D.device))
    return SparseRows(cols, vals, nnz)


def rr_expand(V: SparseRows, R: torch.Tensor, k2: int) -> SparseRows:
    """Step 6: ``V'_i = mean_{r < k2} V_{R[i, r]}`` (``k2`` clamped to ``R``'s width); ``k2 == 1`` returns ``V``."""
    if k2 == 1:
        return V
    n, k = R.shape
    k2 = min(k2, k)
    cap = V.cols.shape[1]
    ocap = k2 * cap
    cols = torch.zeros(n, ocap, dtype=torch.int32, device=R.device)
    vals = torch.zeros(n, ocap, dtype=torch.float32, device=R.device)
    nnz = torch.empty(n, dtype=torch.int32, device=R.device)
    _rr_call("flpr_rr_expand", native.ptr(V.cols), native.ptr(V.vals), native.ptr(V.nnz), native.ptr(R),
             native.ptr(cols), native.ptr(vals), native.ptr(nnz), n, k, k2, cap, ocap, native.stream_of(R.device))
    return SparseRows(cols, vals, nnz)


def rr_index(Vq: SparseRows, num_query: int):
    """Inverted index of the gallery rows of ``V'``: ``(off [N + 1], row [E], val [E])``; the entries of column ``j``
    are ``off[j] .. off[j + 1]`` (gallery rows numbered from 0)."""
    n, cap = Vq.cols.shape
    g = n - num_query
    dev = Vq.cols.device
    total = int(Vq.nnz[num_query:].sum()) if g > 0 else 0
    cnt = torch.empty(n, dtype=torch.int32, device=dev)
    off = torch.empty(n + 1, dtype=torch.int32, device=dev)
    rows = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
    vals = torch.empty(max(total, 1), dtype=torch.float32, device=dev)
    _rr_call("flpr_rr_index", native.ptr(Vq.cols), native.ptr(Vq.vals), native.ptr(Vq.nnz), num_query, g, n, cap,
             native.ptr(cnt), native.ptr(off), native.ptr(rows), native.ptr(vals), native.stream_of(dev))
    return off, rows, vals


def rr_jaccard(Vq: SparseRows, D: torch.Tensor, num_query: int, lambda_value: float, tile: int = 0) -> torch.Tensor:
    """Steps 7-8: ``[Q, G]`` fp32 ``(1 - lambda) J + lambda D[:Q, Q:]``. ``tile``: gallery items per block (0 = as many
    as fit in shared memory)."""
    n = D.shape[0]
    g = n - num_query
    off, rows, vals = rr_index(Vq, num_query)
    out = torch.empty(num_query, g, dtype=torch.float32, device=D.device)
    _rr_call("flpr_rr_jaccard", native.ptr(Vq.cols), native.ptr(Vq.vals), native.ptr(Vq.nnz), Vq.cols.shape[1],
             native.ptr(off), native.ptr(rows), native.ptr(vals), native.ptr(D), D.stride(0), native.ptr(out),
             num_query, g, int(tile), float(lambda_value), native.stream_of(D.device))
    return out


def re_ranking_from_distance(D: torch.Tensor, num_query: int, k1: int = 20, k2: int = 6, lambda_value: float = 0.3,
                             tile: int = 0) -> torch.Tensor:
    """Steps 2-8 on the kernels, from a given fp32 ``D`` (``[N, N]``, contiguous, as :func:`rr_distance` leaves it)."""
    k1, k2, lambda_value = check_re_ranking_params(k1, k2, lambda_value)
    R = rr_topk(D, k1)
    V = rr_encode(D, R, k1)
    Vq = rr_expand(V, R, k2)
    return rr_jaccard(Vq, D, num_query, lambda_value, tile)


def re_ranking(query: torch.Tensor, gallery: torch.Tensor, k1: int = 20, k2: int = 6,
               lambda_value: float = 0.3) -> torch.Tensor:
    """k-reciprocal re-ranking (Zhong et al., CVPR 2017): ``[Q, G]`` fp32 distance, smaller = more similar.

    CUDA tensors: the similarity GEMM of :func:`similarity` (hi/lo split, ~fp32) and the stages of ``csrc/rerank.cu``;
    memory is about ``4 N^2`` bytes for ``D`` plus ``O(N k2 cap)`` for the sparse rows (``N = Q + G``). CPU tensors:
    :func:`re_ranking_reference` in float64, returned as fp32."""
    k1, k2, lambda_value = check_re_ranking_params(k1, k2, lambda_value)
    if not native.on_device(query, "flpr_rr_topk"):
        return re_ranking_reference(query, gallery, k1, k2, lambda_value).float()
    x = torch.cat([query, gallery]).float().contiguous()
    D = rr_distance(similarity(x, x, precise=True).contiguous(), x)
    return re_ranking_from_distance(D, query.shape[0], k1, k2, lambda_value)


_re_ranking = re_ranking
