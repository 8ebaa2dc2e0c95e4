"""Exact expected results of one contig-mode sample on the device ABI, from the sorted delta events of each contig instead of
a dense depth array: the same rules as tests/device_reference.py::expected (whose helpers it reuses for the record filter,
the trim indices and the trimmed-mean walk), restated as runs of constant depth so that contigs of 2^31 - 1 bases cost only
their events.

  * a contig's events are +1 at every aligned block's start and -1 at its end unless the block reaches the contig end;
    between two consecutive event positions the depth is constant, from 0 before the first to the last one's depth at L;
  * window reductions over [E, L - E) (only when 2E < L) are those runs clipped to the window; the histogram holds each
    run's clipped length at its depth, and depth 0 gets the window length minus the covered bases (closed form);
  * trimmed_total walks that histogram densely by depth (depths are bounded by the contig's read count), the variance sums
    are taken modulo 2^64, and the histogram fields and pairs exist for contigs with at least one counted record.
"""
import math

import numpy as np

import device_reference as ref


def depth_runs(L, s, e):
    """(starts, ends, depths) of the runs of constant depth that cover [0, L), from block starts `s` and ends `e`."""
    s = np.asarray(s, dtype=np.int64)
    e = np.asarray(e, dtype=np.int64)
    inside = e < L
    pos = np.concatenate([s, e[inside]])
    delta = np.concatenate([np.ones(len(s), dtype=np.int64), -np.ones(int(inside.sum()), dtype=np.int64)])
    order = np.argsort(pos, kind="stable")
    pos, delta = pos[order], delta[order]
    cuts, first = np.unique(pos, return_index=True)
    step = np.add.reduceat(delta, first) if len(pos) else np.zeros(0, dtype=np.int64)
    starts = np.concatenate([[0], cuts])
    ends = np.concatenate([cuts, [L]])
    depths = np.concatenate([[0], np.cumsum(step)])
    keep = ends > starts
    return starts[keep], ends[keep], depths[keep]


def window_stats(L, s, e, E, p, hist):
    """The window / histogram fields of one contig (device_reference.window_stats, from runs)."""
    starts, ends, depths = depth_runs(L, s, e)
    cov = depths > 0
    out = dict(covered_full=int((ends - starts)[cov].sum()))
    if not 2 * E < L:
        return out, None
    lo, hi = E, L - E
    n = np.maximum(0, np.minimum(ends, hi) - np.maximum(starts, lo))
    wcov = cov & (n > 0)
    out["covered_window"] = int(n[wcov].sum())
    out["sum_depth_window"] = int((n[wcov] * depths[wcov]).sum())
    if not hist:
        return out, None
    T = L - 2 * E
    counts = np.zeros(int(depths[wcov].max()) + 1 if wcov.any() else 1, dtype=np.int64)
    np.add.at(counts, depths[wcov], n[wcov])
    counts[0] = T - out["covered_window"]
    present = np.flatnonzero(counts)
    k = int(present[0])
    tmin, tmax = ref.trim_indices(p["trim_min"], p["trim_max"], T)
    ex = ex2 = 0
    for x in present:
        c = int(counts[x])
        ex += (int(x) - k) * c
        ex2 += (int(x) - k) ** 2 * c
    out.update(trimmed_total=ref.trimmed_total(counts, tmin, tmax), trim_min_index=tmin, trim_max_index=tmax, var_k=k,
               var_ex=ex & ref.MASK64, var_ex2=ex2 & ref.MASK64, hist_count=len(present))
    return out, (present.astype(np.uint32), counts[present].astype(np.uint32))


def expected(lens, p, cols, shard=None):
    """Contig mode of device_reference.expected: rows, pairs and error of the records `cols` on contigs `lens` (shard
    [tid_begin, tid_end)).  Load counts are not predicted."""
    lens = [int(x) for x in lens]
    n_ref = len(lens)
    tid = np.asarray(cols["tid"], dtype=np.int64)
    keep, nm_err = ref._record_filter(cols, p)
    valid_tid = (tid >= 0) & (tid < n_ref)
    E = int(p["contig_end_exclusion"])
    hist = bool(p["want"] & (ref.WANT_HIST | ref.WANT_HIST_CSR))
    flag = np.asarray(cols["flag"], dtype=np.int64)
    primary = (flag & 0x900) == 0
    nonsupp = (flag & 0x800) == 0
    nm = np.asarray(cols["nm"], dtype=np.int64)
    aligned = np.asarray(cols["aligned"], dtype=np.int64)
    indel = np.asarray(cols["ins"], dtype=np.int64) + np.asarray(cols["del_"], dtype=np.int64)
    with np.errstate(all="ignore"):
        identity = np.where(aligned > 0, (aligned.astype(np.float64) - nm) / aligned, 0.0)

    kt = tid[keep & valid_tid]
    bounds = bool((keep & ~valid_tid).any())
    own, s, e = ref._intervals(cols, keep & valid_tid)
    L_of = np.asarray(lens, dtype=np.int64)[tid[own]] if len(own) else np.zeros(0, dtype=np.int64)
    bad = (s < 0) | (s >= L_of)
    tb, te = shard if shard is not None else (0, n_ref)
    mine = keep & valid_tid & (tid >= tb) & (tid < te)
    bounds |= bool((bad & mine[own]).any())
    out = ref.Expected(n_ref)
    for t in np.unique(tid[mine]):
        r = mine & (tid == t)
        out.rows[t].update(n_records=int(r.sum()), n_primary=int((r & primary).sum()), n_nonsupp=int((r & nonsupp).sum()),
                           sum_edit=int(nm[r].sum()), sum_indel=int(indel[r].sum()),
                           sum_identity_primary=math.fsum(identity[r & primary & (aligned > 0)]),
                           sum_identity_nonsupp=math.fsum(identity[r & nonsupp & (aligned > 0)]))
    ok = mine[own] & ~bad
    ev_seg, ev_s, ev_e = tid[own[ok]], s[ok], e[ok]
    order = np.argsort(ev_seg, kind="stable")
    ev_seg, ev_s, ev_e = ev_seg[order], ev_s[order], ev_e[order]
    bounds_of = np.searchsorted(ev_seg, np.arange(n_ref + 1))
    for t in range(tb, te):
        a, b = bounds_of[t], bounds_of[t + 1]
        fields, pairs = window_stats(lens[t], ev_s[a:b], ev_e[a:b], E, p, hist and out.rows[t]["n_records"] > 0)
        out.rows[t].update(fields)
        out.pairs[t] = pairs

    if (np.diff(kt) < 0).any():
        out.error = ref.CMB_E_UNSORTED
    elif nm_err.any():
        out.error = ref.CMB_E_NM
    elif bounds:
        out.error = ref.CMB_E_BOUNDS
    return out
