"""Exact expected results of one sample on the device ABI (include/coverm_b200.h), in plain numpy and Python integers.

Restated from what the header promises and the reference rules it cites -- never from the kernels:
  * flag filter (lib.rs:59-79) and the single-read thresholds of ReferenceSortedBamFilter (filter.rs:243-279) in float32;
  * per-contig delta events (contig.rs:166-211): +1 at an aligned block's start, -1 at its end unless the block reaches the
    contig end, then a cumulative sum -- one dense int64 array per contig;
  * window reductions (EST:366-502) over [E, L - E), which exists only when 2E < L;
  * trimmed-mean walk (EST:591-642) with float32 trim indices, walked literally over the dense depth histogram;
  * variance sums (EST:790-805) modulo 2^64 like the reference's usize;
  * gene mode as the cmb_set_genes comment states it: a gene's depth is its contig's depth cut to [start, end), and records
    count for the genes that contain their leftmost position.
It also predicts what K2 fetches (the `#k2_load` line CMB_PIPELINE_STATS=1 prints): a segment (contig of the shard, or gene)
occupies max(1, ceil(L / 32)) 32-element spans of the arena, 256 spans make a chunk, and a span is occupied when an event of a
kept, in-shard record falls in it -- a +1 and a -1 that cancel still occupy it.  A chunk with at least D occupied spans is
loaded whole (256 spans), any other one span by span.

Pair filtering is not modelled here (tests/pair_reference.py models it): `filtering` must select the single-read filter.
"""
import math

import numpy as np

WANT_HIST, WANT_HIST_CSR = 1, 2
IV_PAD = -(1 << 31)
CMB_E_UNSORTED, CMB_E_NM, CMB_E_BOUNDS = -4, -5, -6
SPAN = 32            # arena elements per span (one bitmap bit)
CHUNK_SPANS = 256    # spans per chunk
MASK64 = (1 << 64) - 1

INT_FIELDS = ["n_records", "n_primary", "n_nonsupp", "sum_edit", "sum_indel", "sum_depth_window", "covered_window",
              "covered_full", "trimmed_total", "trim_min_index", "trim_max_index", "var_k", "var_ex", "var_ex2", "hist_count"]
FLOAT_FIELDS = ["sum_identity_primary", "sum_identity_nonsupp"]


def default_params(**kw):
    """cmb_params as a dict: no filtering, every flag included except secondary / supplementary, E = 0, trim 5-95 %."""
    p = dict(include_improper_pairs=1, include_supplementary=0, include_secondary=0, filtering=0, min_mapq=255,
             min_aligned_length_single=0, min_percent_identity_single=0.0, min_aligned_percent_single=0.0,
             min_aligned_length_pair=0, min_percent_identity_pair=0.0, min_aligned_percent_pair=0.0,
             contig_end_exclusion=0, trim_min=0.05, trim_max=0.95, want=0)
    unknown = set(kw) - set(p)
    assert not unknown, unknown
    p.update(kw)
    return p


def filter_mode(p):
    """(filter_single_reads, filter_pairs) as filter.rs:48-61 derives them."""
    f32 = np.float32
    single = p["min_aligned_length_single"] > 0 or f32(p["min_percent_identity_single"]) > 0 or f32(p["min_aligned_percent_single"]) > 0
    pair = p["min_aligned_length_pair"] > 0 or f32(p["min_percent_identity_pair"]) > 0 or f32(p["min_aligned_percent_pair"]) > 0
    fs = single or (not pair and p["min_mapq"] != 255)
    fp = pair or ((not fs or not p["include_improper_pairs"]) and p["min_mapq"] != 255)
    return (fs, fp) if p["filtering"] else (False, False)


def trim_indices(trim_min, trim_max, T):
    """EST:591-592: `(min * total_bases as f32).floor() as usize`, the product in float32."""
    Tf = np.float32(T)
    lo = np.float32(trim_min) * Tf
    hi = np.float32(trim_max) * Tf
    assert isinstance(lo, np.float32) and isinstance(hi, np.float32)
    return max(0, math.floor(lo)), max(0, math.ceil(hi))


def trimmed_total(counts, min_index, max_index):
    """The ascending walk of EST:598-642 over the dense histogram `counts` (counts[i] = bases at depth i): its `total`."""
    acc = total = 0
    started = False
    for i, n in enumerate(counts):
        n = int(n)
        acc += n
        if acc < min_index:
            continue
        if started:
            if acc > max_index:
                excess = acc - n
                total += (max_index - excess + 1 if max_index >= excess else 0) * i
                break
            total += n * i
        elif acc > max_index:
            total = (max_index - min_index + 1) * i
            started = True
        else:
            total = (acc - min_index + 1) * i
            started = True
    return total & MASK64


def window_stats(depth, E, p, hist):
    """Window / histogram fields of one segment from its depth array; `hist`: fill the histogram-derived ones."""
    L = len(depth)
    out = dict(covered_full=int(np.count_nonzero(depth)))
    if not 2 * E < L:
        return out, None
    w = depth[E:L - E]
    out["covered_window"] = int(np.count_nonzero(w))
    out["sum_depth_window"] = int(w.sum(dtype=np.int64))
    if not hist:
        return out, None
    counts = np.bincount(w)
    depths = np.flatnonzero(counts)
    k = int(depths[0])
    lo, hi = trim_indices(p["trim_min"], p["trim_max"], L - 2 * E)
    ex = ex2 = 0
    for x in depths:
        n = int(counts[x])
        ex += (int(x) - k) * n
        ex2 += (int(x) - k) ** 2 * n
    out.update(trimmed_total=trimmed_total(counts, lo, hi), trim_min_index=lo, trim_max_index=hi, var_k=k,
               var_ex=ex & MASK64, var_ex2=ex2 & MASK64, hist_count=len(depths))
    return out, (depths.astype(np.uint32), counts[depths].astype(np.uint32))


class Expected:
    """rows: one dict per result row (every field of INT_FIELDS and FLOAT_FIELDS); pairs: per row, (depths, counts) of its
    histogram when the row's histogram fields are filled, else None; error: 0 or the CMB_E_* code cmb_end_sample returns;
    contig_seen / kept_primary: gene mode's cmb_fetch_gene_extras."""

    def __init__(self, n_rows):
        self.rows = [dict.fromkeys(INT_FIELDS, 0) | dict.fromkeys(FLOAT_FIELDS, 0.0) for _ in range(n_rows)]
        self.pairs = [None] * n_rows
        self.error = 0
        self.contig_seen = None
        self.kept_primary = None
        self.seg_spans = None      # spans of each arena segment
        self.occupied = None       # sorted global ids of the occupied spans

    @property
    def n_chunks(self):
        return max(1, -(-int(self.seg_spans.sum()) // CHUNK_SPANS))

    def chunk_pop(self):
        """Occupied spans per chunk."""
        return np.bincount(self.occupied // CHUNK_SPANS, minlength=self.n_chunks)

    def load_counts(self, dense_spans):
        """(spans loaded, chunks loaded whole) for the dense threshold `dense_spans`."""
        pop = self.chunk_pop()
        dense = pop >= dense_spans
        return int(np.where(dense, CHUNK_SPANS, pop).sum()), int(dense.sum())


def _record_filter(cols, p):
    """(kept mask, NM error mask) of every record."""
    flag = np.asarray(cols["flag"], dtype=np.int64)
    unmapped, sec, sup, proper = (flag & 0x4) != 0, (flag & 0x100) != 0, (flag & 0x800) != 0, (flag & 0x2) != 0
    flag_pass = ~(sec & (not p["include_secondary"])) & ~(sup & (not p["include_supplementary"])) & \
        ~(~proper & (not p["include_improper_pairs"]))
    keep = flag_pass & ~unmapped
    nm_ok = np.asarray(cols["nm_state"]) == 1
    nm_err = np.zeros_like(keep)
    if p["filtering"]:
        fs, fp = filter_mode(p)
        if fp or not fs:
            raise NotImplementedError("only the single-read filter is modelled")
        mapq = np.asarray(cols["mapq"], dtype=np.int64)
        mq_fail = (mapq < p["min_mapq"]) | (mapq == 255) if p["min_mapq"] != 255 else np.zeros_like(keep)
        f32 = np.float32
        al = np.asarray(cols["aligned"]).astype(f32)
        with np.errstate(all="ignore"):
            thresholds = (np.asarray(cols["aligned"]) >= p["min_aligned_length_single"]) & \
                (al / np.asarray(cols["l_seq"]).astype(f32) >= f32(p["min_aligned_percent_single"])) & \
                (f32(1) - np.asarray(cols["nm"]).astype(f32) / al >= f32(p["min_percent_identity_single"]))
        nm_err |= ~mq_fail & ~nm_ok  # nm() is reached once the MAPQ test passed
        keep &= (bool(p["include_supplementary"]) | ~sup) & (bool(p["include_secondary"]) | ~sec) & ~mq_fail & thresholds
    nm_err |= keep & ~nm_ok
    return keep, nm_err


def _intervals(cols, recs):
    """(record, start, end) of every non-pad aligned block of the records `recs` (a boolean mask)."""
    ivb = np.asarray(cols["iv_begin"], dtype=np.int64)
    owner = np.repeat(np.arange(len(ivb) - 1), np.diff(ivb))
    s = np.asarray(cols["iv_start"], dtype=np.int64)[:ivb[-1]]
    e = s + np.asarray(cols["iv_len"], dtype=np.int64)[:ivb[-1]]
    sel = recs[owner] & (s != IV_PAD)
    return owner[sel], s[sel], e[sel]


def _depth(L, s, e):
    delta = np.zeros(L + 1, dtype=np.int64)
    np.add.at(delta, s, 1)
    inside = e < L
    np.add.at(delta, e[inside], -1)
    return np.cumsum(delta[:L])


def expected(lens, p, cols, shard=None, genes=None):
    """Expected cmb_end_sample result of the records `cols` (cmb_read_batch columns by name, `iv_begin` with n + 1 entries)
    on a reference of contig lengths `lens` with parameters `p` (default_params), on the shard [tid_begin, tid_end) or, with
    `genes` ((tid, start, end) sorted by (tid, start)), per gene."""
    lens = [int(x) for x in lens]
    n_ref = len(lens)
    tid = np.asarray(cols["tid"], dtype=np.int64)
    n = len(tid)
    keep, nm_err = _record_filter(cols, p)
    valid_tid = (tid >= 0) & (tid < n_ref)
    E = int(p["contig_end_exclusion"])
    hist = bool(p["want"] & (WANT_HIST | WANT_HIST_CSR))
    flag = np.asarray(cols["flag"], dtype=np.int64)
    primary = (flag & 0x900) == 0
    nonsupp = (flag & 0x800) == 0
    nm = np.asarray(cols["nm"], dtype=np.int64)
    aligned = np.asarray(cols["aligned"], dtype=np.int64)
    indel = np.asarray(cols["ins"], dtype=np.int64) + np.asarray(cols["del_"], dtype=np.int64)
    pos = np.asarray(cols["pos"], dtype=np.int64)
    with np.errstate(all="ignore"):
        identity = np.where(aligned > 0, (aligned.astype(np.float64) - nm) / aligned, 0.0)

    # errors, in the order cmb_end_sample reports them
    kt = tid[keep & valid_tid]
    bounds = bool((keep & ~valid_tid).any())
    own, s, e = _intervals(cols, keep & valid_tid)
    L_of = np.asarray(lens, dtype=np.int64)[tid[own]] if len(own) else np.zeros(0, dtype=np.int64)
    bad = (s < 0) | (s >= L_of)
    bad_rec = np.zeros(n, dtype=bool)
    bad_rec[own[bad]] = True

    if genes is None:
        tb, te = shard if shard is not None else (0, n_ref)
        mine = keep & valid_tid & (tid >= tb) & (tid < te)
        bounds |= bool((bad & mine[own]).any())
        out = Expected(n_ref)
        seg_lens = lens[tb:te]
        for t in np.unique(tid[mine]):
            r = mine & (tid == t)
            row = out.rows[t]
            row.update(n_records=int(r.sum()), n_primary=int((r & primary).sum()), n_nonsupp=int((r & nonsupp).sum()),
                       sum_edit=int(nm[r].sum()), sum_indel=int(indel[r].sum()),
                       sum_identity_primary=math.fsum(identity[r & primary & (aligned > 0)]),
                       sum_identity_nonsupp=math.fsum(identity[r & nonsupp & (aligned > 0)]))
        ok = mine[own] & ~bad
        ev_seg, ev_s, ev_e = tid[own[ok]], s[ok], e[ok]
        for t in range(tb, te):
            sel = ev_seg == t
            depth = _depth(lens[t], ev_s[sel], ev_e[sel])
            fields, pairs = window_stats(depth, E, p, hist and out.rows[t]["n_records"] > 0)
            out.rows[t].update(fields)
            out.pairs[t] = pairs
        # events in arena coordinates: (segment, offset in it)
        ev = [(ev_seg - tb, ev_s), (ev_seg - tb, ev_e)]
        ev_inside = [np.ones(len(ev_s), dtype=bool), ev_e < L_of[ok]]
    else:
        bounds |= bool(bad.any())
        out = Expected(max(1, len(genes)))
        seg_lens = [g[2] - g[1] for g in genes] or [1]
        gk = keep & valid_tid & ~bad_rec
        out.contig_seen = np.zeros(n_ref, dtype=np.uint8)
        out.contig_seen[np.unique(kt)] = 1
        out.kept_primary = int((keep & valid_tid & primary).sum())
        ok = gk[own]
        depth_of = {t: _depth(lens[t], s[ok & (tid[own] == t)], e[ok & (tid[own] == t)]) for t in np.unique(tid[gk])}
        ev_seg, ev_s, ev_e, ev_in = [], [], [], []
        for g, (t, gs, ge) in enumerate(genes):
            row = out.rows[g]
            r = gk & (tid == t) & (pos >= gs) & (pos < ge)
            row.update(n_records=int(r.sum()), n_primary=int((r & primary).sum()),
                       sum_edit=int(np.maximum(nm[r] - indel[r], 0).sum()),
                       sum_identity_primary=math.fsum(identity[r & primary & (aligned > 0)]))
            if not out.contig_seen[t]:
                continue
            depth = depth_of[t][gs:ge] if t in depth_of else np.zeros(ge - gs, dtype=np.int64)
            fields, pairs = window_stats(depth, E, p, hist)
            row.update(fields)
            out.pairs[g] = pairs
            # the block clipped to the gene: +1 at its first base inside, -1 where it ends if that is inside
            sel = ok & (tid[own] == t) & (e > gs) & (s < ge)
            ev_seg.append(np.full(int(sel.sum()), g))
            ev_s.append(np.maximum(s[sel], gs) - gs)
            ev_e.append(e[sel] - gs)
            ev_in.append(e[sel] - gs < ge - gs)
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, dtype=np.int64)  # noqa: E731
        ev_seg, ev_s, ev_e, ev_in = cat(ev_seg), cat(ev_s), cat(ev_e), cat(ev_in).astype(bool)
        ev = [(ev_seg, ev_s), (ev_seg, ev_e)]
        ev_inside = [np.ones(len(ev_s), dtype=bool), ev_in]

    seg_spans = np.array([max(1, -(-L // SPAN)) for L in seg_lens], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(seg_spans)])
    out.seg_spans = seg_spans
    out.occupied = np.unique(np.concatenate(
        [off[sg[m].astype(np.int64)] + x[m] // SPAN for (sg, x), m in zip(ev, ev_inside)]).astype(np.int64))

    if (np.diff(kt) < 0).any():
        out.error = CMB_E_UNSORTED
    elif nm_err.any():
        out.error = CMB_E_NM
    elif bounds:
        out.error = CMB_E_BOUNDS
    return out
