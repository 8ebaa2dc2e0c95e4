"""Named, deterministic inputs for the kernel-level tests, and the harness that runs one on a cmb_* library and checks every
result against tests/device_reference.py.

Each scenario is a reference (contig lengths, optionally a shard or a gene list) and one or more samples run one after the
other on the same context.  tests/test_device_reference.py runs them on the CPU emulator of the ABI, which checks the
reference and this harness without a GPU; tests/test_device_kernels.py runs them on the CUDA library, where the integer fields
must match exactly, the identity sums to 1e-12, the histogram pairs exactly, and K2's load counts exactly.
"""
import random
from dataclasses import dataclass, field

import numpy as np

import coverm_b200
import device_reference as ref

CHUNK = ref.SPAN * ref.CHUNK_SPANS      # 8192 arena elements
K1B_BLOCK_ELEMS = 1024 * CHUNK          # chunks per K1b block x chunk
WANTS = {"nohist": 0, "hist": ref.WANT_HIST, "hist_csr": ref.WANT_HIST | ref.WANT_HIST_CSR}
EDGE_LENS = [1, 31, 32, 33, 1023, 1024, 1025, 8191, 8192, 8193, 3 * 8192 + 5]


class Records:
    """Builds cmb_read_batch columns.  A record is its aligned (M/=/X) blocks as absolute (start, length) pairs, the first
    one at `pos` like a real CIGAR's; `ins` / `dels` are its I / D lengths, `pads` CMB_IV_PAD slots put among its blocks."""

    def __init__(self):
        self.recs = []

    def add(self, tid, pos, length=None, blocks=None, flag=0, mapq=60, nm=0, ins=0, dels=0, clip=0, pads=0):
        blocks = list(blocks) if blocks is not None else [(pos, length)]
        assert blocks[0][0] == pos and all(n >= 0 for _, n in blocks)
        ivs = [(s, n) for s, n in blocks]
        for k in range(pads):
            ivs.insert((k * 7) % (len(ivs) + 1), (ref.IV_PAD, 0))
        m = sum(n for _, n in blocks)
        self.recs.append(dict(tid=tid, pos=pos, flag=flag, mapq=mapq, nm_state=1, nm=nm, l_seq=m + ins + clip,
                              aligned=m + ins + dels, del_=dels, ins=ins, ivs=ivs))
        return self

    def columns(self):
        recs = sorted(self.recs, key=lambda r: (r["tid"], r["pos"]))
        cols = {k: np.array([r[k] for r in recs], dtype=dt) for k, dt in
                [("tid", np.int32), ("pos", np.int32), ("flag", np.uint16), ("mapq", np.uint8), ("nm_state", np.uint8),
                 ("nm", np.uint32), ("l_seq", np.uint32), ("aligned", np.uint32), ("del_", np.uint32), ("ins", np.uint32)]}
        cols["iv_begin"] = np.concatenate([[0], np.cumsum([len(r["ivs"]) for r in recs])]).astype(np.uint32)
        ivs = [iv for r in recs for iv in r["ivs"]]
        cols["iv_start"] = np.array([s for s, _ in ivs], dtype=np.int32)
        cols["iv_len"] = np.array([n for _, n in ivs], dtype=np.int32)
        return cols


@dataclass
class Sample:
    records: dict
    params: dict
    fixed_want: bool = False  # the sample's own `want` is kept (the seeded sweep draws it)


@dataclass
class Scenario:
    name: str
    lens: list
    samples: list
    shard: tuple = None
    genes: list = None
    batch_records: int = 1 << 16
    env: dict = field(default_factory=dict)  # set before the context is created


def _reads(rng, recs, tid, L, n, max_len=300, max_blocks=3, pads=False):
    """`n` random records on contig `tid` of length L: up to `max_blocks` blocks separated by N or D gaps, every block
    starting inside the contig (it may run past its end)."""
    for _ in range(n):
        pos = rng.randrange(L)
        blocks, cur, dels = [], pos, 0
        for _ in range(rng.randint(1, max_blocks)):
            if cur >= L:
                break
            ln = rng.randint(1, max_len)
            blocks.append((cur, ln))
            gap = rng.randint(1, 60)
            if rng.random() < 0.5:
                dels += gap
            cur += ln + gap
        m = sum(n for _, n in blocks)
        recs.add(tid, pos, blocks=blocks, nm=rng.randint(0, max(0, m // 10)), ins=rng.randint(0, 3), dels=dels,
                 clip=rng.randint(0, 5), flag=rng.choice([0, 16, 0x2 | 0x40, 0x100, 0x800, 0x4, 16 | 0x800]),
                 mapq=rng.choice([0, 5, 30, 60, 255]), pads=rng.randint(0, 2) if pads else 0)


# --------------------------------------------------------------------------------------------------------- a. layout edges
def layout_edges():
    """Contig lengths around span (32), bitmap word (1024) and chunk (8192) sizes, so that contig starts land mid-word, on a
    word, on a chunk start and after padding; blocks at both contig ends, one base long, across those boundaries, records
    with several blocks and with pad slots."""
    rng = random.Random(11)
    lens = list(EDGE_LENS)
    recs = Records()
    for t, L in enumerate(lens):
        recs.add(t, 0, 1)                      # one base at 0
        recs.add(t, L - 1, 1)                  # one base at L-1, ends at L: no -1
        recs.add(t, 0, L)                      # the whole contig
        recs.add(t, L - 1, 5)                  # runs past the end
        if L > 2:
            recs.add(t, 1, L - 2)              # ends at L-1
        for b in (32, 1024, 8192):
            if b + 1 < L:
                recs.add(t, b - 1, 2)          # across the boundary
                recs.add(t, b, 1)
                recs.add(t, max(0, b - 40), min(80, L - max(0, b - 40)))
        if L > 100:                            # several blocks with N skips, and pad slots
            recs.add(t, 3, blocks=[(3, 10), (20, 5), (L - 30, 30)], pads=1)
            recs.add(t, 5, blocks=[(5, 1), (6, 1), (40, 33)], dels=1, pads=2)
        _reads(rng, recs, t, L, 5 + L // 400, pads=True)
    cols = recs.columns()
    return Scenario("a_layout_edges", lens, [Sample(cols, ref.default_params()),
                                            Sample(cols, ref.default_params(contig_end_exclusion=7, trim_min=0.1, trim_max=0.9))])


# ------------------------------------------------------------------------------------------------ b. load-path threshold
LOAD_POPS = [0, 1, 31, 32, 33, 159, 160, 161, 255, 256]
WARP_PATTERNS = [[0], [31], [7, 8, 9], [0, 1, 2, 3], [0, 1, 2, 3, 4], list(range(96, 128)), [w * 32 + 5 for w in range(8)]]


def load_path_span_sets():
    """Spans (0..255) holding events in each chunk of the load-path scenario's first contig."""
    rng = random.Random(5)
    sets = [sorted(rng.sample(range(ref.CHUNK_SPANS), p)) for p in LOAD_POPS]
    return sets + [sorted(s) for s in WARP_PATTERNS]


def load_path():
    """A contig whose successive chunks hold events in exactly LOAD_POPS spans, then chunks with rows {0}, {31}, {7..9},
    {0..3}, {0..4}, all 32 rows of one warp and one row in every warp (the row copies hand out four rows per instruction
    round); reads between them carry depth across the chunks in between.
    A short contig starting on the next chunk boundary follows."""
    sets = load_path_span_sets()
    L = len(sets) * CHUNK
    recs = Records()
    occupied = []
    for k, spans in enumerate(sets):
        for s in spans:
            recs.add(0, k * CHUNK + s * ref.SPAN + 3, 20)  # +1 and -1 in span s
            occupied.append(k * CHUNK + s * ref.SPAN)
    for a, b in zip(occupied, occupied[1:]):  # carries: blocks from one occupied span into the next
        if b // CHUNK != a // CHUNK:
            recs.add(0, a + 7, b + 9 - (a + 7))
    recs.add(1, 10, 50)
    cols = recs.columns()
    return Scenario("b_load_path", [L, 100], [Sample(cols, ref.default_params(contig_end_exclusion=100))])


# ------------------------------------------------------------------------------------------------------------ c. carries
BIG = 20_000_001  # odd, so that T = L - 2E is odd and float32(T) rounds


def carries():
    """Aligned blocks of 20 000 and 100 000 bases that cover whole chunks without an event in them (depth from the chunk carry
    alone), and a 20 Mbp contig spanning more than two K1b blocks, with reads across every chunk boundary of it and one block
    that covers a whole K1b block."""
    rng = random.Random(7)
    lens = [5000, 300_000, BIG, 777]
    recs = Records()
    _reads(rng, recs, 0, 5000, 40)
    for p0 in (1000, 50_000, 150_000):
        recs.add(1, p0, 20_000)
        recs.add(1, p0 + 5, 100_000)
    recs.add(1, 299_000, 5000)
    for b in range(CHUNK, BIG, CHUNK):  # the arena offset of this contig is not chunk aligned: also cross its own multiples
        recs.add(2, b - rng.randint(1, 400), rng.randint(401, 900))
    recs.add(2, 8_000_000, 8_600_000)   # holds global arena elements [8 388 608, 16 777 216): K1b block 1 whole
    recs.add(2, 1_000_000, 18_999_000)
    recs.add(2, BIG - 10, 10)
    _reads(rng, recs, 2, BIG, 300, max_len=5000)
    _reads(rng, recs, 3, 777, 10)
    cols = recs.columns()
    return Scenario("c_carries", lens, [Sample(cols, ref.default_params()),
                                        Sample(cols, ref.default_params(contig_end_exclusion=1000, trim_min=0.1, trim_max=0.9))])


# ---------------------------------------------------------------------------------------------------------- d. histogram
def hist_slots():
    """12 covered 500-base contigs in one chunk: more contigs than K2 has shared-memory histogram slots."""
    rng = random.Random(3)
    lens = [500] * 12 + [3000]
    recs = Records()
    for t in range(12):
        recs.add(t, 100 + 10 * t, 50)
        _reads(rng, recs, t, 500, 3 + 4 * t, max_len=200, max_blocks=1)
    _reads(rng, recs, 12, 3000, 30)
    return Scenario("d_hist_slots", lens, [Sample(recs.columns(), ref.default_params(contig_end_exclusion=10))])


def overflow_bins():
    """Depth stepping from 0 to 300 inside one chunk: depths 128 apart share a direct-mapped bin (the overflow list)."""
    recs = Records()
    for i in range(300):
        recs.add(0, 10 + 20 * i, 7000 - 20 * i)
    recs.add(0, 9000, 100)
    return Scenario("d_overflow_bins", [2 * CHUNK], [Sample(recs.columns(), ref.default_params())])


def k3_windows():
    """Depths from 0 to 1100 in one contig: K3 merges its histogram in several 512-depth windows."""
    recs = Records()
    for i in range(1100):
        recs.add(0, 7 + 10 * i, 15_000 - 10 * i)
    recs.add(1, 0, 40)
    return Scenario("d_k3_windows", [20_000, 64], [Sample(recs.columns(), ref.default_params(contig_end_exclusion=3))])


def end_exclusion():
    """E in {0, 1, 49, 50, 51} on contigs of 100 and 101 bases: windows of 2E = L-2, L-1 and L, and none."""
    rng = random.Random(13)
    lens = [100, 101, 102, 99, 1000]
    recs = Records()
    for t, L in enumerate(lens):
        _reads(rng, recs, t, L, 12, max_len=60)
    cols = recs.columns()
    return Scenario("d_end_exclusion", lens, [Sample(cols, ref.default_params(contig_end_exclusion=E)) for E in (0, 1, 49, 50, 51)])


TRIMS = [(0.0, 1.0), (0.05, 0.95), (0.1, 0.9), (0.7, 0.9), (0.1, 0.3)]  # the last two round differently in f32 and f64 at T=10


def trims():
    """Trim pairs (0, 1), (0.05, 0.95), (0.1, 0.9), and two whose indices at T = 10 differ between float32 and float64."""
    rng = random.Random(17)
    lens = [10, 1000, 4321]
    recs = Records()
    recs.add(0, 0, 3).add(0, 1, 9).add(0, 2, 2).add(0, 6, 1)
    for t in (1, 2):
        _reads(rng, recs, t, lens[t], 40)
    cols = recs.columns()
    return Scenario("d_trims", lens, [Sample(cols, ref.default_params(trim_min=a, trim_max=b)) for a, b in TRIMS])


# ------------------------------------------------------------------------------------------- e. batches, shards and genes
def _mixed(seed, lens, n):
    rng = random.Random(seed)
    recs = Records()
    for _ in range(n):
        t = rng.randrange(len(lens))
        _reads(rng, recs, t, lens[t], 1, pads=True)
    return recs.columns()


def batches():
    """5000 records through staging batches of 1000 records."""
    lens = [30_000, 1, 8192, 50_000, 777]
    return Scenario("e_batches", lens, [Sample(_mixed(19, lens, 5000), ref.default_params(contig_end_exclusion=20))],
                    batch_records=1000)


def shard():
    """The shard [2, 6) of 8 contigs: rows outside it stay zero, its loads come from its own records only."""
    lens = [9000, 300, 17_000, 1025, 8193, 40, 12_000, 500]
    return Scenario("e_shard", lens, [Sample(_mixed(23, lens, 3000), ref.default_params(contig_end_exclusion=5))],
                    shard=(2, 6))


def genes():
    """Overlapping genes, genes at contig ends and across chunk boundaries, and reads that start before a gene."""
    lens = [5000, 3000, 20_000]
    gl = [(0, 0, 10), (0, 100, 900), (0, 500, 1500), (0, 1400, 1450), (0, 1400, 4000), (0, 4990, 5000),
          (1, 0, 3000), (1, 2999, 3000), (2, 0, 9000), (2, 8191, 8300), (2, 8192, 16_385), (2, 11_000, 20_000)]
    rng = random.Random(29)
    recs = Records()
    for t, L in enumerate(lens):
        _reads(rng, recs, t, L, 150)
    recs.add(0, 80, 100).add(0, 450, blocks=[(450, 20), (480, 600)]).add(2, 8000, 500)
    cols = recs.columns()
    return Scenario("e_genes", lens, [Sample(cols, ref.default_params()),
                                      Sample(cols, ref.default_params(contig_end_exclusion=4, trim_min=0.0, trim_max=1.0))],
                    genes=gl)


# ------------------------------------------------------------------------------------------------------------- f. reuse
def _reuse_samples():
    lens = [4 * CHUNK, 2 * CHUNK + 100, 3000]
    a = Records()  # every span of the first four chunks
    for p0 in range(0, 4 * CHUNK, 16):
        a.add(0, p0, 40)
    b = Records()  # a few spans, most of them where A had none
    rng = random.Random(31)
    for _ in range(40):
        t = rng.choice([0, 1, 1, 2])
        b.add(t, rng.randrange(lens[t]), rng.randint(1, 50))
    bad = Records().add(1, 10, 30).add(2, 3000, 1)  # a block starting at the contig end
    pa, pb = ref.default_params(contig_end_exclusion=2), ref.default_params()
    A, B = Sample(a.columns(), pa), Sample(b.columns(), pb)
    return lens, [A, B, A, Sample(bad.columns(), pb), B]


def reuse():
    """On one context: A (dense everywhere), B (sparse, mostly in other spans), A again, a sample rejected with CMB_E_BOUNDS,
    then B.  Stale span bits or arena values left by an earlier sample would show up in B's loads or numbers."""
    lens, samples = _reuse_samples()
    return Scenario("f_reuse", lens, samples)


def reuse_no_clean():
    """The same with CMB_CLEAN_AS_YOU_GO=0: the arena and bitmap are zeroed at the start of every sample instead."""
    lens, samples = _reuse_samples()
    return Scenario("f_reuse_no_clean", lens, samples, env={"CMB_CLEAN_AS_YOU_GO": "0"})


# ---------------------------------------------------------------------------------------------------------- g. sweep
def sweep(seed):
    """Lengths from the edge set and random ones, random records sorted by (tid, pos), random E / trim / want / flags /
    single-read filter, every fourth seed on a random shard."""
    rng = random.Random(1000 + seed)
    lens = [rng.choice(EDGE_LENS) if rng.random() < 0.5 else rng.randint(1, 60_000) for _ in range(rng.randint(1, 14))]
    recs = Records()
    for _ in range(rng.randint(0, 2500)):
        t = rng.randrange(len(lens))
        _reads(rng, recs, t, lens[t], 1, max_len=rng.choice([5, 100, 2000]), pads=True)
    tmin = rng.choice([0.0, 0.05, 0.1, 0.25, rng.random() * 0.5])
    p = ref.default_params(contig_end_exclusion=rng.choice([0, 1, 5, 50, 500, rng.randint(0, 30_000)]),
                           trim_min=tmin, trim_max=rng.choice([1.0, 0.95, 0.9, tmin + (1 - tmin) * rng.random()]),
                           want=rng.choice(list(WANTS.values())), include_secondary=rng.randint(0, 1),
                           include_supplementary=rng.randint(0, 1), include_improper_pairs=rng.randint(0, 1))
    if seed % 3 == 1:  # the single-read filter (filter.rs:243-279); improper pairs included keeps the pair filter off
        p.update(filtering=1, include_improper_pairs=1, min_mapq=rng.choice([0, 10, 40]),
                 min_aligned_length_single=rng.choice([0, 20, 100]), min_percent_identity_single=rng.choice([0.0, 0.9, 0.95]),
                 min_aligned_percent_single=rng.choice([0.0, 0.5, 0.97]))
    tb = rng.randrange(len(lens))
    sh = (tb, rng.randint(tb + 1, len(lens))) if seed % 4 == 3 else None
    return Scenario(f"g_sweep_{seed}", lens, [Sample(recs.columns(), p, fixed_want=True)], shard=sh)


BUILDERS = {"a_layout_edges": layout_edges, "b_load_path": load_path, "c_carries": carries, "d_hist_slots": hist_slots,
            "d_overflow_bins": overflow_bins, "d_k3_windows": k3_windows, "d_end_exclusion": end_exclusion, "d_trims": trims,
            "e_batches": batches, "e_shard": shard, "e_genes": genes, "f_reuse": reuse, "f_reuse_no_clean": reuse_no_clean}
SWEEP_SEEDS = list(range(40))


def build(name):
    return BUILDERS[name]()


# ------------------------------------------------------------------------------------------------------------ harness
def to_params(p):
    prm = coverm_b200.Params()
    for k, v in p.items():
        setattr(prm, k, v)
    return prm


def _compare(where, rows, pairs, exp, csr):
    for f in ref.INT_FIELDS:
        want = np.array([r[f] for r in exp.rows], dtype=np.uint64)
        bad = np.flatnonzero(rows[f] != want)
        assert not len(bad), f"{where}: {f} differs in rows {bad[:10].tolist()}: got {rows[f][bad[:10]].tolist()}, " \
                             f"expected {want[bad[:10]].tolist()}"
    for f in ref.FLOAT_FIELDS:
        want = np.array([r[f] for r in exp.rows], dtype=np.float64)
        bad = np.flatnonzero(~np.isclose(rows[f], want, rtol=1e-12, atol=0.0))
        assert not len(bad), f"{where}: {f} differs in rows {bad[:10].tolist()}: got {rows[f][bad[:10]].tolist()}, " \
                             f"expected {want[bad[:10]].tolist()}"
    if not csr:
        assert not rows["hist_offset"].any() and len(pairs) == 0, f"{where}: histogram pairs without CMB_WANT_HIST_CSR"
        return
    assert len(pairs) == int(rows["hist_count"].sum()), f"{where}: {len(pairs)} pairs for {int(rows['hist_count'].sum())} bins"
    for r, hp in enumerate(exp.pairs):
        if hp is None:
            continue
        o, n = int(rows["hist_offset"][r]), int(rows["hist_count"][r])
        got = pairs[o:o + n]
        assert np.array_equal(got["depth"], hp[0]) and np.array_equal(got["count"], hp[1]), \
            f"{where}: histogram of row {r} differs: got {list(zip(got['depth'][:8], got['count'][:8]))}..., expected " \
            f"{list(zip(hp[0][:8], hp[1][:8]))}..."


def run_scenario(lib, sc, want, dense_spans=None, read_loads=None):
    """Every sample of `sc` on a new context of `lib`, `want` overriding the samples' own unless they fix it.  With
    `read_loads` (returns the last `#k2_load` line's fields of the sample just ended) the load counts are checked as well,
    for the dense threshold `dense_spans`."""
    ctx = coverm_b200.DeviceContext(lib=lib, batch_records=sc.batch_records)
    try:
        if sc.genes is not None:
            ctx.set_genes(sc.lens, sc.genes)
        else:
            ctx.set_reference(sc.lens, *(sc.shard or (0, len(sc.lens))))
        for i, smp in enumerate(sc.samples):
            p = dict(smp.params)
            if not smp.fixed_want:
                p["want"] = want
            where = f"{sc.name} sample {i} (want={p['want']}, E={p['contig_end_exclusion']}, trim={p['trim_min']}..{p['trim_max']})"
            exp = ref.expected(sc.lens, p, smp.records, shard=sc.shard, genes=sc.genes)
            ctx.set_params(to_params(p))
            ctx.begin_sample()
            ctx.submit_columns(smp.records)
            if exp.error:
                try:
                    ctx.end_sample()
                except coverm_b200.CmbError as e:
                    assert e.code == exp.error, f"{where}: expected error {exp.error}, got {e}"
                else:
                    raise AssertionError(f"{where}: expected error {exp.error}, the sample succeeded")
                continue
            rows, pairs = ctx.end_sample(want_pairs=True)
            _compare(where, rows, pairs, exp, bool(p["want"] & ref.WANT_HIST_CSR))
            if sc.genes is not None:
                seen, kept = ctx.fetch_gene_extras()
                assert np.array_equal(seen, exp.contig_seen) and kept == exp.kept_primary, f"{where}: gene extras differ"
            if read_loads is not None:
                got = read_loads()
                spans, dense = exp.load_counts(dense_spans)
                want_loads = dict(spans_loaded=spans, dense_chunks=dense, spans=exp.n_chunks * ref.CHUNK_SPANS, chunks=exp.n_chunks)
                assert got == want_loads, f"{where}: K2 loads {got}, expected {want_loads}"
    finally:
        ctx.close()
