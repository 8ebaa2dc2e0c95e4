"""coverm_b200 — H100-native replacement for CoverM's per-contig coverage hot path.

The product is the native library ``coverm_b200/libcoverm_b200.so`` (hand-written sm_90a CUDA kernels behind the C
ABI declared in ``include/coverm_b200.h`` and ``include/coverm_b200_host.h``) plus the ``coverm_b200/bin/coverm``
command-line binary.  This module is only a thin ctypes binding over that ABI for tests, ``bench.py`` and
``__graft_entry__.py``; there is no Python or CPU fallback — importing works anywhere, but every compute entry
point raises if the library or a CUDA device is missing.
"""
import ctypes as C
import os

ROOT = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(ROOT, "libcoverm_b200.so")
COVERM_BIN = os.path.join(ROOT, "bin", "coverm")
BAMGEN_BIN = os.path.join(ROOT, "bin", "bamgen")

CMBH_MAX_SAMPLES = 64


class CmbError(RuntimeError):
    """A failed cmb_* / cmbh_* call; `code` is the negative CMB_E_* value when the call returned one."""

    def __init__(self, msg, code=None):
        super().__init__(msg)
        self.code = code


# ---------------------------------------------------------------------------------------------- device ABI structs
class DeviceCfg(C.Structure):
    _fields_ = [("device", C.c_int32), ("batch_records", C.c_uint32), ("batch_intervals", C.c_uint32),
                ("n_staging", C.c_uint32)]


class Params(C.Structure):
    _fields_ = [("include_improper_pairs", C.c_uint8), ("include_supplementary", C.c_uint8),
                ("include_secondary", C.c_uint8), ("filtering", C.c_uint8), ("min_mapq", C.c_uint8),
                ("reserved0", C.c_uint8 * 3), ("min_aligned_length_single", C.c_uint32),
                ("min_percent_identity_single", C.c_float), ("min_aligned_percent_single", C.c_float),
                ("min_aligned_length_pair", C.c_uint32), ("min_percent_identity_pair", C.c_float),
                ("min_aligned_percent_pair", C.c_float), ("contig_end_exclusion", C.c_uint64),
                ("trim_min", C.c_float), ("trim_max", C.c_float), ("want", C.c_uint32), ("reserved1", C.c_uint32)]


class FilterMode(C.Structure):
    _fields_ = [("filter_single_reads", C.c_uint8), ("filter_pairs", C.c_uint8)]


class ReadBatch(C.Structure):
    _fields_ = [("capacity_records", C.c_uint32), ("capacity_intervals", C.c_uint32),
                ("tid", C.c_void_p), ("pos", C.c_void_p), ("flag", C.c_void_p), ("mapq", C.c_void_p),
                ("nm_state", C.c_void_p), ("nm", C.c_void_p), ("l_seq", C.c_void_p), ("aligned", C.c_void_p),
                ("del_", C.c_void_p), ("ins", C.c_void_p), ("iv_begin", C.c_void_p), ("iv_start", C.c_void_p),
                ("iv_len", C.c_void_p)]


class ContigStats(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_primary", C.c_uint64), ("n_nonsupp", C.c_uint64),
                ("sum_edit", C.c_uint64), ("sum_indel", C.c_uint64), ("sum_identity_primary", C.c_double),
                ("sum_identity_nonsupp", C.c_double), ("sum_depth_window", C.c_uint64),
                ("covered_window", C.c_uint64), ("covered_full", C.c_uint64), ("trimmed_total", C.c_uint64),
                ("trim_min_index", C.c_uint64), ("trim_max_index", C.c_uint64), ("var_k", C.c_uint64),
                ("var_ex", C.c_uint64), ("var_ex2", C.c_uint64), ("hist_offset", C.c_uint64),
                ("hist_count", C.c_uint32), ("reserved", C.c_uint32)]


class HistPair(C.Structure):
    _fields_ = [("depth", C.c_uint32), ("count", C.c_uint32)]


class Gene(C.Structure):
    _fields_ = [("tid", C.c_uint32), ("start", C.c_uint32), ("end", C.c_uint32)]


class SampleTiming(C.Structure):
    _fields_ = [("ms_zero", C.c_float), ("ms_accumulate", C.c_float), ("ms_scan", C.c_float),
                ("ms_finalize", C.c_float), ("ms_total", C.c_float), ("arena_elems", C.c_uint64),
                ("n_records", C.c_uint64), ("n_intervals", C.c_uint64), ("k1_launches", C.c_uint32),
                ("k2_launches", C.c_uint32), ("k3_launches", C.c_uint32), ("reserved", C.c_uint32)]


# ---------------------------------------------------------------------------------------------- host ABI structs
class MemInput(C.Structure):
    _fields_ = [("path", C.c_char_p), ("data", C.c_void_p), ("size", C.c_size_t)]


class SampleInfo(C.Structure):
    _fields_ = [("num_mapped_reads", C.c_uint64), ("num_reads", C.c_uint64), ("n_records", C.c_uint64),
                ("total_s", C.c_double), ("decode_s", C.c_double), ("submit_wait_s", C.c_double),
                ("end_sample_s", C.c_double), ("k0_ms", C.c_float), ("k1_ms", C.c_float), ("k2_ms", C.c_float),
                ("k3_ms", C.c_float), ("device_total_ms", C.c_float), ("k1_launches", C.c_uint32),
                ("k2_launches", C.c_uint32), ("k3_launches", C.c_uint32), ("arena_elems", C.c_uint64),
                ("n_intervals", C.c_uint64), ("h2d_bytes", C.c_uint64), ("device_decode", C.c_uint32),
                ("decode_host_blocks", C.c_uint32), ("decode_copy_inflate_ms", C.c_float), ("decode_chain_ms", C.c_float),
                ("decode_extract_ms", C.c_float), ("decode_launches", C.c_uint32), ("group_ranks", C.c_uint32),
                ("shard_blocks", C.c_uint32), ("total_blocks", C.c_uint32), ("range_probes", C.c_uint32), ("tid_begin", C.c_uint32), ("tid_end", C.c_uint32), ("decode_second_pass_blocks", C.c_uint32),
                ("gather_s", C.c_double), ("decode_copy_enqueue_wall_ms", C.c_float), ("decode_host_wall_ms", C.c_float)]


class HostResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("out", C.c_void_p), ("out_len", C.c_size_t), ("err", C.c_void_p),
                ("err_len", C.c_size_t), ("n_samples", C.c_uint32), ("samples", SampleInfo * CMBH_MAX_SAMPLES)]


DEVICE_SYMBOLS = ["cmb_abi_version", "cmb_create", "cmb_destroy", "cmb_last_error", "cmb_set_reference",
                  "cmb_set_params", "cmb_begin_sample", "cmb_acquire_batch", "cmb_submit_batch",
                  "cmb_submit_device_batch", "cmb_submit_bgzf", "cmb_decode_bgzf", "cmb_filter_plan", "cmb_filter_fetch", "cmb_filter_bgzf", "cmb_set_genes",
                  "cmb_deflate_begin", "cmb_deflate_feed", "cmb_deflate_finish", "cmb_filter_bgzf_deflate",
                  "cmb_set_genes_range", "cmb_fetch_gene_extras", "cmb_grow_buffers", "cmb_last_bgzf_batch", "cmb_end_sample", "cmb_comm_unique_id",
                  "cmb_comm_init", "cmb_comm_init_local", "cmb_comm_destroy", "cmb_comm_allgather", "cmb_allgather_stats", "cmb_kept_tid_range", "cmb_fetch_pairs", "cmb_end_sample_device",
                  "cmb_get_timing", "cmb_stream", "cmb_host_alloc", "cmb_host_free", "cmb_nvtx_push", "cmb_nvtx_pop",
                  "cmb_shard_begin", "cmb_shard_add", "cmb_shard_finish", "cmb_shard_begin_range", "cmb_shard_score",
                  "cmb_shard_exchange", "cmb_shard_export", "cmb_shard_import", "cmb_shard_choose", "cmb_shard_finish_group"]
class Tuples(C.Structure):
    _fields_ = [("n_contigs", C.c_uint32), ("contig_len", C.POINTER(C.c_uint64)), ("n_records", C.c_uint64),
                ("n_intervals", C.c_uint64), ("tid", C.POINTER(C.c_int32)), ("pos", C.POINTER(C.c_int32)),
                ("flag", C.POINTER(C.c_uint16)), ("mapq", C.POINTER(C.c_uint8)), ("nm_state", C.POINTER(C.c_uint8)),
                ("nm", C.POINTER(C.c_uint32)), ("l_seq", C.POINTER(C.c_uint32)), ("aligned", C.POINTER(C.c_uint32)),
                ("del_", C.POINTER(C.c_uint32)), ("ins", C.POINTER(C.c_uint32)), ("iv_begin", C.POINTER(C.c_uint32)),
                ("iv_start", C.POINTER(C.c_int32)), ("iv_len", C.POINTER(C.c_int32))]


HOST_SYMBOLS = ["cmbh_session_create", "cmbh_session_destroy", "cmbh_last_error", "cmbh_session_set_shard", "cmbh_session_set_group", "cmbh_session_set_group_output", "cmbh_session_ctx",
                "cmbh_run", "cmbh_plan_params", "cmbh_free_result", "cmbh_main", "cmbh_extract_tuples", "cmbh_free_tuples"]


def extract_tuples(path, threads=None):
    """Decode a BAM/SAM file into the SoA tuple columns of cmb_read_batch (host numpy arrays, no GPU)."""
    import numpy as np
    lib = load_library()
    t = Tuples()
    rc = lib.cmbh_extract_tuples(path.encode(), None, 0, int(threads or os.cpu_count() or 1), C.byref(t))
    if rc != 0:
        raise CmbError("cmbh_extract_tuples failed: " + lib.cmbh_last_error().decode())
    n, ni = t.n_records, t.n_intervals
    out = {"contig_len": np.ctypeslib.as_array(t.contig_len, (t.n_contigs,)).copy(), "n_records": n, "n_intervals": ni}
    for name, cnt in [("tid", n), ("pos", n), ("flag", n), ("mapq", n), ("nm_state", n), ("nm", n), ("l_seq", n),
                      ("aligned", n), ("del_", n), ("ins", n), ("iv_begin", n + 1), ("iv_start", ni), ("iv_len", ni)]:
        out[name] = np.ctypeslib.as_array(getattr(t, name), (cnt,)).copy() if cnt else np.zeros(0, dtype=np.int32)
    lib.cmbh_free_tuples(C.byref(t))
    return out

_lib = None


ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)


def comm_unique_id():
    """128 bytes identifying a new NCCL communicator (cmb_comm_unique_id); rank 0 creates it and shares it."""
    lib = load_library()
    buf = (C.c_uint8 * 128)()
    if lib.cmb_comm_unique_id(buf) != 0:
        raise CmbError("cmb_comm_unique_id failed: " + lib.cmb_last_error(None).decode())
    return bytes(buf)


def plan_params(argv):
    """cmb_params the `coverm <argv>` command line would hand to the device library (cmbh_plan_params)."""
    lib = load_library()
    args = (C.c_char_p * len(argv))(*[a.encode() for a in argv])
    prm = Params()
    if lib.cmbh_plan_params(len(argv), args, C.byref(prm)) != 0:
        raise CmbError("cmbh_plan_params failed: " + lib.cmbh_last_error().decode())
    return prm


def load_library(path=None):
    """Load libcoverm_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly if it is missing.
    `path` is for tests that bind another build of the same ABI explicitly; the product always uses LIB_PATH."""
    global _lib
    if path is None and _lib is not None:
        return _lib
    lib_path = path or LIB_PATH
    if not os.path.exists(lib_path):
        raise CmbError(f"{lib_path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no Python/CPU fallback)")
    lib = C.CDLL(lib_path)
    lib.cmb_abi_version.restype = C.c_int
    lib.cmb_create.argtypes = [C.POINTER(DeviceCfg), C.POINTER(C.c_void_p)]
    lib.cmb_destroy.argtypes = [C.c_void_p]
    lib.cmb_destroy.restype = None
    lib.cmb_last_error.argtypes = [C.c_void_p]
    lib.cmb_last_error.restype = C.c_char_p
    lib.cmb_set_reference.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_uint32, C.c_uint32]
    lib.cmb_set_params.argtypes = [C.c_void_p, C.POINTER(Params), C.POINTER(FilterMode)]
    lib.cmb_begin_sample.argtypes = [C.c_void_p]
    lib.cmb_acquire_batch.argtypes = [C.c_void_p, C.POINTER(ReadBatch)]
    lib.cmb_submit_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    lib.cmb_submit_device_batch.argtypes = [C.c_void_p, C.POINTER(ReadBatch), C.c_uint32, C.c_uint32]
    lib.cmb_end_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.cmb_fetch_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.cmb_set_genes.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(Gene)]
    if hasattr(lib, "cmb_set_genes_range"):  # libcoverm_b200 has it; the CPU emulator of the ABI used by tests may not
        lib.cmb_set_genes_range.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.c_uint32, C.POINTER(Gene), C.c_uint32,
                                            C.c_uint32]
    lib.cmb_fetch_gene_extras.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.cmb_end_sample_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    lib.cmb_get_timing.argtypes = [C.c_void_p, C.POINTER(SampleTiming)]
    lib.cmb_stream.argtypes = [C.c_void_p]
    lib.cmb_stream.restype = C.c_void_p
    lib.cmbh_session_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.cmbh_session_destroy.argtypes = [C.c_void_p]
    lib.cmbh_session_destroy.restype = None
    lib.cmbh_last_error.restype = C.c_char_p
    lib.cmbh_session_set_shard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    lib.cmbh_run.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(MemInput), C.c_int,
                             C.POINTER(HostResult)]
    lib.cmb_last_bgzf_batch.argtypes = [C.c_void_p, C.POINTER(ReadBatch), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    lib.cmbh_session_set_group_output.argtypes = [C.c_void_p, C.c_int]
    lib.cmbh_session_set_group.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.cmb_comm_unique_id.argtypes = [C.c_void_p]
    lib.cmb_allgather_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    lib.cmbh_session_ctx.argtypes = [C.c_void_p]
    lib.cmbh_session_ctx.restype = C.c_void_p
    lib.cmbh_plan_params.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_void_p]
    lib.cmbh_free_result.argtypes = [C.POINTER(HostResult)]
    lib.cmbh_free_result.restype = None
    lib.cmbh_extract_tuples.argtypes = [C.c_char_p, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(Tuples)]
    lib.cmbh_free_tuples.argtypes = [C.POINTER(Tuples)]
    lib.cmbh_free_tuples.restype = None
    if path is None:
        _lib = lib
    return lib


class RunResult:
    """status / stdout / stderr of one in-process `coverm` run.  The table text stays in the buffer the C ABI returned
    (``out_len`` bytes, freed with this object); ``out_bytes`` / ``out`` copy / decode it on first use."""

    def __init__(self, lib, res, err, samples):
        self._lib, self._res = lib, res
        self.status, self.out_len, self.err, self.samples = res.status, res.out_len, err, samples
        self._bytes = self._out = None

    @property
    def out_bytes(self):
        if self._bytes is None:
            self._bytes = C.string_at(self._res.out, self._res.out_len) if self._res.out else b""
        return self._bytes

    @property
    def out(self):
        if self._out is None:
            self._out = self.out_bytes.decode()
        return self._out

    def __del__(self):
        try:
            if self._res is not None:
                self._lib.cmbh_free_result(C.byref(self._res))
                self._res = None
        except Exception:
            pass


class Session:
    """One GPU context + host thread pool (cmbh_session): ``run(argv)`` is `coverm <argv...>` in-process."""

    def __init__(self, device=0, threads=None, lib=None):
        lib = lib or load_library()
        self._lib = lib
        self._h = C.c_void_p()
        threads = threads or (os.cpu_count() or 1)
        rc = lib.cmbh_session_create(int(device), int(threads), C.byref(self._h))
        if rc != 0:
            raise CmbError("cmbh_session_create failed: " + lib.cmbh_last_error().decode())

    def set_shard(self, tid_begin, tid_end):
        self._lib.cmbh_session_set_shard(self._h, tid_begin, tid_end)

    def set_group_output(self, every_rank_prints):
        self._lib.cmbh_session_set_group_output(self._h, 1 if every_rank_prints else 0)

    def set_group(self, rank, n_ranks, nccl_id=None, allgather=None):
        """Make this session rank `rank` of `n_ranks` processing every sample together (contig sharding).  `nccl_id`: the 128
        bytes of comm_unique_id() shared by the caller; or `allgather(send: bytes, n_ranks) -> bytes` (the ranks' buffers
        concatenated in rank order) for hosts without NCCL between them."""
        cb = None
        if allgather is not None:
            def _cb(user, send, nbytes, recv):
                try:
                    out = allgather(C.string_at(send, nbytes))
                    C.memmove(recv, out, nbytes * n_ranks)
                    return 0
                except Exception:
                    import traceback
                    traceback.print_exc()
                    return 1
            cb = ALLGATHER_FN(_cb)
        self._group_cb = cb  # keep the trampoline alive
        idbuf = (C.c_uint8 * 128).from_buffer_copy(nccl_id) if nccl_id is not None else None
        rc = self._lib.cmbh_session_set_group(self._h, int(rank), int(n_ranks), C.cast(idbuf, C.c_void_p) if idbuf is not None else None,
                                              C.cast(cb, C.c_void_p) if cb is not None else None, None)
        if rc != 0:
            raise CmbError("cmbh_session_set_group failed: " + self._lib.cmbh_last_error().decode())

    def device_context(self):
        """The session's cmb_ctx as a (borrowed) DeviceContext: continue on the device ABI after run()."""
        return DeviceContext(borrowed=self._lib.cmbh_session_ctx(self._h), lib=self._lib)

    def run(self, argv, memory_inputs=None):
        """memory_inputs: {path: bytes-like (e.g. numpy uint8 array / bytes)} read instead of the filesystem."""
        lib = self._lib
        args = (C.c_char_p * len(argv))(*[a.encode() for a in argv])
        mem = None
        keep = []
        n_mem = 0
        if memory_inputs:
            n_mem = len(memory_inputs)
            mem = (MemInput * n_mem)()
            for i, (path, buf) in enumerate(memory_inputs.items()):
                if hasattr(buf, "ctypes"):  # numpy array
                    ptr, size = buf.ctypes.data, buf.nbytes
                else:
                    cb = (C.c_char * len(buf)).from_buffer_copy(buf)
                    keep.append(cb)
                    ptr, size = C.addressof(cb), len(buf)
                mem[i].path = path.encode()
                mem[i].data = ptr
                mem[i].size = size
        res = HostResult()
        rc = lib.cmbh_run(self._h, len(argv), args, mem, n_mem, C.byref(res))
        if rc != 0:
            raise CmbError(f"cmbh_run failed with {rc}")
        err = C.string_at(res.err, res.err_len).decode() if res.err else ""
        samples = []
        for i in range(res.n_samples):
            s = res.samples[i]
            samples.append({f[0]: getattr(s, f[0]) for f in SampleInfo._fields_})
        return RunResult(lib, res, err, samples)

    def close(self):
        if self._h:
            self._lib.cmbh_session_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceContext:
    """Direct binding of the device-level ABI (cmb_*), used by bench.py for device-resident timing."""

    def __init__(self, device=0, batch_records=1 << 20, batch_intervals=0, n_staging=2, borrowed=None, lib=None):
        lib = lib or load_library()
        self._lib = lib
        self._h = C.c_void_p()
        self._owned = borrowed is None
        self.n_contigs = 0
        self.n_ref_contigs = 0
        if borrowed is not None:  # a cmb_ctx* owned by someone else (Session.device_context())
            self._h = C.c_void_p(borrowed)
            return
        cfg = DeviceCfg(device, batch_records, batch_intervals, n_staging)
        rc = lib.cmb_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise CmbError("cmb_create failed: " + lib.cmb_last_error(None).decode())

    def last_bgzf_batch(self):
        """(ReadBatch of device pointers, n_records, n_intervals) left in HBM by the last device-side decode."""
        b, nr, ni = ReadBatch(), C.c_uint32(), C.c_uint32()
        self._check(self._lib.cmb_last_bgzf_batch(self._h, C.byref(b), C.byref(nr), C.byref(ni)), "cmb_last_bgzf_batch")
        return b, nr.value, ni.value

    def _check(self, rc, what):
        if rc != 0:
            raise CmbError(f"{what} failed ({rc}): " + self._lib.cmb_last_error(self._h).decode(), rc)

    def set_reference(self, lens, tid_begin=0, tid_end=None):
        import numpy as np
        lens = np.ascontiguousarray(lens, dtype=np.uint64)
        self.n_contigs = len(lens)
        tid_end = self.n_contigs if tid_end is None else tid_end
        self._check(self._lib.cmb_set_reference(self._h, self.n_contigs, lens.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                tid_begin, tid_end), "cmb_set_reference")

    def set_genes(self, contig_lens, genes, tid_begin=None, tid_end=None):
        """Per-gene segments instead of contigs (cmb_set_genes): `genes` is a sequence of (tid, start, end) sorted by
        (tid, start).  Result rows are then one per gene (one placeholder row when there are none).  With `tid_begin` /
        `tid_end` (cmb_set_genes_range) only the records of those contigs count, and only their genes' rows are filled."""
        import numpy as np
        lens = np.ascontiguousarray(contig_lens, dtype=np.uint64)
        arr = (Gene * max(1, len(genes)))(*[Gene(*g) for g in genes])
        lens_p = lens.ctypes.data_as(C.POINTER(C.c_uint64))
        if tid_begin is None and tid_end is None:
            self._check(self._lib.cmb_set_genes(self._h, len(lens), lens_p, len(genes), arr), "cmb_set_genes")
        else:
            tid_begin = 0 if tid_begin is None else tid_begin
            tid_end = len(lens) if tid_end is None else tid_end
            self._check(self._lib.cmb_set_genes_range(self._h, len(lens), lens_p, len(genes), arr, tid_begin, tid_end),
                        "cmb_set_genes_range")
        self.n_contigs = max(1, len(genes))
        self.n_ref_contigs = len(lens)

    def fetch_gene_extras(self):
        """After end_sample in gene mode: (contig_seen as a uint8 array, kept primary records) (cmb_fetch_gene_extras)."""
        import numpy as np
        seen = np.zeros(max(1, self.n_ref_contigs), dtype=np.uint8)
        kept = C.c_uint64()
        self._check(self._lib.cmb_fetch_gene_extras(self._h, seen.ctypes.data, C.byref(kept)), "cmb_fetch_gene_extras")
        return seen[:self.n_ref_contigs], kept.value

    def set_params(self, params):
        mode = FilterMode()
        self._check(self._lib.cmb_set_params(self._h, C.byref(params), C.byref(mode)), "cmb_set_params")
        return mode

    def begin_sample(self):
        self._check(self._lib.cmb_begin_sample(self._h), "cmb_begin_sample")

    def submit_device_batch(self, batch, n_records, n_intervals):
        self._check(self._lib.cmb_submit_device_batch(self._h, C.byref(batch), n_records, n_intervals),
                    "cmb_submit_device_batch")

    def acquire_batch(self):
        b = ReadBatch()
        self._check(self._lib.cmb_acquire_batch(self._h, C.byref(b)), "cmb_acquire_batch")
        return b

    def submit_batch(self, n_records, n_intervals):
        self._check(self._lib.cmb_submit_batch(self._h, n_records, n_intervals), "cmb_submit_batch")

    _RECORD_COLUMNS = [("tid", C.c_int32), ("pos", C.c_int32), ("flag", C.c_uint16), ("mapq", C.c_uint8),
                       ("nm_state", C.c_uint8), ("nm", C.c_uint32), ("l_seq", C.c_uint32), ("aligned", C.c_uint32),
                       ("del_", C.c_uint32), ("ins", C.c_uint32)]

    def submit_columns(self, cols):
        """Copy host columns into the pinned batches of acquire_batch() and submit them, in as many batches as their
        capacity needs.  `cols` maps the cmb_read_batch field names (``del_`` for del) to array-likes; `iv_begin` has
        n_records + 1 entries and indexes `iv_start` / `iv_len`."""
        import numpy as np

        def put(ptr, ctype, values):
            if len(values):
                np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), (len(values),))[:] = values

        n = len(cols["tid"])
        ivb = np.asarray(cols["iv_begin"], dtype=np.int64)
        r0 = 0
        while r0 < n:
            b = self.acquire_batch()
            # as many records as fit both the record and the interval capacity of the batch
            r1 = min(n, r0 + b.capacity_records, int(np.searchsorted(ivb, ivb[r0] + b.capacity_intervals, "right")) - 1)
            if r1 <= r0:
                raise CmbError(f"record {r0} has more intervals than a staging batch holds ({b.capacity_intervals})")
            for name, ctype in self._RECORD_COLUMNS:
                put(getattr(b, name), ctype, np.asarray(cols[name])[r0:r1])
            i0, i1 = int(ivb[r0]), int(ivb[r1])
            put(b.iv_begin, C.c_uint32, ivb[r0:r1 + 1] - i0)  # iv_begin[n] = n_intervals
            put(b.iv_start, C.c_int32, np.asarray(cols["iv_start"])[i0:i1])
            put(b.iv_len, C.c_int32, np.asarray(cols["iv_len"])[i0:i1])
            self.submit_batch(r1 - r0, i1 - i0)
            r0 = r1

    def end_sample_device(self):
        p = C.c_void_p()
        self._check(self._lib.cmb_end_sample_device(self._h, C.byref(p)), "cmb_end_sample_device")
        return p.value

    def allgather_stats(self, tid_cuts):
        """cmb_allgather_stats without host copies: completes the per-contig table on every rank's device (collective)."""
        cuts = (C.c_uint32 * len(tid_cuts))(*tid_cuts)
        self._check(self._lib.cmb_allgather_stats(self._h, cuts, None, None, None), "cmb_allgather_stats")

    def end_sample(self, want_pairs=False):
        """(rows, number of CSR histogram pairs); with want_pairs (rows, pairs), the pairs fetched with cmb_fetch_pairs as a
        HistPair array (row r's are pairs[hist_offset : hist_offset + hist_count])."""
        import numpy as np
        rows = np.zeros(self.n_contigs, dtype=np.dtype(ContigStats))
        n_pairs = C.c_uint64()
        self._check(self._lib.cmb_end_sample(self._h, rows.ctypes.data, None, 0, C.byref(n_pairs)), "cmb_end_sample")
        if not want_pairs:
            return rows, n_pairs.value
        pairs = np.zeros(n_pairs.value, dtype=np.dtype(HistPair))
        if n_pairs.value:
            self._check(self._lib.cmb_fetch_pairs(self._h, pairs.ctypes.data, n_pairs.value), "cmb_fetch_pairs")
        return rows, pairs

    def timing(self):
        t = SampleTiming()
        self._lib.cmb_get_timing(self._h, C.byref(t))
        return {f[0]: getattr(t, f[0]) for f in SampleTiming._fields_}

    def stream(self):
        return self._lib.cmb_stream(self._h)

    def close(self):
        if self._h and self._owned:
            self._lib.cmb_destroy(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
