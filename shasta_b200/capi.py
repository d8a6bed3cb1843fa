"""ctypes binding of the C ABI (include/shasta_b200.h -> shasta_b200/lib/libshasta_b200.so).

There is no CPU fallback: importing this module without the built library, or creating a Context
without an H100 (sm_90), raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libshasta_b200.so")


class ShastaB200Error(RuntimeError):
    """Mirrors the std::runtime_error the reference throws (src/SHASTA_ASSERT.hpp, src/LowHash0.cpp:86)."""

    def __init__(self, status, message):
        super().__init__(message)
        self.status = status


class LowHashParams(C.Structure):
    _fields_ = [("m", C.c_uint64), ("hashFraction", C.c_double), ("minHashIterationCount", C.c_uint64),
                ("alignmentCandidatesPerRead", C.c_double), ("log2MinHashBucketCount", C.c_uint64),
                ("minBucketSize", C.c_uint64), ("maxBucketSize", C.c_uint64), ("minFrequency", C.c_uint64),
                ("threadCount", C.c_uint64), ("perIterationMerge", C.c_uint32), ("reserved", C.c_uint32)]


class LowHashResult(C.Structure):
    _fields_ = [("iterations", C.c_uint64), ("log2BucketCount", C.c_uint64), ("lowHashCount", C.c_uint64),
                ("pairCount", C.c_uint64), ("candidateCount", C.c_uint64), ("sweepMs", C.c_double),
                ("totalMs", C.c_double), ("sweepLaunches", C.c_uint64), ("kernelLaunches", C.c_uint64),
                ("candidateDigest", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class AlignOptions(C.Structure):
    """shb_align_options: AlignOptions of src/AssemblerOptions.hpp:177-199 + k."""
    _fields_ = [("alignMethod", C.c_int32), ("maxSkip", C.c_int32), ("maxDrift", C.c_int32), ("maxTrim", C.c_int32),
                ("maxMarkerFrequency", C.c_int32), ("minAlignedMarkerCount", C.c_int32), ("minAlignedFraction", C.c_double),
                ("matchScore", C.c_int32), ("mismatchScore", C.c_int32), ("gapScore", C.c_int32),
                ("downsamplingFactor", C.c_double), ("bandExtend", C.c_int32), ("maxBand", C.c_int32),
                ("sameChannelReadAlignmentSuppressDeltaThreshold", C.c_int32), ("suppressContainments", C.c_int32),
                ("align4DeltaX", C.c_uint64), ("align4DeltaY", C.c_uint64), ("align4MinEntryCountPerCell", C.c_uint64),
                ("align4MaxDistanceFromBoundary", C.c_uint64), ("k", C.c_uint32), ("reserved", C.c_uint32)]


class AlignResult(C.Structure):
    _fields_ = [("candidateCount", C.c_uint64), ("alignmentCount", C.c_uint64), ("skippedCount", C.c_uint64),
                ("dpCells", C.c_uint64), ("dpMs", C.c_double), ("totalMs", C.c_double), ("kernelLaunches", C.c_uint64),
                ("outputCopyMs", C.c_double), ("hostWallMs", C.c_double), ("dpUsefulCells", C.c_uint64),
                ("tooWideCount", C.c_uint64), ("workers", C.c_uint64), ("alignmentDataDigest", C.c_uint64),
                ("compressedDigest", C.c_uint64)]


class MarkerResult(C.Structure):
    _fields_ = [("readCount", C.c_uint64), ("baseCount", C.c_uint64), ("markerCount", C.c_uint64), ("totalMs", C.c_double),
                ("kernelLaunches", C.c_uint64), ("h2dBytes", C.c_uint64)]


class DistTiming(C.Structure):
    _fields_ = [("sweepSeconds", C.c_double), ("partitionSeconds", C.c_double), ("exchangeSeconds", C.c_double),
                ("processSeconds", C.c_double), ("finalSeconds", C.c_double), ("gatherSeconds", C.c_double),
                ("totalSeconds", C.c_double), ("entriesReceived", C.c_uint64), ("pairsReceived", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# Defaults of src/AssemblerOptions.cpp:380-489
ALIGN_DEFAULTS = dict(alignMethod=3, maxSkip=30, maxDrift=30, maxTrim=30, maxMarkerFrequency=10, minAlignedMarkerCount=100,
                      minAlignedFraction=0.4, matchScore=6, mismatchScore=-1, gapScore=-1, downsamplingFactor=0.1,
                      bandExtend=10, maxBand=1000, sameChannelReadAlignmentSuppressDeltaThreshold=0, suppressContainments=0,
                      align4DeltaX=200, align4DeltaY=10, align4MinEntryCountPerCell=10, align4MaxDistanceFromBoundary=100,
                      k=10, reserved=0)


def make_align_options(**kw):
    d = dict(ALIGN_DEFAULTS)
    d.update(kw)
    return AlignOptions(**d)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ShastaB200Error(2, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                     "(the CUDA extension is required; there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.shb_last_error.restype = C.c_char_p
        L.shb_context_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.shb_context_destroy.argtypes = [C.c_void_p]
        L.shb_free.argtypes = [C.c_void_p]
        L.shb_trim_host_cache.argtypes = []
        L.shb_trim_host_cache.restype = None
        L.shb_set_markers.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.shb_set_markers_device.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.shb_lowhash0.argtypes = [C.c_void_p, C.POINTER(LowHashParams), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                   C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(LowHashResult)]
        L.shb_find_alignment_candidates_lowhash0.argtypes = [
            C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LowHashParams),
            C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(LowHashResult)]
        L.shb_compute_alignments.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(AlignOptions), C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                             C.POINTER(AlignResult)]
        L.shb_compute_alignment_table.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_find_markers.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(MarkerResult)]
        L.shb_dist_unique_id.argtypes = [C.c_void_p]
        L.shb_dist_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.shb_dist_attach.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.shb_dist_finalize.argtypes = [C.c_void_p]
        L.shb_dist_finalize.restype = None
        L.shb_lowhash0_sharded.argtypes = [C.c_void_p, C.POINTER(LowHashParams), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                                           C.c_void_p, C.POINTER(LowHashResult)]
        L.shb_compute_alignments_sharded.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(AlignOptions), C.POINTER(C.c_void_p),
                                                     C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                                     C.POINTER(AlignResult)]
        L.shb_dist_timing_get.argtypes = [C.c_void_p, C.POINTER(DistTiming)]
        L.shb_align_oriented_reads.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(AlignOptions), C.POINTER(C.c_void_p),
                                               C.POINTER(C.c_uint64), C.c_void_p]
        L.shb_compute_candidate_table.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_create_read_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.POINTER(C.c_void_p),
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_digest_records.restype = C.c_uint64
        L.shb_digest_records.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32]
        L.shb_digest_compressed.restype = C.c_uint64
        L.shb_digest_compressed.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.shb_synth_generate.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_double, C.c_double, C.c_uint64, C.c_void_p, C.c_void_p,
                                         C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_device_free.argtypes = [C.c_void_p]
        L.shb_markers_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.shb_lowhash_begin.argtypes = [C.c_void_p, C.POINTER(LowHashParams), C.POINTER(C.c_uint64)]
        L.shb_lowhash_sweep.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
        L.shb_lowhash_slab.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_device_partition.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                           C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.shb_lowhash_process_entries.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.shb_lowhash_local_pairs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.shb_lowhash_set_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.shb_lowhash_emit.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.shb_lowhash_stats_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.shb_lowhash_counters.argtypes = [C.c_void_p, C.POINTER(LowHashResult)]
        L.shb_copy_device_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        _lib = L
    return _lib


def _check(status):
    if status != 0:
        raise ShastaB200Error(status, lib().shb_last_error().decode())


def make_lowhash_params(m=4, hashFraction=0.01, minHashIterationCount=10, alignmentCandidatesPerRead=20.0,
                        log2MinHashBucketCount=0, minBucketSize=0, maxBucketSize=10, minFrequency=2,
                        threadCount=0, perIterationMerge=0):
    return LowHashParams(m, hashFraction, minHashIterationCount, alignmentCandidatesPerRead, log2MinHashBucketCount,
                         minBucketSize, maxBucketSize, minFrequency, threadCount, perIterationMerge, 0)


def _ptr(a):
    return a.ctypes.data if a is not None else None


class Context:
    """One per GPU (shb_context)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        _check(lib().shb_context_create(device, C.byref(self._h)))
        self.read_count = 0
        self._keep = None

    def close(self):
        if self._h:
            lib().shb_context_destroy(self._h)
            self._h = C.c_void_p()

    def find_markers(self, k, word_offsets, words, base_counts, flags, kmer_table=None, is_marker_bitmap=None, want_host=True):
        """Assembler::findMarkers on the device (shb_find_markers). Reads in LongBaseSequences layout. Returns
        (toc uint64[2R+1], data7 uint8[7M]) when want_host, and the MarkerResult; the context then holds the markers."""
        word_offsets = np.ascontiguousarray(word_offsets, np.uint64)
        words = np.ascontiguousarray(words, np.uint64)
        base_counts = np.ascontiguousarray(base_counts, np.uint64)
        flags = np.ascontiguousarray(flags, np.uint8)
        R = len(base_counts)
        kt = None if kmer_table is None else np.ascontiguousarray(kmer_table, np.uint8)
        bm = None if is_marker_bitmap is None else np.ascontiguousarray(is_marker_bitmap, np.uint32)
        toc, data = C.c_void_p(), C.c_void_p()
        res = MarkerResult()
        _check(lib().shb_find_markers(self._h, int(k), R, _ptr(word_offsets), _ptr(words), _ptr(base_counts), _ptr(kt), _ptr(bm),
                                      _ptr(flags), C.byref(toc) if want_host else None, C.byref(data) if want_host else None, C.byref(res)))
        self.read_count = R
        if not want_host:
            return None, None, res
        tocn = np.ctypeslib.as_array(C.cast(toc, C.POINTER(C.c_uint64)), (2 * R + 1,)).copy()
        M = int(tocn[-1])
        datan = np.ctypeslib.as_array(C.cast(data, C.POINTER(C.c_uint8)), (7 * M,)).copy() if M else np.zeros(0, np.uint8)
        lib().shb_free(toc)
        lib().shb_free(data)
        return tocn, datan, res

    # ---- multi-GPU (one process per GPU; NCCL inside the library) -------------------------------------------------
    def dist_init(self, world, rank, unique_id: bytes):
        """Collective: joins the NCCL communicator described by unique_id (dist_unique_id() of rank 0)."""
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        _check(lib().shb_dist_init(self._h, int(world), int(rank), buf))

    def dist_finalize(self):
        lib().shb_dist_finalize(self._h)

    def lowhash0_sharded(self, params: LowHashParams, want_stats=True):
        """Collective. Returns (this rank's block of the candidates uint32[n,3], stats uint64[R,3] | None, LowHashResult)."""
        cand = C.c_void_p()
        n = C.c_uint64()
        res = LowHashResult()
        stats = np.zeros((self.read_count, 3), np.uint64) if want_stats else None
        _check(lib().shb_lowhash0_sharded(self._h, C.byref(params), C.byref(cand), C.byref(n), _ptr(stats), C.byref(res)))
        out = _records_to_array(cand, n.value)
        return out, stats, res

    def dist_timing(self):
        t = DistTiming()
        _check(lib().shb_dist_timing_get(self._h, C.byref(t)))
        return t

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_markers(self, toc, data7, flags, read_begin=0, read_end=None, read_count_total=None, total_marker_count=None):
        toc = np.ascontiguousarray(toc, dtype=np.uint64)
        data7 = np.ascontiguousarray(data7, dtype=np.uint8)
        flags = np.ascontiguousarray(flags, dtype=np.uint8)
        n_local = (len(toc) - 1) // 2
        if read_count_total is None:
            read_count_total = n_local
        if read_end is None:
            read_end = read_begin + n_local
        if total_marker_count is None:
            total_marker_count = int(toc[-1])
        _check(lib().shb_set_markers(self._h, read_count_total, read_begin, read_end, _ptr(toc), _ptr(data7), _ptr(flags), total_marker_count))
        self.read_count = read_count_total

    def set_markers_device(self, toc, kmer_ids_device_ptr, flags, keepalive=None, read_begin=0, read_end=None,
                           read_count_total=None, total_marker_count=None):
        toc = np.ascontiguousarray(toc, dtype=np.uint64)
        flags = np.ascontiguousarray(flags, dtype=np.uint8)
        n_local = (len(toc) - 1) // 2
        if read_count_total is None:
            read_count_total = n_local
        if read_end is None:
            read_end = read_begin + n_local
        if total_marker_count is None:
            total_marker_count = int(toc[-1])
        _check(lib().shb_set_markers_device(self._h, read_count_total, read_begin, read_end, _ptr(toc),
                                            C.c_void_p(kmer_ids_device_ptr), _ptr(flags), total_marker_count))
        self._keep = keepalive
        self.read_count = read_count_total

    def lowhash0(self, params: LowHashParams, want_stats=True, max_iter_summary=0):
        """Returns (candidates uint32[n,3] = (readId0, readId1, isSameStrand), stats uint64[R,3] | None,
        iterSummary uint64[iters,2] | None, LowHashResult)."""
        cand = C.c_void_p()
        n = C.c_uint64()
        res = LowHashResult()
        stats = np.zeros((self.read_count, 3), np.uint64) if want_stats else None
        summ = np.zeros((max_iter_summary, 2), np.uint64) if max_iter_summary else None
        _check(lib().shb_lowhash0(self._h, C.byref(params), C.byref(cand), C.byref(n), _ptr(stats), _ptr(summ),
                                  max_iter_summary, C.byref(res)))
        out = _records_to_array(cand, n.value)
        if summ is not None:
            summ = summ[:min(res.iterations, max_iter_summary)]
        return out, stats, summ, res

    def find_alignment_candidates_lowhash0(self, toc, data7, flags, params: LowHashParams, want_stats=True):
        """Host buffers in, host buffers out: the call a reference maintainer binds (INTEGRATION.md)."""
        toc = np.ascontiguousarray(toc, dtype=np.uint64)
        data7 = np.ascontiguousarray(data7, dtype=np.uint8)
        flags = np.ascontiguousarray(flags, dtype=np.uint8)
        R = (len(toc) - 1) // 2
        cand = C.c_void_p()
        n = C.c_uint64()
        res = LowHashResult()
        stats = np.zeros((R, 3), np.uint64) if want_stats else None
        _check(lib().shb_find_alignment_candidates_lowhash0(self._h, R, _ptr(toc), _ptr(data7), _ptr(flags), C.byref(params),
                                                           C.byref(cand), C.byref(n), _ptr(stats), C.byref(res)))
        self.read_count = R
        out = _records_to_array(cand, n.value)
        return out, stats, res


def trim_host_cache():
    """Return the recycled host result buffers to the operating system (shb_trim_host_cache)."""
    lib().shb_trim_host_cache()


class DeviceMarkers:
    """Synthetic markers generated on the device (bench/test utility)."""

    def __init__(self, toc, flags, kmer_ptr, data7_ptr):
        self.toc = toc
        self.flags = flags
        self.kmer_ptr = kmer_ptr
        self.data7_ptr = data7_ptr
        self.marker_count = int(toc[-1])

    def kmer_ids_to_host(self):
        out = np.empty(self.marker_count, np.uint32)
        _check(lib().shb_copy_device_to_host(_ptr(out), C.c_void_p(self.kmer_ptr), out.nbytes))
        return out

    def data7_to_host(self, out=None):
        if out is None:
            out = np.empty(self.marker_count * 7, np.uint8)
        _check(lib().shb_copy_device_to_host(_ptr(out), C.c_void_p(self.data7_ptr), self.marker_count * 7))
        return out

    def free(self, names=("kmer_ptr", "data7_ptr")):
        for name in names:
            p = getattr(self, name)
            if p:
                lib().shb_device_free(C.c_void_p(p))
                setattr(self, name, None)


def synth_generate_device(ctx: Context, p, want_data7=True, read_begin=0, read_end=None) -> DeviceMarkers:
    """shasta_b200.synth.generate(p) on the GPU: bit-identical markers, device resident. With read_begin/read_end
    only that read range is generated (toc relative to it; flags cover all reads)."""
    from . import synth
    gk, gpos = synth.genome(p)
    start, span, rev = synth.read_windows(p)
    if read_end is None:
        read_end = p.reads
    n = read_end - read_begin
    gk = np.ascontiguousarray(gk, np.uint32)
    gpos = np.ascontiguousarray(gpos, np.uint64)
    toc = np.zeros(2 * n + 1, np.uint64)
    kptr = C.c_void_p()
    dptr = C.c_void_p()
    _check(lib().shb_synth_generate(ctx._h, p.seed, p.k, p.drop, p.ins, len(gk), _ptr(gk), _ptr(gpos), read_begin, n,
                                    _ptr(np.ascontiguousarray(start[read_begin:read_end], np.int64)),
                                    _ptr(np.ascontiguousarray(span[read_begin:read_end], np.int64)),
                                    _ptr(np.ascontiguousarray(rev[read_begin:read_end], np.uint8)), _ptr(toc), C.byref(kptr),
                                    C.byref(dptr) if want_data7 else None))
    return DeviceMarkers(toc, synth.read_flags(p), kptr.value, dptr.value if want_data7 else None)


def _owned_array(ptr, count, dtype):
    """numpy view (no copy) of a host buffer returned by the library; shb_free runs when the array is garbage collected."""
    import weakref
    dtype = np.dtype(dtype)
    nbytes = int(count) * dtype.itemsize
    if not ptr or nbytes == 0:
        if ptr:
            lib().shb_free(ptr)
        return np.zeros(0, dtype)
    address = ptr.value if isinstance(ptr, C.c_void_p) else int(ptr)
    buf = (C.c_uint8 * nbytes).from_address(address)
    weakref.finalize(buf, lib().shb_free, C.c_void_p(address))
    return np.frombuffer(buf, dtype=dtype)


def candidates_to_records(cand):
    """uint32[n,3] (readId0, readId1, isSameStrand) -> n 12-byte OrientedReadPair records (as uint32[n,3])."""
    # The library reads byte 0 of the third word (0 / 1); no copy when the array already has the record layout.
    return np.ascontiguousarray(cand, dtype=np.uint32).reshape(-1, 3)


def compute_alignments(ctx: Context, candidates, options: AlignOptions):
    """Assembler::computeAlignments on the markers held by ctx.
    Returns (records uint32[count,16], compressedToc uint64[count+1], compressedData uint8[], AlignResult)."""
    cand = candidates_to_records(candidates)
    rec = C.c_void_p()
    cnt = C.c_uint64()
    toc = C.c_void_p()
    data = C.c_void_p()
    res = AlignResult()
    _check(lib().shb_compute_alignments(ctx._h, _ptr(cand), len(cand), C.byref(options), C.byref(rec), C.byref(cnt),
                                        C.byref(toc), C.byref(data), C.byref(res)))
    n = cnt.value
    tocn = _owned_array(toc, n + 1, np.uint64)
    nb = int(tocn[-1])
    records = _owned_array(rec, 16 * n, np.uint32).reshape(n, 16)
    datan = _owned_array(data, nb, np.uint8)
    return records, tocn, datan, res


def dist_unique_id() -> bytes:
    """128-byte NCCL unique id (rank 0 creates it and ships it to the other ranks)."""
    buf = (C.c_uint8 * 128)()
    _check(lib().shb_dist_unique_id(buf))
    return bytes(buf)


def compute_alignments_sharded(ctx: Context, candidates, options: AlignOptions):
    """Assembler::computeAlignments on this rank's block of candidates; the k-mer ids of all ranks are gathered into this
    GPU on the first call after the markers changed (collective then). Same returns as compute_alignments."""
    cand = candidates_to_records(candidates)
    rec = C.c_void_p()
    cnt = C.c_uint64()
    toc = C.c_void_p()
    data = C.c_void_p()
    res = AlignResult()
    _check(lib().shb_compute_alignments_sharded(ctx._h, _ptr(cand), len(cand), C.byref(options), C.byref(rec), C.byref(cnt),
                                                C.byref(toc), C.byref(data), C.byref(res)))
    n = cnt.value
    tocn = _owned_array(toc, n + 1, np.uint64)
    nb = int(tocn[-1])
    records = _owned_array(rec, 16 * n, np.uint32).reshape(n, 16)
    datan = _owned_array(data, nb, np.uint8)
    return records, tocn, datan, res


def compute_alignment_table(ctx: Context, records, read_count):
    """Assembler::computeAlignmentTable. Returns (toc uint32[2R+1], table uint32[4n])."""
    rec = np.ascontiguousarray(records, np.uint32).reshape(-1, 16)
    toc = C.c_void_p()
    data = C.c_void_p()
    _check(lib().shb_compute_alignment_table(ctx._h, _ptr(rec), len(rec), read_count, C.byref(toc), C.byref(data)))
    tocn = np.ctypeslib.as_array(C.cast(toc, C.POINTER(C.c_uint32)), (2 * read_count + 1,)).copy()
    datan = np.ctypeslib.as_array(C.cast(data, C.POINTER(C.c_uint32)), (4 * len(rec),)).copy() if len(rec) else np.zeros(0, np.uint32)
    lib().shb_free(toc)
    lib().shb_free(data)
    return tocn, datan


def create_read_graph(ctx: Context, records, read_count, max_alignment_count):
    """Assembler::createReadGraph, ReadGraph.creationMethod 0 (shb_create_read_graph). records uint32[n,16] must be a writable,
    C-contiguous array: AlignmentInfo::isInReadGraph is updated in place.
    Returns (keep uint8[n], edges uint32[E,4] = 16-byte ReadGraphEdge records, connectivityToc uint32[2R+1], connectivityData uint32[2E]);
    each connectivity row lists its edges in decreasing edge index, the reference's order. A kept alignment whose edge is not
    ordered (readIds[0] > readIds[1], or a read aligned to itself) raises ShastaB200Error (SHB_ERR_INVALID), records untouched."""
    assert records.dtype == np.uint32 and records.flags["C_CONTIGUOUS"] and records.flags["WRITEABLE"]
    rec = records.reshape(-1, 16)
    keep, edges, toc, data = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    e = C.c_uint64()
    _check(lib().shb_create_read_graph(ctx._h, _ptr(rec), len(rec), int(read_count), int(max_alignment_count), C.byref(keep), C.byref(edges),
                                       C.byref(e), C.byref(toc), C.byref(data)))
    keepn = _owned_array(keep, len(rec), np.uint8)
    edgesn = _owned_array(edges, 4 * e.value, np.uint32).reshape(-1, 4)
    tocn = _owned_array(toc, 2 * int(read_count) + 1, np.uint32)
    datan = _owned_array(data, 2 * e.value, np.uint32)
    return keepn, edgesn, tocn, datan


class ReadGraph2Criteria(C.Structure):
    _fields_ = [("minAlignedFraction", C.c_double), ("minAlignedMarkerCount", C.c_uint64), ("maxDrift", C.c_uint64),
                ("maxSkip", C.c_uint64), ("maxTrim", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def create_read_graph2(ctx: Context, records, read_count, max_alignment_count, marker_count_percentile, aligned_fraction_percentile,
                       max_skip_percentile, max_drift_percentile, max_trim_percentile):
    """Assembler::createReadGraph2, ReadGraph.creationMethod 2 (shb_create_read_graph2). records as in create_read_graph.
    Returns (criteria dict, keep, edges, connectivityToc, connectivityData), and refuses what create_read_graph refuses."""
    assert records.dtype == np.uint32 and records.flags["C_CONTIGUOUS"] and records.flags["WRITEABLE"]
    rec = records.reshape(-1, 16)
    keep, edges, toc, data = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    e = C.c_uint64()
    crit = ReadGraph2Criteria()
    f = lib().shb_create_read_graph2
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                  C.POINTER(ReadGraph2Criteria), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64),
                  C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    _check(f(ctx._h, _ptr(rec), len(rec), int(read_count), int(max_alignment_count), float(marker_count_percentile),
             float(aligned_fraction_percentile), float(max_skip_percentile), float(max_drift_percentile), float(max_trim_percentile),
             C.byref(crit), C.byref(keep), C.byref(edges), C.byref(e), C.byref(toc), C.byref(data)))
    keepn = _owned_array(keep, len(rec), np.uint8)
    edgesn = _owned_array(edges, 4 * e.value, np.uint32).reshape(-1, 4)
    tocn = _owned_array(toc, 2 * int(read_count) + 1, np.uint32)
    datan = _owned_array(data, 2 * e.value, np.uint32)
    return crit.asdict(), keepn, edgesn, tocn, datan


def align_oriented_reads(ctx: Context, oriented_read_id0, oriented_read_id1, options: AlignOptions):
    """Single pair in the orientation given (shb_align_oriented_reads). Returns (ordinals uint32[n,2], info uint32[13])."""
    ords = C.c_void_p()
    n = C.c_uint64()
    info = np.zeros(13, np.uint32)
    _check(lib().shb_align_oriented_reads(ctx._h, int(oriented_read_id0), int(oriented_read_id1), C.byref(options), C.byref(ords),
                                          C.byref(n), _ptr(info)))
    if not ords or n.value == 0:
        if ords:
            lib().shb_free(ords)
        return np.zeros((0, 2), np.uint32), info
    out = np.ctypeslib.as_array(C.cast(ords, C.POINTER(C.c_uint32)), (n.value, 2)).copy()
    lib().shb_free(ords)
    return out, info


def compute_candidate_table(ctx: Context, candidates, read_count):
    """AlignmentCandidates::computeCandidateTable. Returns (toc uint64[2R+1], table uint64[4n])."""
    cand = candidates_to_records(candidates)
    toc = C.c_void_p()
    data = C.c_void_p()
    _check(lib().shb_compute_candidate_table(ctx._h, _ptr(cand), len(cand), read_count, C.byref(toc), C.byref(data)))
    tocn = np.ctypeslib.as_array(C.cast(toc, C.POINTER(C.c_uint64)), (2 * read_count + 1,)).copy()
    datan = np.ctypeslib.as_array(C.cast(data, C.POINTER(C.c_uint64)), (4 * len(cand),)).copy() if len(cand) else np.zeros(0, np.uint64)
    lib().shb_free(toc)
    lib().shb_free(data)
    return tocn, datan


def digest_records(records, words):
    """shb_digest_records on a host array of `words`-word records (order independent; sums over partitions)."""
    r = np.ascontiguousarray(records, np.uint32).reshape(-1, words)
    return int(lib().shb_digest_records(_ptr(r), len(r), words))


def digest_candidates(cand):
    """Digest of candidates given as uint32[n,3] (readId0, readId1, isSameStrand)."""
    return digest_records(candidates_to_records(cand), 3)


def digest_compressed(records, ctoc, cdata):
    r = np.ascontiguousarray(records, np.uint32).reshape(-1, 16)
    t = np.ascontiguousarray(ctoc, np.uint64)
    d = np.ascontiguousarray(cdata, np.uint8)
    return int(lib().shb_digest_compressed(_ptr(r), len(r), _ptr(t), _ptr(d)))


def _records_to_array(ptr, n):
    """12-byte OrientedReadPair records -> uint32[n,3] with column 2 = isSameStrand (byte 0 of the third word)."""
    if n == 0:
        if ptr:
            lib().shb_free(ptr)
        return np.zeros((0, 3), np.uint32)
    # No copy: the library writes the third word as 0 / 1 (byte 0 = isSameStrand, padding bytes zero).
    return _owned_array(ptr, 3 * n, np.uint32).reshape(n, 3)


# ---- flagPalindromicReads (shb_flag_palindromic_reads) ---------------------------------------------------------------
class PalindromicParams(C.Structure):
    """shb_palindromic_params: the arguments of Assembler::flagPalindromicReads (threadCount is ignored)."""
    _fields_ = [("maxSkip", C.c_uint32), ("maxDrift", C.c_uint32), ("maxMarkerFrequency", C.c_uint32), ("deltaThreshold", C.c_uint32),
                ("alignedFractionThreshold", C.c_double), ("nearDiagonalFractionThreshold", C.c_double), ("threadCount", C.c_uint64)]


class PalindromicResult(C.Structure):
    _fields_ = [("readCount", C.c_uint64), ("palindromicReadCount", C.c_uint64), ("exactReadCount", C.c_uint64),
                ("vertexCount", C.c_uint64), ("edgeCount", C.c_uint64), ("heapPushCount", C.c_uint64),
                ("heapsortFallbackCount", C.c_uint64), ("totalMs", C.c_double), ("exactMs", C.c_double),
                ("kernelLaunches", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def make_palindromic_params(maxSkip=100, maxDrift=100, maxMarkerFrequency=10, alignedFractionThreshold=0.1,
                            nearDiagonalFractionThreshold=0.1, deltaThreshold=100, threadCount=0):
    return PalindromicParams(maxSkip=int(maxSkip), maxDrift=int(maxDrift), maxMarkerFrequency=int(maxMarkerFrequency),
                             deltaThreshold=int(deltaThreshold), alignedFractionThreshold=float(alignedFractionThreshold),
                             nearDiagonalFractionThreshold=float(nearDiagonalFractionThreshold), threadCount=int(threadCount))


def flag_palindromic_reads(ctx: Context, params: PalindromicParams, read_flags=None, want_counts=True):
    """Flags palindromic reads on the markers ctx holds. read_flags (uint8[R], optional) is updated in place (bit 0 only).
    Returns (aligned uint32[R] or None, nearDiagonal uint32[R] or None, PalindromicResult). For reads decided without an
    alignment the counts are the prefilter's bounds (see include/shasta_b200.h)."""
    L = lib()
    f = L.shb_flag_palindromic_reads
    f.argtypes = [C.c_void_p, C.POINTER(PalindromicParams), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PalindromicResult)]
    R = ctx.read_count
    aligned = np.zeros(R, np.uint32) if want_counts else None
    near = np.zeros(R, np.uint32) if want_counts else None
    if read_flags is not None:
        assert read_flags.dtype == np.uint8 and read_flags.flags["C_CONTIGUOUS"] and len(read_flags) == R
    res = PalindromicResult()
    _check(f(ctx._h, C.byref(params), None if read_flags is None else read_flags.ctypes.data,
             None if aligned is None else aligned.ctypes.data, None if near is None else near.ctypes.data, C.byref(res)))
    return aligned, near, res


def palindromic_read_alignment(ctx: Context, read_id, params: PalindromicParams):
    """The alignment of read_id against its reverse complement (method 0). Returns ordinals uint32[n,2]."""
    L = lib()
    f = L.shb_palindromic_read_alignment
    f.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(PalindromicParams), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    ords = C.c_void_p()
    n = C.c_uint64()
    _check(f(ctx._h, int(read_id), C.byref(params), C.byref(ords), C.byref(n)))
    out = np.ctypeslib.as_array(C.cast(ords, C.POINTER(C.c_uint32)), (n.value, 2)).copy() if n.value else np.zeros((0, 2), np.uint32)
    if ords:
        L.shb_free(ords)
    return out


# ---- createMarkerGraphVertices (shb_create_marker_graph_vertices) ----------------------------------------------------
class MarkerGraphParams(C.Structure):
    """shb_marker_graph_params: the arguments of Assembler::createMarkerGraphVertices (threadCount is ignored)."""
    _fields_ = [("minCoverage", C.c_uint64), ("maxCoverage", C.c_uint64), ("minCoveragePerStrand", C.c_uint64),
                ("allowDuplicateMarkers", C.c_uint64), ("peakFinderMinAreaFraction", C.c_double),
                ("peakFinderAreaStartIndex", C.c_uint64), ("threadCount", C.c_uint64)]


class MarkerGraphResult(C.Structure):
    _fields_ = [("markerCount", C.c_uint64), ("minCoverageUsed", C.c_uint64), ("peakFinderFailed", C.c_uint64),
                ("peakFinderObservedAreaFraction", C.c_double), ("edgePairsUsed", C.c_uint64), ("edgePairsSkipped", C.c_uint64),
                ("alignedMarkerPairs", C.c_uint64), ("disjointSetCount", C.c_uint64), ("keptDisjointSetCount", C.c_uint64),
                ("badDisjointSetCount", C.c_uint64), ("vertexCount", C.c_uint64), ("histogramSize", C.c_uint64),
                ("peakDeviceBytes", C.c_uint64), ("deviceMs", C.c_double), ("totalMs", C.c_double), ("kernelLaunches", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def make_marker_graph_params(minCoverage=10, maxCoverage=100, minCoveragePerStrand=0, allowDuplicateMarkers=False,
                             peakFinderMinAreaFraction=0.08, peakFinderAreaStartIndex=2, threadCount=0):
    """Defaults of src/AssemblerOptions.cpp:577-685."""
    return MarkerGraphParams(int(minCoverage), int(maxCoverage), int(minCoveragePerStrand), int(bool(allowDuplicateMarkers)),
                             float(peakFinderMinAreaFraction), int(peakFinderAreaStartIndex), int(threadCount))


def uint40_to_uint64(a):
    """Uint40 little-endian records (uint8[5n]) -> uint64[n]."""
    b = np.asarray(a, np.uint8).reshape(-1, 5)
    out = np.zeros((len(b), 8), np.uint8)
    out[:, :5] = b
    return out.view(np.uint64).reshape(-1)


def uint64_to_uint40(a):
    return np.ascontiguousarray(np.asarray(a, np.uint64).reshape(-1, 1).view(np.uint8)[:, :5]).reshape(-1)


def create_marker_graph_vertices(ctx: Context, params: MarkerGraphParams, edges, compressed_toc, compressed_data, read_flags):
    """Assembler::createMarkerGraphVertices on the markers ctx holds. edges: uint32[E,4] ReadGraphEdge records.
    Returns (vertexTable uint8[5M] (Uint40), verticesToc uint8[5(V+1)] (Uint40), verticesData uint64[], histogram uint64[],
    MarkerGraphResult)."""
    L = lib()
    f = L.shb_create_marker_graph_vertices
    f.argtypes = [C.c_void_p, C.POINTER(MarkerGraphParams), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                  C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                  C.POINTER(MarkerGraphResult)]
    e = np.ascontiguousarray(edges, np.uint32).reshape(-1, 4)
    t = np.ascontiguousarray(compressed_toc, np.uint64)
    d = np.ascontiguousarray(compressed_data, np.uint8)
    fl = np.ascontiguousarray(read_flags, np.uint8)
    table, vtoc, vdata, hist = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    res = MarkerGraphResult()
    _check(f(ctx._h, C.byref(params), _ptr(e), len(e), _ptr(t), _ptr(d), len(t) - 1, _ptr(fl), C.byref(table), C.byref(vtoc),
             C.byref(vdata), C.byref(hist), C.byref(res)))
    V = res.vertexCount
    tocn = _owned_array(vtoc, 5 * (V + 1), np.uint8)
    n = int(uint40_to_uint64(tocn)[-1]) if V else 0
    if not V:
        tocn = np.zeros(5, np.uint8)
    return (_owned_array(table, 5 * res.markerCount, np.uint8), tocn, _owned_array(vdata, n, np.uint64),
            _owned_array(hist, res.histogramSize, np.uint64), res)


def find_marker_graph_reverse_complement_vertices(ctx: Context, vertex_table, vertices_toc, vertices_data):
    """Assembler::findMarkerGraphReverseComplementVertices. vertex_table / vertices_toc: Uint40 bytes. Returns uint64[V]."""
    L = lib()
    f = L.shb_find_marker_graph_reverse_complement_vertices
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
    t = np.ascontiguousarray(vertex_table, np.uint8)
    vt = np.ascontiguousarray(vertices_toc, np.uint8)
    vd = np.ascontiguousarray(vertices_data, np.uint64)
    V = len(vt) // 5 - 1
    rc = C.c_void_p()
    _check(f(ctx._h, _ptr(t), _ptr(vt), _ptr(vd), V, C.byref(rc)))
    return _owned_array(rc, V, np.uint64)


def peak_finder_cutoff(histogram, min_area_fraction=0.08, start_index=2):
    """The library's PeakFinder restatement (host only). Returns (threw, cutoff, observedPercentArea)."""
    L = lib()
    f = L.shb_peak_finder_cutoff
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
    y = np.ascontiguousarray(histogram, np.uint64)
    cutoff, observed = C.c_uint64(0), C.c_double(0)
    threw = f(_ptr(y) if len(y) else None, len(y), float(min_area_fraction), int(start_index), C.byref(cutoff), C.byref(observed))
    return int(threw), int(cutoff.value), float(observed.value)
