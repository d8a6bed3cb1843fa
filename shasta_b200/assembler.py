"""`shasta.Assembler`-shaped host API for the hot path (src/PythonModule.cpp:135-360 of chanzuckerberg/shasta).

The method names, keyword arguments, defaults and `Data/` file names are the reference's, so the reference's driver scripts
for this path (scripts/FindAlignmentCandidatesLowHash0.py, scripts/ComputeAlignments.py) run against this class unchanged:

    a = Assembler()                       # largeDataFileNamePrefix="Data/", createNew=False
    a.accessKmers(); a.accessMarkers()
    a.findAlignmentCandidatesLowHash0(m=4, hashFraction=0.01, minHashIterationCount=10, alignmentCandidatesPerRead=20.,
                                      minBucketSize=5, maxBucketSize=30, minFrequency=5)
    a.accessAlignmentCandidates()
    a.computeAlignments(alignOptions, threadCount=0)

Files are read and written in the reference's `MemoryMapped::Vector` format (4 KiB header {headerSize, objectSize,
objectCount, pageSize, pageCount, fileSize, capacity, magic 0xa3756fd4b5d8bcc1} + raw POD array, page rounded;
src/MemoryMappedVector.hpp:165-231) and `VectorOfVectors` = `name.toc` + `name.data`
(src/MemoryMappedVectorOfVectors.hpp:28-42), so the unmodified reference can continue from the outputs
(tests/test_assembler_files.py opens them with the reference's own MemoryMapped code).

All compute goes through the C ABI (libshasta_b200.so); errors surface as RuntimeError like pybind11's mapping of the
reference's std::runtime_error.
"""
from __future__ import annotations

import os

import numpy as np

MAGIC = 0xa3756fd4b5d8bcc1
HEADER_BYTES = 4096
EDGE_BYTES = 14                 # sizeof(MarkerGraph::Edge) (src/MarkerGraph.hpp:179-244)


def mm_write_vector(path, array, object_size=None, page_size=4096):
    """Write a MemoryMapped::Vector<T> file. `array` is any contiguous numpy array; object_size = sizeof(T)
    (defaults to the array's itemsize)."""
    a = np.ascontiguousarray(array)
    raw = a.view(np.uint8).reshape(-1)
    if object_size is None:
        object_size = a.dtype.itemsize
    assert raw.size % object_size == 0
    n = raw.size // object_size
    page_count = (HEADER_BYTES + raw.size - 1) // page_size + 1 if (HEADER_BYTES + raw.size) > 0 else 1
    file_size = page_count * page_size
    header = np.zeros(HEADER_BYTES // 8, np.uint64)
    header[0] = HEADER_BYTES
    header[1] = object_size
    header[2] = n
    header[3] = page_size
    header[4] = page_count
    header[5] = file_size
    header[6] = (file_size - HEADER_BYTES) // object_size
    header[7] = MAGIC
    with open(path, "wb") as f:
        f.write(header.tobytes())
        f.write(raw.tobytes())
        f.write(b"\0" * (file_size - HEADER_BYTES - raw.size))


def mm_read_vector(path, dtype=np.uint8, object_size=None):
    """Read a MemoryMapped::Vector<T> file; returns a numpy array of `dtype` (memory mapped, read only)."""
    header = np.fromfile(path, dtype=np.uint64, count=8)
    if len(header) < 8 or int(header[7]) != MAGIC or int(header[0]) != HEADER_BYTES:
        raise RuntimeError(f"Error accessing {path}: not a MemoryMapped::Vector file.")
    obj, n = int(header[1]), int(header[2])
    if object_size is not None and obj != object_size:
        raise RuntimeError(f"Unexpected object size {obj} in {path} (expected {object_size}).")
    itemsize = np.dtype(dtype).itemsize
    if (obj * n) % itemsize:
        raise RuntimeError(f"Size of {path} is inconsistent with the requested element type.")
    if n == 0:
        return np.zeros(0, dtype)
    return np.memmap(path, dtype=dtype, mode="r", offset=HEADER_BYTES, shape=(obj * n // itemsize,))


def mm_write_vector_of_vectors(name, toc, data, data_object_size=None, toc_dtype=np.uint64, page_size=4096):
    mm_write_vector(name + ".toc", np.asarray(toc, dtype=toc_dtype), page_size=page_size)
    mm_write_vector(name + ".data", data, object_size=data_object_size, page_size=page_size)


def _ostream_double(x):
    """A double as C++'s `ostream << double` prints it with default flags (precision 6, %g)."""
    return "%g" % x


def write_read_low_hash_statistics_csv(path, stats, marker_toc, read_flags, m):
    """ReadLowHashStatistics.csv as LowHash0 writes it (src/LowHash0.cpp:220-243). stats: uint64[R,3]; marker_toc: the Markers toc
    (2R+1 entries); read_flags: uint8[R] (bit 0 = palindromic)."""
    stats = np.asarray(stats, np.uint64).reshape(-1, 3)
    toc = np.asarray(marker_toc, np.uint64)
    with open(path, "w") as csv:
        csv.write("ReadId,Palindromic,Features,Sparse,Good,Crowded,Total,FeatureSampling,SparseFraction,GoodFraction,CrowdedFraction\n")
        for read_id in range(len(stats)):
            c = [int(v) for v in stats[read_id]]
            # std::accumulate(..., 0): the sum is carried in an int and converted to uint64_t (src/LowHash0.cpp:224)
            total = (sum(c) + 2**31) % 2**32 - 2**31
            total &= 2**64 - 1
            feature_count = (int(toc[2 * read_id + 1]) - int(toc[2 * read_id]) - (m - 1)) & (2**64 - 1)
            sampling = float(total) / float(feature_count) if feature_count else (float("nan") if total == 0 else float("inf"))
            row = [str(read_id), "Yes" if (int(read_flags[read_id]) & 1) else "No", str(feature_count), str(c[0]), str(c[1]), str(c[2]),
                   str(total), _ostream_double(sampling).replace("nan", "-nan" if total == 0 and feature_count == 0 else "nan")]
            if total == 0:
                csv.write(",".join(row) + ",,,\n")
            else:
                csv.write(",".join(row) + "," + ",".join(_ostream_double(float(v) / float(total)) for v in c) + "\n")


class AlignOptions:
    """shasta.AlignOptions (src/PythonModule.cpp:85-107; defaults src/AssemblerOptions.cpp:380-489)."""

    def __init__(self):
        self.alignMethod = 3
        self.maxSkip = 30
        self.maxDrift = 30
        self.maxTrim = 30
        self.maxMarkerFrequency = 10
        self.minAlignedMarkerCount = 100
        self.minAlignedFraction = 0.
        self.matchScore = 6
        self.mismatchScore = -1
        self.gapScore = -1
        self.downsamplingFactor = 0.1
        self.bandExtend = 10
        self.maxBand = 1000
        self.sameChannelReadAlignmentSuppressDeltaThreshold = 0
        self.suppressContainments = False
        self.align4DeltaX = 200
        self.align4DeltaY = 10
        self.align4MinEntryCountPerCell = 10
        self.align4MaxDistanceFromBoundary = 100


class OrientedReadPair:
    """shasta.OrientedReadPair (src/PythonModule.cpp:42-45)."""

    def __init__(self, r0, r1, same):
        self.readIds = [int(r0), int(r1)]
        self.isSameStrand = bool(same)


class Assembler:
    def __init__(self, largeDataFileNamePrefix="Data/", createNew=False, readRepresentation=1,
                 largeDataPageSize=2 * 1024 * 1024, device=0):
        self.prefix = largeDataFileNamePrefix
        self.page_size = 4096          # files are written with 4 KiB pages (valid for any filesystem)
        self.device = device
        if createNew and self.prefix and os.path.dirname(self.prefix):
            os.makedirs(os.path.dirname(self.prefix), exist_ok=True)
        self._ctx = None
        self.k = None
        self._markers = None
        self._candidates = None
        self._alignment_data = None
        self._compressed = None

    # ------------------------------------------------------------------ helpers
    def _name(self, n):
        if not self.prefix:
            raise RuntimeError("Anonymous memory mode is not supported by this facade: give a Data/ prefix.")
        return self.prefix + n

    def _context(self):
        if self._ctx is None:
            from . import capi
            self._ctx = capi.Context(self.device)
            self._markers_on_device = False
        return self._ctx

    def _upload_markers(self):
        self.checkMarkersAreOpen()
        ctx = self._context()
        if not self._markers_on_device:
            toc, data, flags = self._markers
            ctx.set_markers(toc, data, flags)
            self._markers_on_device = True
        return ctx

    # ------------------------------------------------------------------ access functions (reference names)
    def accessKmers(self):
        """Data/Kmers: Vector<KmerInfo>, 24 bytes each, 4^k entries (src/AssemblerKmers.cpp:15-21). Only k is needed here:
        the method-3 downsampling hash is recomputed on the device."""
        kmers = mm_read_vector(self._name("Kmers"), np.uint8, object_size=24)
        count = len(kmers) // 24
        k = (count.bit_length() - 1) // 2
        if count != 1 << (2 * k):
            raise RuntimeError("Size of k-mer vector is inconsistent with stored value of k.")
        self.k = k

    def checkKmersAreOpen(self):
        if self.k is None:
            raise RuntimeError("Kmers are not accessible.")

    def accessMarkers(self):
        toc = mm_read_vector(self._name("Markers.toc"), np.uint64, object_size=8)
        data = mm_read_vector(self._name("Markers.data"), np.uint8, object_size=7)
        flags = mm_read_vector(self._name("ReadFlags"), np.uint8, object_size=1)
        if len(toc) != 2 * len(flags) + 1:
            raise RuntimeError("Markers and ReadFlags are inconsistent.")
        self._markers = (np.asarray(toc), np.asarray(data), np.asarray(flags))
        self._markers_on_device = False

    def checkMarkersAreOpen(self):
        if self._markers is None:
            raise RuntimeError("Markers are not accessible.")

    def accessAlignmentCandidates(self):
        c = mm_read_vector(self._name("AlignmentCandidates"), np.uint32, object_size=12)
        self._candidates = np.asarray(c).reshape(-1, 3).copy()
        self._candidates[:, 2] &= 0xff

    def checkAlignmentCandidatesAreOpen(self):
        if self._candidates is None:
            raise RuntimeError("Alignment candidates are not accessible.")

    def getAlignmentCandidates(self):
        self.checkAlignmentCandidatesAreOpen()
        return [OrientedReadPair(r0, r1, s) for r0, r1, s in self._candidates.tolist()]

    def accessAlignmentData(self):
        self._alignment_data = np.asarray(mm_read_vector(self._name("AlignmentData"), np.uint32, object_size=64)).reshape(-1, 16)

    def accessCompressedAlignments(self):
        toc = mm_read_vector(self._name("CompressedAlignments.toc"), np.uint64, object_size=8)
        data = mm_read_vector(self._name("CompressedAlignments.data"), np.uint8, object_size=1)
        self._compressed = (np.asarray(toc), np.asarray(data))

    def computeSortedMarkers(self, threadCount=0):
        """Assembler::computeSortedMarkers (src/AssemblerAlign4.cpp:190-261, binding src/PythonModule.cpp:210-212).
        Kept for script compatibility (scripts/ComputeSortedMarkers.py): the markers sorted by k-mer id that Align4 needs are
        derived on the device from the resident k-mer ids the first time an alignment method 4 call needs them and cached per
        marker set (csrc/align.cu buildSortedMarkers), so there is no Data/SortedMarkers file to write."""
        self.checkMarkersAreOpen()

    def accessSortedMarkers(self):
        """Assembler::accessSortedMarkers (src/PythonModule.cpp:213-214): nothing to open, see computeSortedMarkers."""
        self.checkMarkersAreOpen()

    def flagPalindromicReads(self, maxSkip, maxDrift, maxMarkerFrequency, alignedFractionThreshold,
                             nearDiagonalFractionThreshold, deltaThreshold, threadCount=0):
        """Assembler::flagPalindromicReads (src/AssemblerAlign.cpp:652-770, binding src/PythonModule.cpp:251-259) on the
        device: bit 0 of every read's flags is reset, then set on the reads whose alignment with their own reverse
        complement passes both thresholds. Data/ReadFlags is rewritten; the markers stay on the device, with the new flags,
        for the LowHash0 and alignment calls that follow. threadCount is accepted and ignored."""
        from . import capi
        ctx = self._upload_markers()
        toc, data, flags = self._markers
        flags = np.array(flags, dtype=np.uint8)
        params = capi.make_palindromic_params(maxSkip=maxSkip, maxDrift=maxDrift, maxMarkerFrequency=maxMarkerFrequency,
                                              alignedFractionThreshold=alignedFractionThreshold,
                                              nearDiagonalFractionThreshold=nearDiagonalFractionThreshold,
                                              deltaThreshold=deltaThreshold, threadCount=threadCount)
        _, _, res = capi.flag_palindromic_reads(ctx, params, read_flags=flags, want_counts=False)
        mm_write_vector(self._name("ReadFlags"), flags, object_size=1)
        self._markers = (toc, data, flags)
        readCount = len(flags)
        print(f"Flagged {res.palindromicReadCount} reads as palindromic out of {readCount} total.")
        print(f"Palindromic fraction is {_ostream_double(res.palindromicReadCount / readCount if readCount else float('nan'))}")

    def alignOrientedReads4(self, readId0, strand0, readId1, strand1, deltaX, deltaY, minEntryCountPerCell,
                            maxDistanceFromBoundary, minAlignedMarkerCount, minAlignedFraction, maxSkip, maxDrift, maxTrim,
                            maxBand, matchScore, mismatchScore, gapScore):
        """Single-pair Align4 (src/AssemblerAlign4.cpp:13-61, binding src/PythonModule.cpp:302-327; scripts/AlignOrientedReads4.py).
        Prints the reference's line and returns the number of aligned markers. The two oriented reads are aligned in exactly
        the orientation and order given (shb_align_oriented_reads): read 0 is the horizontal sequence of the cell grid and of
        the DP, as in the reference. matchScore / mismatchScore / gapScore are accepted for signature compatibility: Align4
        hard-codes 6 / -1 / -1 (src/Align4.hpp:159-161)."""
        from . import capi
        self.checkKmersAreOpen()
        ctx = self._upload_markers()
        o = capi.make_align_options(alignMethod=4, k=int(self.k), maxSkip=int(maxSkip), maxDrift=int(maxDrift), maxTrim=int(maxTrim),
                                    minAlignedMarkerCount=int(minAlignedMarkerCount), minAlignedFraction=float(minAlignedFraction),
                                    maxBand=int(maxBand), matchScore=int(matchScore), mismatchScore=int(mismatchScore),
                                    gapScore=int(gapScore), suppressContainments=0, align4DeltaX=int(deltaX), align4DeltaY=int(deltaY),
                                    align4MinEntryCountPerCell=int(minEntryCountPerCell),
                                    align4MaxDistanceFromBoundary=int(maxDistanceFromBoundary))
        try:
            ords, _ = capi.align_oriented_reads(ctx, 2 * int(readId0) + int(strand0), 2 * int(readId1) + int(strand1), o)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self._last_alignment = ords
        print(f"The alignment has {len(ords)} markers.")
        return len(ords)

    def computeCandidateTable(self):
        """Assembler::computeCandidateTable (src/AssemblerAlignmentCandidates.cpp:379-448, called at srcMain/main.cpp:706).
        Writes Data/CandidateTable.{toc,data} (VectorOfVectors<uint64_t,uint64_t>)."""
        from . import capi
        self.checkAlignmentCandidatesAreOpen()
        self.checkMarkersAreOpen()
        try:
            toc, table = capi.compute_candidate_table(self._context(), self._candidates, len(self._markers[2]))
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self._candidate_table = (toc, table)
        mm_write_vector_of_vectors(self._name("CandidateTable"), toc, table, data_object_size=8, toc_dtype=np.uint64,
                                   page_size=self.page_size)

    def createReadGraph(self, maxAlignmentCount, maxTrim=0):
        """Assembler::createReadGraph (src/AssemblerReadGraph.cpp:35-175; ReadGraph.creationMethod 0; maxTrim is unused there
        too). Sets AlignmentInfo::isInReadGraph in Data/AlignmentData and writes Data/ReadGraphEdges (16-byte ReadGraphEdge) and
        Data/ReadGraphConnectivity.{toc,data} (VectorOfVectors<uint32_t,uint32_t>)."""
        from . import capi
        self.checkMarkersAreOpen()
        if self._alignment_data is None:
            raise RuntimeError("Alignment data are not accessible.")
        rec = np.ascontiguousarray(np.array(self._alignment_data, np.uint32)).reshape(-1, 16)
        try:
            keep, edges, toc, data = capi.create_read_graph(self._context(), rec, len(self._markers[2]), maxAlignmentCount)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self._alignment_data = rec
        self._read_graph = (np.array(edges), np.array(toc), np.array(data))
        mm_write_vector(self._name("AlignmentData"), rec, object_size=64, page_size=self.page_size)
        mm_write_vector(self._name("ReadGraphEdges"), np.array(edges), object_size=16, page_size=self.page_size)
        mm_write_vector_of_vectors(self._name("ReadGraphConnectivity"), np.array(toc), np.array(data), data_object_size=4,
                                   toc_dtype=np.uint32, page_size=self.page_size)
        return int(keep.sum())

    def createReadGraph2(self, maxAlignmentCount, markerCountPercentile, alignedFractionPercentile, maxSkipPercentile,
                         maxDriftPercentile, maxTrimPercentile):
        """Assembler::createReadGraph2 (src/AssemblerReadGraph2.cpp:182-248, Python src/PythonModule.cpp:366-367;
        ReadGraph.creationMethod 2). Same outputs as createReadGraph; the automatically selected criteria are kept in
        self.readGraph2Criteria and printed like the reference does (:155-160)."""
        from . import capi
        self.checkMarkersAreOpen()
        if self._alignment_data is None:
            raise RuntimeError("Alignment data are not accessible.")
        rec = np.ascontiguousarray(np.array(self._alignment_data, np.uint32)).reshape(-1, 16)
        try:
            crit, keep, edges, toc, data = capi.create_read_graph2(self._context(), rec, len(self._markers[2]), maxAlignmentCount,
                                                                  markerCountPercentile, alignedFractionPercentile, maxSkipPercentile,
                                                                  maxDriftPercentile, maxTrimPercentile)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self.readGraph2Criteria = crit
        print("Automatically selected alignment criteria:\n\tminAlignedFraction:\t%g\n\tminAlignedMarkerCount:\t\t%d\n\tmaxDrift:\t\t%d\n"
              "\tmaxSkip:\t\t%d\n\tmaxTrim:\t\t%d" % (crit["minAlignedFraction"], crit["minAlignedMarkerCount"], crit["maxDrift"],
                                                   crit["maxSkip"], crit["maxTrim"]))
        print("Keeping %d alignments of %d" % (int(keep.sum()), len(rec)))
        self._alignment_data = rec
        self._read_graph = (np.array(edges), np.array(toc), np.array(data))
        mm_write_vector(self._name("AlignmentData"), rec, object_size=64, page_size=self.page_size)
        mm_write_vector(self._name("ReadGraphEdges"), np.array(edges), object_size=16, page_size=self.page_size)
        mm_write_vector_of_vectors(self._name("ReadGraphConnectivity"), np.array(toc), np.array(data), data_object_size=4,
                                   toc_dtype=np.uint32, page_size=self.page_size)
        return int(keep.sum())

    def _read_graph_for_flags(self):
        """(edges, toc, data, alignment records) of this session's read graph, else of Data/ (writable copies)."""
        if getattr(self, "_read_graph", None) is not None:
            edges, toc, data = self._read_graph
        else:
            edges = mm_read_vector(self._name("ReadGraphEdges"), np.uint32, object_size=16)
            toc = mm_read_vector(self._name("ReadGraphConnectivity.toc"), np.uint32)
            data = mm_read_vector(self._name("ReadGraphConnectivity.data"), np.uint32, object_size=4)
        if self._alignment_data is None:
            raise RuntimeError("Alignment data are not accessible.")
        rec = np.ascontiguousarray(np.array(self._alignment_data, np.uint32)).reshape(-1, 16)
        return np.array(edges, np.uint32).reshape(-1, 4), np.asarray(toc, np.uint32), np.asarray(data, np.uint32), rec

    def _store_read_graph_flags(self, edges, toc, data, rec):
        self._alignment_data = rec
        self._read_graph = (edges, toc, data)
        self._read_graph_edges = edges
        mm_write_vector(self._name("AlignmentData"), rec, object_size=64, page_size=self.page_size)
        mm_write_vector(self._name("ReadGraphEdges"), edges, object_size=16, page_size=self.page_size)

    def flagCrossStrandReadGraphEdges1(self, maxDistance, threadCount=0):
        """Assembler::flagCrossStrandReadGraphEdges1 (src/AssemblerReadGraph.cpp:775-1041, binding src/PythonModule.cpp:388-393;
        ReadGraph.strandSeparationMethod 1) on the device. Rewrites crossesStrands in Data/ReadGraphEdges and clears
        AlignmentInfo::isInReadGraph in Data/AlignmentData for the edges it flags; the session's read graph is updated, so a
        following createMarkerGraphVertices sees the flags. Prints the reference's lines. threadCount is ignored."""
        from . import capi
        edges, toc, data, rec = self._read_graph_for_flags()
        try:
            res = capi.flag_cross_strand_read_graph_edges1(self._context(), maxDistance, edges, toc, data, rec)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self._store_read_graph_flags(edges, toc, data, rec)
        self.crossStrandResult = res
        if maxDistance == 0:
            print("Skipped flagCrossStrandReadGraphEdges.")
            return
        print(f"Of {len(toc) - 1} vertices in the read graph, {res['nearStrandJumpReportedCount']} are within distance "
              f"{maxDistance} of their reverse complement.")
        print(f"Found {res['regionCount']} strand jump regions.")
        print(f"Marked {res['crossStrandEdgeCount']} read graph edges out of {len(edges)} total as cross-strand.")

    def flagChimericReads(self, maxChimericReadDistance, threadCount=0):
        """Assembler::flagChimericReads (src/AssemblerReadGraph.cpp:355-583, binding src/PythonModule.cpp:394-397) on the
        device. Rewrites the isChimeric bit of Data/ReadFlags and clears AlignmentInfo::isInReadGraph in Data/AlignmentData for
        every alignment of a chimeric read. Prints the reference's lines. threadCount is ignored."""
        from . import capi
        edges, toc, data, rec = self._read_graph_for_flags()
        if self._markers is not None:
            flags = np.array(self._markers[2], np.uint8)
        else:
            flags = np.array(mm_read_vector(self._name("ReadFlags"), np.uint8, object_size=1), np.uint8)
        try:
            res = capi.flag_chimeric_reads(self._context(), maxChimericReadDistance, edges, toc, data, flags, rec)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        self._store_read_graph_flags(edges, toc, data, rec)
        mm_write_vector(self._name("ReadFlags"), flags, object_size=1)
        if self._markers is not None:
            self._markers = (self._markers[0], self._markers[1], flags)
        self.chimericResult = res
        if maxChimericReadDistance == 0:
            return
        readCount = len(flags)
        print(f"Flagged {res['chimericReadCount']} reads as chimeric out of {readCount} total.")
        print(f"Chimera rate is {_ostream_double(res['chimericReadCount'] / readCount if readCount else float('nan'))}")

    # ------------------------------------------------------------------ the two hot-path entry points
    def findAlignmentCandidatesLowHash0(self, m, hashFraction, minHashIterationCount, alignmentCandidatesPerRead,
                                        minBucketSize, maxBucketSize, minFrequency, log2MinHashBucketCount=0, threadCount=0):
        """Assembler::findAlignmentCandidatesLowHash0 (src/AssemblerLowHash.cpp:10-55). Writes Data/AlignmentCandidates and
        Data/ReadLowHashStatistics."""
        from . import capi
        self.checkKmersAreOpen()
        ctx = self._upload_markers()
        p = capi.make_lowhash_params(m=m, hashFraction=hashFraction, minHashIterationCount=minHashIterationCount,
                                     alignmentCandidatesPerRead=alignmentCandidatesPerRead,
                                     log2MinHashBucketCount=log2MinHashBucketCount, minBucketSize=minBucketSize,
                                     maxBucketSize=maxBucketSize, minFrequency=minFrequency, threadCount=threadCount)
        try:
            cand, stats, _, res = ctx.lowhash0(p, want_stats=True)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        print(f"LowHash0 algorithm will use 2^{res.log2BucketCount} = {1 << res.log2BucketCount} buckets. ")
        print(f"Found {len(cand)} alignment candidates.")
        rows = 2 * len(self._markers[2])
        print(f"Average number of alignment candidates per oriented read is {2. * len(cand) / max(rows, 1)}.")
        self._candidates = cand
        rec = cand.copy()          # 12-byte OrientedReadPair records: third word = isSameStrand byte + zero padding
        mm_write_vector(self._name("AlignmentCandidates"), rec, object_size=12, page_size=self.page_size)
        mm_write_vector(self._name("ReadLowHashStatistics"), stats, object_size=24, page_size=self.page_size)
        # the reference also leaves ReadLowHashStatistics.csv in the working directory (src/LowHash0.cpp:220-243)
        write_read_low_hash_statistics_csv("ReadLowHashStatistics.csv", stats, self._markers[0], self._markers[2], m)

    def computeAlignments(self, alignOptions, threadCount=0):
        """Assembler::computeAlignments (src/AssemblerAlign.cpp:208-304). Writes Data/AlignmentData,
        Data/CompressedAlignments.{toc,data} and Data/AlignmentTable.{toc,data}."""
        from . import capi
        self.checkKmersAreOpen()
        self.checkAlignmentCandidatesAreOpen()
        ctx = self._upload_markers()
        o = capi.make_align_options(
            alignMethod=int(alignOptions.alignMethod), maxSkip=int(alignOptions.maxSkip), maxDrift=int(alignOptions.maxDrift),
            maxTrim=int(alignOptions.maxTrim), maxMarkerFrequency=int(alignOptions.maxMarkerFrequency),
            minAlignedMarkerCount=int(alignOptions.minAlignedMarkerCount), minAlignedFraction=float(alignOptions.minAlignedFraction),
            matchScore=int(alignOptions.matchScore), mismatchScore=int(alignOptions.mismatchScore), gapScore=int(alignOptions.gapScore),
            downsamplingFactor=float(alignOptions.downsamplingFactor), bandExtend=int(alignOptions.bandExtend),
            maxBand=int(alignOptions.maxBand),
            sameChannelReadAlignmentSuppressDeltaThreshold=int(alignOptions.sameChannelReadAlignmentSuppressDeltaThreshold),
            suppressContainments=int(bool(alignOptions.suppressContainments)), align4DeltaX=int(alignOptions.align4DeltaX),
            align4DeltaY=int(alignOptions.align4DeltaY), align4MinEntryCountPerCell=int(alignOptions.align4MinEntryCountPerCell),
            align4MaxDistanceFromBoundary=int(alignOptions.align4MaxDistanceFromBoundary), k=int(self.k))
        try:
            rec, ctoc, cdata, res = capi.compute_alignments(ctx, self._candidates, o)
            ttoc, tdata = capi.compute_alignment_table(ctx, rec, len(self._markers[2]))
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        print(f"Found and stored {len(rec)} good alignments.")
        self._alignment_data = rec
        self._compressed = (ctoc, cdata)
        mm_write_vector(self._name("AlignmentData"), rec, object_size=64, page_size=self.page_size)
        mm_write_vector_of_vectors(self._name("CompressedAlignments"), ctoc, cdata, data_object_size=1, page_size=self.page_size)
        mm_write_vector_of_vectors(self._name("AlignmentTable"), ttoc, tdata, data_object_size=4, toc_dtype=np.uint32,
                                   page_size=self.page_size)

    # ------------------------------------------------------------------ marker graph vertices
    def accessReadGraph(self):
        """Data/ReadGraphEdges: 16-byte ReadGraphEdge records (src/ReadGraph.hpp:37-57)."""
        self._read_graph_edges = np.asarray(mm_read_vector(self._name("ReadGraphEdges"), np.uint32, object_size=16)).reshape(-1, 4)

    def createMarkerGraphVertices(self, minCoverage, maxCoverage, minCoveragePerStrand, allowDuplicateMarkers,
                                  peakFinderMinAreaFraction, peakFinderAreaStartIndex, threadCount=0):
        """Assembler::createMarkerGraphVertices (src/AssemblerMarkerGraph.cpp:38-518, binding src/PythonModule.cpp:428-436).
        Writes Data/MarkerGraphVertexTable (Uint40 per marker), Data/MarkerGraphVertices.{toc,data} (VectorOfVectors<MarkerId,
        Uint40>) and DisjointSetsHistogram.csv, and prints the reference's lines. Vertices are numbered in increasing order of
        their first marker. Data/ReadFlags is read now: flagChimericReads may have changed it. threadCount is ignored."""
        from . import capi
        self.checkMarkersAreOpen()
        edges = getattr(self, "_read_graph_edges", None)
        if edges is None and getattr(self, "_read_graph", None) is not None:
            edges = self._read_graph[0]                 # created in this session by createReadGraph / createReadGraph2
        if edges is None:
            raise RuntimeError("Read graph is not accessible.")
        if self._compressed is None:
            raise RuntimeError("Compressed alignments are not accessible.")
        ctx = self._upload_markers()
        flags = np.asarray(mm_read_vector(self._name("ReadFlags"), np.uint8, object_size=1))
        params = capi.make_marker_graph_params(minCoverage, maxCoverage, minCoveragePerStrand, allowDuplicateMarkers,
                                               peakFinderMinAreaFraction, peakFinderAreaStartIndex, threadCount)
        try:
            table, vtoc, vdata, hist, res = capi.create_marker_graph_vertices(ctx, params, edges, self._compressed[0],
                                                                              self._compressed[1], flags)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        write_disjoint_sets_histogram_csv("DisjointSetsHistogram.csv", hist)
        if minCoverage == 0:
            if res.peakFinderFailed:
                print("Unable to automatically select MarkerGraph.minCoverage. No significant cutoff found in disjoint sets size "
                      f"distribution. Observed peak has percent total area of {_ostream_double(res.peakFinderObservedAreaFraction)}\n"
                      f"minPercentArea is {_ostream_double(peakFinderMinAreaFraction)}\n"
                      f"See DisjointSetsHistogram.csv.Using MarkerGraph.minCoverage = {res.minCoverageUsed}")
            else:
                print(f"Automatically selected value of MarkerGraph.minCoverage is {res.minCoverageUsed}")
        print(f"Kept {res.keptDisjointSetCount} disjoint sets with coverage in the requested range.")
        print(f"Found {res.badDisjointSetCount} disjoint sets with more than one marker on a single oriented read or with less than "
              f"{minCoveragePerStrand} supporting oriented reads on each strand.")
        self.markerGraphMinCoverageUsed = res.minCoverageUsed
        self._marker_graph = (table, vtoc, vdata)
        mm_write_vector(self._name("MarkerGraphVertexTable"), table, object_size=5, page_size=self.page_size)
        mm_write_vector(self._name("MarkerGraphVertices.toc"), vtoc, object_size=5, page_size=self.page_size)
        mm_write_vector(self._name("MarkerGraphVertices.data"), vdata, object_size=8, page_size=self.page_size)

    def accessMarkerGraphVertices(self, readWriteAccess=False):
        """Data/MarkerGraphVertexTable and Data/MarkerGraphVertices.{toc,data} (src/AssemblerMarkerGraph.cpp)."""
        table = mm_read_vector(self._name("MarkerGraphVertexTable"), np.uint8, object_size=5)
        vtoc = mm_read_vector(self._name("MarkerGraphVertices.toc"), np.uint8, object_size=5)
        vdata = mm_read_vector(self._name("MarkerGraphVertices.data"), np.uint64, object_size=8)
        self._marker_graph = (np.asarray(table), np.asarray(vtoc), np.asarray(vdata))

    def findMarkerGraphReverseComplementVertices(self, threadCount=0):
        """Assembler::findMarkerGraphReverseComplementVertices (:1134-1230). Writes Data/MarkerGraphReverseComplementeVertex
        (the reference's file name), uint64 per vertex. Works on vertices in any numbering, the reference's included."""
        from . import capi
        if getattr(self, "_marker_graph", None) is None:
            raise RuntimeError("Marker graph vertices are not accessible.")
        ctx = self._upload_markers()
        table, vtoc, vdata = self._marker_graph
        try:
            rc = capi.find_marker_graph_reverse_complement_vertices(ctx, table, vtoc, vdata)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        mm_write_vector(self._name("MarkerGraphReverseComplementeVertex"), rc, object_size=8, page_size=self.page_size)

    # ------------------------------------------------------------------ marker graph edges
    def createMarkerGraphEdges(self, threadCount=0):
        """Assembler::createMarkerGraphEdges (src/AssemblerMarkerGraph.cpp:2028-2213) on Data/MarkerGraphVertexTable and
        Data/MarkerGraphVertices.{toc,data}. Writes Data/GlobalMarkerGraphEdges (14-byte Edge records),
        Data/GlobalMarkerGraphEdgeMarkerIntervals.{toc,data} (VectorOfVectors<MarkerInterval, uint64_t>) and
        Data/GlobalMarkerGraphEdgesBySource / ...ByTarget.{toc,data} (VectorOfVectors<Uint40, uint64_t>), as the reference
        run with one thread writes them, and prints the reference's line. threadCount is ignored."""
        from . import capi
        self.checkMarkersAreOpen()
        self.accessMarkerGraphVertices()
        table, vtoc, vdata = self._marker_graph
        ctx = self._upload_markers()
        try:
            out, res = capi.create_marker_graph_edges(ctx, table, vtoc, vdata)
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        print(f"Found {res.edgeCount} edges for {res.vertexCount} vertices.")
        self._write_marker_graph_edges(out)
        self._marker_graph_edges = out

    def _write_marker_graph_edges(self, out):
        ps = self.page_size
        mm_write_vector(self._name("GlobalMarkerGraphEdges"), out["edges"], object_size=EDGE_BYTES, page_size=ps)
        mm_write_vector_of_vectors(self._name("GlobalMarkerGraphEdgeMarkerIntervals"), out["intervalsToc"], out["intervalsData"],
                                   data_object_size=12, page_size=ps)
        for name, key in (("GlobalMarkerGraphEdgesBySource", "bySource"), ("GlobalMarkerGraphEdgesByTarget", "byTarget")):
            mm_write_vector_of_vectors(self._name(name), out[key + "Toc"], out[key + "Data"], data_object_size=5, page_size=ps)

    def accessMarkerGraphEdges(self, accessEdgesReadWrite=False, accessConnectivityReadWrite=False):
        """The five edge file sets createMarkerGraphEdges writes (read only here: the flags say how the reference maps them)."""
        itoc = mm_read_vector(self._name("GlobalMarkerGraphEdgeMarkerIntervals.toc"), np.uint64, object_size=8)
        self._marker_graph_edges = dict(
            edges=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdges"), np.uint8, object_size=EDGE_BYTES)).reshape(-1, 14),
            intervalsToc=np.asarray(itoc),
            intervalsData=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdgeMarkerIntervals.data"), np.uint32,
                                                    object_size=12)).reshape(-1, 3),
            bySourceToc=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdgesBySource.toc"), np.uint64, object_size=8)),
            bySourceData=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdgesBySource.data"), np.uint8, object_size=5)),
            byTargetToc=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdgesByTarget.toc"), np.uint64, object_size=8)),
            byTargetData=np.asarray(mm_read_vector(self._name("GlobalMarkerGraphEdgesByTarget.data"), np.uint8, object_size=5)))

    def findMarkerGraphReverseComplementEdges(self, threadCount=0):
        """Assembler::findMarkerGraphReverseComplementEdges (:1244-1389) on the edges of this session or of accessMarkerGraphEdges
        and on Data/MarkerGraphReverseComplementeVertex. Writes Data/MarkerGraphReverseComplementeEdge (the reference's file
        name), uint64 per edge. Works on edges in any numbering, parallel edges included. threadCount is ignored."""
        from . import capi
        edges = getattr(self, "_marker_graph_edges", None)
        if edges is None:
            raise RuntimeError("Marker graph edges are not accessible.")
        rc_vertex = mm_read_vector(self._name("MarkerGraphReverseComplementeVertex"), np.uint64, object_size=8)
        ctx = self._upload_markers()
        try:
            rc, _ = capi.find_marker_graph_reverse_complement_edges(ctx, rc_vertex, edges["edges"], edges["intervalsToc"],
                                                                    edges["intervalsData"], edges["bySourceToc"], edges["bySourceData"])
        except capi.ShastaB200Error as e:
            raise RuntimeError(str(e)) from None
        mm_write_vector(self._name("MarkerGraphReverseComplementeEdge"), rc, object_size=8, page_size=self.page_size)
        self._marker_graph_rc_edge = rc

    def accessMarkerGraphReverseComplementEdge(self):
        """Data/MarkerGraphReverseComplementeEdge: uint64 per edge."""
        self._marker_graph_rc_edge = np.asarray(mm_read_vector(self._name("MarkerGraphReverseComplementeEdge"), np.uint64, object_size=8))


def write_disjoint_sets_histogram_csv(path, histogram):
    """DisjointSetsHistogram.csv as createMarkerGraphVertices writes it (src/AssemblerMarkerGraph.cpp:224-231): nonzero rows."""
    with open(path, "w") as csv:
        csv.write("Coverage,Frequency\n")
        for coverage, frequency in enumerate(np.asarray(histogram, np.uint64).tolist()):
            if frequency:
                csv.write(f"{coverage},{frequency}\n")
