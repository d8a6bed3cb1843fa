// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// Glue that exposes the *unmodified* reference implementation of the LowHash0
// half of the hot path through a small extern "C" surface, so that tests here
// and bench.py --impl reference can run the real reference code.
//
// This TU is compiled together with reference translation units taken from
// /root/reference/src where they lie (see oracle/Makefile, target ref); no
// reference source is copied into this repository. Output: oracle/_ref/libshasta_ref.so
//
// Reference entry points driven from here:
//   ReadLoader            src/ReadLoader.hpp:28-36     (FASTA -> RLE reads)
//   MarkerFinder          src/MarkerFinder.hpp:26-31   (reads -> CompressedMarker rows)
//   LowHash0::LowHash0    src/LowHash0.cpp:23-257      (markers -> candidates + per-read stats)
// The k-mer table construction below restates Assembler::initializeKmerTable /
// randomlySelectKmers (src/AssemblerKmers.cpp:33-185) because the Assembler class
// itself cannot be linked here (it drags boost-dependent TUs).

#include <sstream>
#include <filesystem>
#include <iostream>
#include <fstream>
#include <chrono>
#include "LongBaseSequence.hpp"
#include "MemoryMappedVectorOfVectors.hpp"
#include "MemoryMappedObject.hpp"
#include "MultithreadedObject.hpp"
#include "ReadFlags.hpp"
#include "ReadId.hpp"
#include "Base.hpp"
#include "span.hpp"
#define private public      // test-only: lets the glue fill Reads::readFlags for marker-space inputs
#include "Reads.hpp"
#undef private
#include "ReadLoader.hpp"
#include "MarkerFinder.hpp"
#include "LowHash0.hpp"
#include "MurmurHash2.hpp"
#include "Kmer.hpp"
#include "Marker.hpp"
#include "OrientedReadPair.hpp"
#include "timestamp.hpp"

#include <random>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <unistd.h>

using namespace shasta;

// The real src/timestamp.cpp needs boost::date_time, absent here.
std::ostream& shasta::timestamp(std::ostream& s) { return s; }

namespace {

// src/AssemblerKmers.cpp:139-185 (initializeKmerTable) + :33-100 (randomlySelectKmers).
void buildKmerTable(MemoryMapped::Vector<KmerInfo>& kmerTable, size_t k, double probability, int seed)
{
    const size_t kmerCount = 1ULL << (2ULL*k);
    kmerTable.createNew("", 4096);
    kmerTable.resize(kmerCount);
    for(uint64_t kmerId=0; kmerId<kmerCount; kmerId++) {
        const Kmer kmer(kmerId, k);
        kmerTable[kmerId].frequency = 0;
        kmerTable[kmerId].isMarker = false;
        kmerTable[kmerId].reverseComplementedKmerId = KmerId(kmer.reverseComplement(k).id(k));
        bool isRle = true;
        for(size_t i=1; i<k; i++) {
            if(kmer[i-1] == kmer[i]) { isRle = false; break; }
        }
        kmerTable[kmerId].isRleKmer = isRle;
    }
    for(uint64_t kmerId=0; kmerId<kmerCount; kmerId++) {
        const uint64_t n = kmerId + kmerTable[kmerId].reverseComplementedKmerId;
        kmerTable[kmerId].hash = MurmurHash2(&n, sizeof(n), 13477);
    }
    const double p = 1. - std::sqrt(1. - probability);
    std::mt19937 randomSource(seed);
    std::uniform_real_distribution<> uniformDistribution;
    for(uint64_t kmerId=0; kmerId<kmerCount; kmerId++) {
        const double x = uniformDistribution(randomSource);
        if(x <= p) {
            kmerTable[kmerId].isMarker = true;
            kmerTable[kmerTable[kmerId].reverseComplementedKmerId].isMarker = true;
        }
    }
}

// Captures everything the reference writes to cout (its per-iteration summary lines are a
// parity signal, src/LowHash0.cpp:193-196); echoes it afterwards unless quiet.
struct QuietCout {
    std::streambuf* old;
    std::ostringstream sink;
    bool quiet;
    QuietCout(bool quiet) : old(std::cout.rdbuf(sink.rdbuf())), quiet(quiet) {}
    ~QuietCout() { std::cout.rdbuf(old); if(!quiet) std::cout << sink.str(); }
};

} // namespace


extern "C" {

// FASTA -> markers through the reference's own ReadLoader + MarkerFinder.
// Outputs are malloc'ed; caller frees with ref_free.
// Returns 0 on success.
int ref_markers_from_fasta(
    const char* fastaPath, uint64_t k, double markerProbability, int seed,
    uint64_t minReadLength, uint64_t threadCount,
    uint64_t* readCountOut, uint64_t** tocOut, uint8_t** dataOut, uint8_t** flagsOut,
    uint32_t** kmerHashOut /* may be null: receives kmerTable[].hash, 4^k entries */)
{
    try {
        QuietCout quiet(true);
        Reads reads;
        reads.createNew(1, "", "", "", "", "", "", 4096);
        {
            ReadLoader loader(fastaPath, 1, minReadLength, false, threadCount, "", 4096, reads);
        }
        MemoryMapped::Vector<KmerInfo> kmerTable;
        buildKmerTable(kmerTable, k, markerProbability, seed);
        MemoryMapped::VectorOfVectors<CompressedMarker, uint64_t> markers;
        markers.createNew("", 4096);
        {
            MarkerFinder finder(k, kmerTable, reads, markers, threadCount);
        }
        const uint64_t R = reads.readCount();
        *readCountOut = R;
        uint64_t* toc = (uint64_t*)malloc(sizeof(uint64_t)*(2*R+1));
        uint64_t total = 0;
        for(uint64_t i=0; i<2*R; i++) { toc[i] = total; total += markers.size(i); }
        toc[2*R] = total;
        uint8_t* data = (uint8_t*)malloc(total*7 + 8);
        for(uint64_t i=0; i<2*R; i++) {
            memcpy(data + 7*toc[i], markers.begin(i), 7*markers.size(i));
        }
        uint8_t* flags = (uint8_t*)malloc(R ? R : 1);
        for(uint64_t r=0; r<R; r++) {
            flags[r] = *reinterpret_cast<const uint8_t*>(&reads.getFlags(ReadId(r)));
        }
        *tocOut = toc; *dataOut = data; *flagsOut = flags;
        if(kmerHashOut) {
            const uint64_t n = 1ULL << (2*k);
            uint32_t* h = (uint32_t*)malloc(sizeof(uint32_t)*n);
            for(uint64_t i=0; i<n; i++) h[i] = kmerTable[i].hash;
            *kmerHashOut = h;
        }
        markers.remove();
        kmerTable.remove();
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_markers_from_fasta: %s\n", e.what());
        return 1;
    }
}


// FASTA -> the INPUTS of the reference's MarkerFinder, as the reference itself stores them: the run-length encoded reads
// in LongBaseSequences layout (src/LongBaseSequence.hpp:33-41: per read two uint64 words per 64 bases, low bit plane then
// high bit plane, base 0 in the most significant bit), their base counts, and kmerTable[].isMarker (one byte per k-mer).
// Used to generate the golden fixture of the device MarkerFinder (tests/golden/make_marker_golden.py).
int ref_reads_from_fasta(
    const char* fastaPath, uint64_t k, double markerProbability, int seed,
    uint64_t minReadLength, uint64_t threadCount,
    uint64_t* readCountOut, uint64_t** wordOffsetsOut /* R+1 */, uint64_t** wordsOut, uint64_t** baseCountsOut /* R */,
    uint8_t** isMarkerOut /* 4^k */)
{
    try {
        QuietCout quiet(true);
        Reads reads;
        reads.createNew(1, "", "", "", "", "", "", 4096);
        {
            ReadLoader loader(fastaPath, 1, minReadLength, false, threadCount, "", 4096, reads);
        }
        MemoryMapped::Vector<KmerInfo> kmerTable;
        buildKmerTable(kmerTable, k, markerProbability, seed);
        const uint64_t R = reads.readCount();
        *readCountOut = R;
        uint64_t* offsets = (uint64_t*)malloc(sizeof(uint64_t) * (R + 1));
        uint64_t* baseCounts = (uint64_t*)malloc(sizeof(uint64_t) * (R ? R : 1));
        uint64_t total = 0;
        for(uint64_t r=0; r<R; r++) {
            const LongBaseSequenceView v = reads.getRead(ReadId(r));
            offsets[r] = total; baseCounts[r] = v.baseCount;
            total += LongBaseSequenceView::wordCount(v.baseCount);
        }
        offsets[R] = total;
        uint64_t* words = (uint64_t*)malloc(sizeof(uint64_t) * (total ? total : 1));
        for(uint64_t r=0; r<R; r++) {
            const LongBaseSequenceView v = reads.getRead(ReadId(r));
            memcpy(words + offsets[r], v.begin, sizeof(uint64_t) * (offsets[r+1] - offsets[r]));
        }
        const uint64_t n = 1ULL << (2*k);
        uint8_t* isMarker = (uint8_t*)malloc(n);
        for(uint64_t i=0; i<n; i++) isMarker[i] = kmerTable[i].isMarker ? 1 : 0;
        *wordOffsetsOut = offsets; *wordsOut = words; *baseCountsOut = baseCounts; *isMarkerOut = isMarker;
        kmerTable.remove();
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_reads_from_fasta: %s\n", e.what());
        return 1;
    }
}


// Run the reference LowHash0 on raw marker arrays.
//   toc: uint64[2R+1]; data: 7-byte CompressedMarker records; flags: 1 byte per read.
// Outputs: candidates as 12-byte OrientedReadPair records written as 3 x uint32
// {readId0, readId1, isSameStrand} (malloc'ed), stats: uint64[R][3] caller-allocated.
// seconds: wall time of the LowHash0 constructor alone.
int ref_lowhash0(
    uint64_t R, const uint64_t* toc, const uint8_t* data, const uint8_t* flags,
    uint64_t m, double hashFraction, uint64_t minHashIterationCount,
    double alignmentCandidatesPerRead, uint64_t log2MinHashBucketCount,
    uint64_t minBucketSize, uint64_t maxBucketSize, uint64_t minFrequency,
    uint64_t threadCount,
    uint32_t** candidatesOut, uint64_t* candidateCountOut, uint64_t* stats,
    double* seconds, int quiet,
    uint64_t* iterSummary /* optional: (highFrequency,total) per iteration */, uint64_t maxIters,
    uint64_t* iterationsOut /* optional */)
{
    try {
        QuietCout q(quiet != 0);
        // LowHash0 writes two CSV files into the cwd; keep them out of the repo.
        char oldCwd[4096];
        if(!getcwd(oldCwd, sizeof(oldCwd))) return 2;
        char tmpl[] = "/tmp/ref_lowhash_XXXXXX";
        char* tmpDir = mkdtemp(tmpl);
        if(!tmpDir || chdir(tmpDir)) return 2;

        Reads reads;
        reads.createNew(1, "", "", "", "", "", "", 4096);
        reads.readFlags.resize(R);
        for(uint64_t r=0; r<R; r++) {
            *reinterpret_cast<uint8_t*>(&reads.readFlags[r]) = flags[r];
        }

        MemoryMapped::VectorOfVectors<CompressedMarker, uint64_t> markers;
        markers.createNew("", 4096);
        markers.beginPass1(2*R);
        for(uint64_t i=0; i<2*R; i++) markers.incrementCount(i, toc[i+1]-toc[i]);
        markers.beginPass2();
        markers.endPass2(false);
        for(uint64_t i=0; i<2*R; i++) {
            memcpy(markers.begin(i), data + 7*toc[i], 7*(toc[i+1]-toc[i]));
        }

        MemoryMapped::Vector<KmerInfo> kmerTable;   // LowHash0 keeps a reference but never reads it.
        kmerTable.createNew("", 4096);
        MemoryMapped::Vector<OrientedReadPair> candidates;
        candidates.createNew("", 4096);
        MemoryMapped::Vector< array<uint64_t, 3> > readLowHashStatistics;
        readLowHashStatistics.createNew("", 4096);

        const auto t0 = std::chrono::steady_clock::now();
        {
            const string prefix;
            LowHash0 lowHash0(m, hashFraction, minHashIterationCount, alignmentCandidatesPerRead,
                log2MinHashBucketCount, minBucketSize, maxBucketSize, minFrequency, threadCount,
                kmerTable, reads, markers, candidates, readLowHashStatistics, prefix, 4096);
        }
        const auto t1 = std::chrono::steady_clock::now();
        if(seconds) *seconds = 1.e-9 * double(std::chrono::duration_cast<std::chrono::nanoseconds>(t1-t0).count());

        const uint64_t n = candidates.size();
        uint32_t* out = (uint32_t*)malloc(12*(n ? n : 1));
        for(uint64_t i=0; i<n; i++) {
            out[3*i+0] = candidates[i].readIds[0];
            out[3*i+1] = candidates[i].readIds[1];
            out[3*i+2] = candidates[i].isSameStrand ? 1 : 0;
        }
        *candidatesOut = out;
        *candidateCountOut = n;
        {
            // Parse "Alignment candidates after lowhash iteration I: high frequency H, total T, capacity C."
            std::istringstream lines(q.sink.str());
            string line; uint64_t it = 0;
            while(std::getline(lines, line)) {
                unsigned long long i, h, t;
                if(sscanf(line.c_str(), "Alignment candidates after lowhash iteration %llu: high frequency %llu, total %llu", &i, &h, &t) == 3) {
                    if(iterSummary && i < maxIters) { iterSummary[2*i] = h; iterSummary[2*i+1] = t; }
                    it = i + 1;
                }
            }
            if(iterationsOut) *iterationsOut = it;
        }
        for(uint64_t r=0; r<R; r++) for(int c=0; c<3; c++) stats[3*r+c] = readLowHashStatistics[r][c];

        candidates.remove();
        readLowHashStatistics.remove();
        markers.remove();
        kmerTable.remove();
        if(chdir(oldCwd)) return 2;
        // The CSV files the reference's constructor leaves in its working directory, for tests of the facade's writers.
        if(const char* keep = getenv("SHB_REF_KEEP_CSV")) {
            const std::string cp = std::string("cp ") + tmpDir + "/ReadLowHashStatistics.csv " + tmpDir + "/LowHashBucketHistogram.csv " + keep + "/ 2>/dev/null";
            if(system(cp.c_str())) {}
        }
        std::string cmd = std::string("rm -rf ") + tmpDir;
        if(system(cmd.c_str())) {}
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_lowhash0: %s\n", e.what());
        return 1;
    }
}

uint64_t ref_murmurhash64a(const void* key, int len, uint64_t seed) { return MurmurHash64A(key, len, seed); }
uint32_t ref_murmurhash2(const void* key, int len, uint32_t seed) { return MurmurHash2(key, len, seed); }

void ref_free(void* p) { free(p); }

} // extern "C"


// ---------------------------------------------------------------------------------------------
// Data/ directory interoperability (test infrastructure): the reference's own MemoryMapped code writes the
// inputs of the path as named files, and opens files written by shasta_b200/assembler.py.
#include "Alignment.hpp"

// Opens a MemoryMapped::Vector file with the reference's accessExistingReadOnly for the given record size and returns the
// object count and a byte checksum of the payload. Returns nonzero (and prints the reference's message) on failure.
template<class T> static int openVector(const char* path, uint64_t* count, uint64_t* checksum)
{
    MemoryMapped::Vector<T> v;
    v.accessExistingReadOnly(path);
    *count = v.size();
    uint64_t h = 1469598103934665603ULL;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(v.begin());
    for(uint64_t i = 0; i < v.size() * sizeof(T); i++) h = (h ^ bytes[i]) * 1099511628211ULL;
    *checksum = h;
    return 0;
}

extern "C" {

// Writes <prefix>Markers.{toc,data}, <prefix>ReadFlags and <prefix>Kmers exactly as the reference would
// (Reads::createNew / MarkerFinder / kmerTable with file-backed MemoryMapped vectors).
int ref_write_data_dir(const char* fastaPath, const char* prefix, uint64_t k, double markerProbability, int seed,
                       uint64_t minReadLength, uint64_t threadCount)
{
    try {
        QuietCout quiet(true);
        const string p(prefix);
        Reads reads;
        reads.createNew(1, p + "Reads", p + "ReadNames", p + "ReadMetaData", p + "ReadRepeatCounts", p + "ReadFlags",
                        p + "ReadIdsSortedByName", 4096);
        {
            ReadLoader loader(fastaPath, 1, minReadLength, false, threadCount, p, 4096, reads);
        }
        MemoryMapped::Vector<KmerInfo> kmerTable;
        {
            // buildKmerTable creates an anonymous table; copy it into a named one.
            MemoryMapped::Vector<KmerInfo> tmp;
            buildKmerTable(tmp, k, markerProbability, seed);
            kmerTable.createNew(p + "Kmers", 4096);
            kmerTable.resize(tmp.size());
            for(uint64_t i = 0; i < tmp.size(); i++) kmerTable[i] = tmp[i];
            tmp.remove();
        }
        MemoryMapped::VectorOfVectors<CompressedMarker, uint64_t> markers;
        markers.createNew(p + "Markers", 4096);
        {
            MarkerFinder finder(k, kmerTable, reads, markers, threadCount);
        }
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_write_data_dir: %s\n", e.what());
        return 1;
    }
}

int ref_open_vector(const char* path, uint64_t objectSize, uint64_t* count, uint64_t* checksum)
{
    try {
        switch(objectSize) {
        case 1: return openVector<uint8_t>(path, count, checksum);
        case 4: return openVector<uint32_t>(path, count, checksum);
        case 7: return openVector<CompressedMarker>(path, count, checksum);
        case 8: return openVector<uint64_t>(path, count, checksum);
        case 12: return openVector<OrientedReadPair>(path, count, checksum);
        case 24: return openVector< array<uint64_t, 3> >(path, count, checksum);
        case 64: return openVector<AlignmentData>(path, count, checksum);
        default: return 2;
        }
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_open_vector: %s\n", e.what());
        return 1;
    }
}

} // extern "C"
