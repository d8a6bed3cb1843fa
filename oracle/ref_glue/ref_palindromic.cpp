// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// extern "C" access to the reference's palindromic-read decision, compiled unmodified from the reference tree by
// oracle/Makefile into oracle/_ref/libshasta_ref_palindromic.so:
//   getMarkersSortedByKmerId        src/AssemblerMarkers.cpp:83-98   (restated here: std::sort of MarkerWithOrdinal)
//   shasta::align / AlignmentGraph  src/AlignmentGraph.cpp:14-136    (compiled unmodified, with ref_glue/shims/boost/graph)
//   the two thresholds              src/AssemblerAlign.cpp:741-766   (restated here)
#include <algorithm>         // before the reference headers: CompactUndirectedGraph.hpp uses std::reverse without it
#include "AlignmentGraph.hpp"
#include "Alignment.hpp"
#include "Marker.hpp"
#include "PngImage.hpp"

#include <cstdlib>
#include <cstring>
#include <vector>

using namespace shasta;

// PngImage is only reachable from AlignmentGraph::writeImage, debug output that is never called here; link-time stubs
// (libpng is absent).
PngImage::PngImage(int w, int h) : width(w), height(h) {}
void PngImage::setPixel(int, int, int, int, int) {}
void PngImage::write(const string&) const {}
void PngImage::writeGrid(int, int, int, int) {}
void PngImage::magnify(int) {}

extern "C" {

// Rows: toc uint64[2R+1] (relative), kmerIds uint32[toc[2R]]; read r is rows 2r (strand 0) and 2r+1 (strand 1).
// Per read: flags[r] (1 = palindromic), aligned[r], nearDiagonal[r]. When pathRead < R, *pathOut gets a malloc'ed
// uint32[2 * *pathCount] of that read's alignment ordinals.
int ref_flag_palindromic(uint64_t R, const uint64_t* toc, const uint32_t* kmerIds,
                         uint32_t maxSkip, uint32_t maxDrift, uint32_t maxMarkerFrequency,
                         double alignedFractionThreshold, double nearDiagonalFractionThreshold, uint32_t deltaThreshold,
                         uint8_t* flags, uint32_t* aligned, uint32_t* nearDiagonal,
                         uint64_t pathRead, uint32_t** pathOut, uint64_t* pathCount)
{
    try {
        AlignmentGraph graph;
        Alignment alignment;
        AlignmentInfo alignmentInfo;
        array<vector<MarkerWithOrdinal>, 2> markersSortedByKmerId;
        for(uint64_t r = 0; r < R; r++) {
            // src/AssemblerMarkers.cpp:83-98, with position = ordinal (positions do not reach the decision).
            for(int strand = 0; strand < 2; strand++) {
                const uint64_t b = toc[2 * r + strand], e = toc[2 * r + strand + 1];
                vector<MarkerWithOrdinal>& m = markersSortedByKmerId[strand];
                m.clear();
                m.resize(e - b);
                for(uint32_t ordinal = 0; ordinal < e - b; ordinal++) {
                    CompressedMarker cm;
                    cm.kmerId = kmerIds[b + ordinal];
                    cm.position = ordinal;
                    m[ordinal] = MarkerWithOrdinal(cm, ordinal);
                }
                sort(m.begin(), m.end());
            }
            // src/AssemblerAlign.cpp:736-766
            align(markersSortedByKmerId, maxSkip, maxDrift, maxMarkerFrequency, false, graph, alignment, alignmentInfo);
            const size_t alignedMarkerCount = alignment.ordinals.size();
            const size_t totalMarkerCount = markersSortedByKmerId[0].size();
            size_t nearDiagonalMarkerCount = 0;
            for(size_t i = 0; i < alignment.ordinals.size(); i++) {
                const int32_t ordinal0 = int32_t(alignment.ordinals[i][0]);
                const int32_t ordinal1 = int32_t(alignment.ordinals[i][1]);
                const uint32_t delta = abs(ordinal0 - ordinal1);
                if(delta < deltaThreshold) nearDiagonalMarkerCount++;
            }
            const double alignedFraction = double(alignedMarkerCount) / double(totalMarkerCount);
            const double nearDiagonalFraction = double(nearDiagonalMarkerCount) / double(totalMarkerCount);
            flags[r] = !(alignedFraction < alignedFractionThreshold) && !(nearDiagonalFraction < nearDiagonalFractionThreshold);
            aligned[r] = uint32_t(alignedMarkerCount);
            nearDiagonal[r] = uint32_t(nearDiagonalMarkerCount);
            if(r == pathRead) {
                const uint64_t k = alignment.ordinals.size();
                uint32_t* out = (uint32_t*)malloc(8 * (k ? k : 1));
                for(uint64_t i = 0; i < k; i++) { out[2*i] = alignment.ordinals[i][0]; out[2*i+1] = alignment.ordinals[i][1]; }
                *pathOut = out;
                *pathCount = k;
            }
        }
        return 0;
    } catch(const std::exception& e) {
        fprintf(stderr, "ref_flag_palindromic: %s\n", e.what());
        return 1;
    }
}

void ref_free_palindromic(void* p) { free(p); }

} // extern "C"
