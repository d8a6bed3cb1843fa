// Device code of flagPalindromicReads (src/AssemblerAlign.cpp:652-770 of chanzuckerberg/shasta): the prefilter of phase A
// and the alignment method 0 of phase B (shasta::align, src/AlignmentGraph.cpp:14-136) of a read against its reverse
// complement.
//
// The reference's path depends on how its unstable std::sort orders equal keys and on how its std::priority_queue breaks
// ties between equal distances, so phase B restates those libstdc++ algorithms step for step (bits/stl_algo.h and
// bits/stl_heap.h of GCC are the specification; the tests hold this code to a CPU restatement of the same algorithms).
#pragma once

#include "common.cuh"

namespace shb {
namespace pal {

struct Marker { uint32_t kmerId, ordinal; };      // MarkerWithOrdinal, ordered by kmerId only
struct Vertex { uint32_t o0, o1; };               // AlignmentGraphVertex, ordered by ordinals[0] only
struct Edge { uint32_t a, b; uint64_t w; };
struct HeapItem { uint64_t d; uint32_t v; };      // pair<distance, vertex>, ordered by distance only (greater)

struct MarkerLess { __device__ bool operator()(const Marker& x, const Marker& y) const { return x.kmerId < y.kmerId; } };
struct VertexLess { __device__ bool operator()(const Vertex& x, const Vertex& y) const { return x.o0 < y.o0; } };
struct HeapLess { __device__ bool operator()(const HeapItem& x, const HeapItem& y) const { return x.d > y.d; } };

// std::__push_heap
template<class T, class L> __device__ void pushHeap(T* f, int64_t hole, int64_t top, T value, L less)
{
    int64_t parent = (hole - 1) / 2;
    while(hole > top && less(f[parent], value)) { f[hole] = f[parent]; hole = parent; parent = (hole - 1) / 2; }
    f[hole] = value;
}
// std::__adjust_heap
template<class T, class L> __device__ void adjustHeap(T* f, int64_t hole, int64_t len, T value, L less)
{
    const int64_t top = hole;
    int64_t child = hole;
    while(child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if(less(f[child], f[child - 1])) child--;
        f[hole] = f[child]; hole = child;
    }
    if((len & 1) == 0 && child == (len - 2) / 2) { child = 2 * (child + 1); f[hole] = f[child - 1]; hole = child - 1; }
    pushHeap(f, hole, top, value, less);
}
template<class T> __device__ void swapAt(T* a, T* b) { const T t = *a; *a = *b; *b = t; }
template<class T, class L> __device__ void linearInsert(T* last, L less)
{
    const T value = *last;
    T* next = last - 1;
    while(less(value, *next)) { *last = *next; last = next; --next; }
    *last = value;
}

// std::sort: __introsort_loop (median of three moved to the first element, unguarded partition, __partial_sort = make_heap
// + sort_heap once the depth limit 2 * floor(log2 n) is used up) and __final_insertion_sort. One thread. The recursion on
// the right part becomes an explicit stack: the parts are disjoint, so the order they are finished in does not matter.
template<class T, class L> __device__ uint32_t stdSort(T* first, int64_t n, L less)
{
    if(n <= 0) return 0;
    uint32_t fallbacks = 0;
    struct Range { T* f; T* l; int depth; };
    Range stack[80];
    int top = 0;
    stack[top++] = Range{first, first + n, 2 * (63 - __clzll((unsigned long long)n))};
    while(top) {
        Range r = stack[--top];
        T* f = r.f; T* l = r.l; int depth = r.depth;
        while(l - f > 16) {
            if(depth == 0) {
                const int64_t len = l - f;
                for(int64_t parent = (len - 2) / 2; ; parent--) { adjustHeap(f, parent, len, f[parent], less); if(parent == 0) break; }
                for(int64_t k = len; k > 1; ) { k--; const T value = f[k]; f[k] = f[0]; adjustHeap(f, int64_t(0), k, value, less); }
                fallbacks++;
                break;
            }
            --depth;
            T* a = f + 1; T* b = f + (l - f) / 2; T* c = l - 1;
            if(less(*a, *b)) {
                if(less(*b, *c)) swapAt(f, b); else if(less(*a, *c)) swapAt(f, c); else swapAt(f, a);
            } else if(less(*a, *c)) swapAt(f, a);
            else if(less(*b, *c)) swapAt(f, c);
            else swapAt(f, b);
            T* lo = f + 1; T* hi = l;
            for(;;) {
                while(less(*lo, *f)) ++lo;
                --hi;
                while(less(*f, *hi)) --hi;
                if(!(lo < hi)) break;
                swapAt(lo, hi); ++lo;
            }
            stack[top++] = Range{lo, l, depth};
            l = lo;
        }
    }
    const int64_t guarded = n < 16 ? n : 16;
    for(T* i = first + 1; i < first + guarded; ++i) {           // __insertion_sort of the first 16
        if(less(*i, *first)) { const T value = *i; for(T* j = i; j > first; --j) *j = *(j - 1); *first = value; }
        else linearInsert(i, less);
    }
    for(T* i = first + guarded; i < first + n; ++i) linearInsert(i, less);     // __unguarded_insertion_sort
    return fallbacks;
}

} // namespace pal
} // namespace shb
