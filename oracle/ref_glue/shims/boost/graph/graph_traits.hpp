// TEST INFRASTRUCTURE shim (boost is absent): a graph_traits<G> that forwards to G's own typedefs, and two category tags.
#pragma once
#include <utility>
namespace boost {
struct allow_parallel_edge_tag {}; struct adjacency_graph_tag {};
template<class G> struct graph_traits {
    using vertex_descriptor = typename G::vertex_descriptor;
    using edge_descriptor = typename G::edge_descriptor;
    using vertex_iterator = typename G::vertex_iterator;
    using edge_iterator = typename G::edge_iterator;
    using out_edge_iterator = typename G::out_edge_iterator;
};
}
