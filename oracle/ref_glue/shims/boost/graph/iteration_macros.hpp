// TEST INFRASTRUCTURE shim (boost is absent): the BGL_FORALL_* loops of src/CompactUndirectedGraph.hpp, src/shortestPath.hpp and
// src/AlignmentGraph.cpp over vertices() / edges() / out_edges().
#pragma once
#include <boost/graph/graph_traits.hpp>
#define SHB_CAT2(a,b) a##b
#define SHB_CAT(a,b) SHB_CAT2(a,b)
#define BGL_FORALL_VERTICES_T(v, g, G) \
  for(auto SHB_CAT(_r,__LINE__) = vertices(g); SHB_CAT(_r,__LINE__).first != SHB_CAT(_r,__LINE__).second; ++SHB_CAT(_r,__LINE__).first) \
    if(bool SHB_CAT(_b,__LINE__) = false) {} else for(typename boost::graph_traits<G>::vertex_descriptor v = *SHB_CAT(_r,__LINE__).first; !SHB_CAT(_b,__LINE__); SHB_CAT(_b,__LINE__) = true)
#define BGL_FORALL_VERTICES(v, g, G) \
  for(auto SHB_CAT(_r,__LINE__) = vertices(g); SHB_CAT(_r,__LINE__).first != SHB_CAT(_r,__LINE__).second; ++SHB_CAT(_r,__LINE__).first) \
    if(bool SHB_CAT(_b,__LINE__) = false) {} else for(boost::graph_traits<G>::vertex_descriptor v = *SHB_CAT(_r,__LINE__).first; !SHB_CAT(_b,__LINE__); SHB_CAT(_b,__LINE__) = true)
#define BGL_FORALL_EDGES(e, g, G) \
  for(auto SHB_CAT(_r,__LINE__) = edges(g); SHB_CAT(_r,__LINE__).first != SHB_CAT(_r,__LINE__).second; ++SHB_CAT(_r,__LINE__).first) \
    if(bool SHB_CAT(_b,__LINE__) = false) {} else for(boost::graph_traits<G>::edge_descriptor e = *SHB_CAT(_r,__LINE__).first; !SHB_CAT(_b,__LINE__); SHB_CAT(_b,__LINE__) = true)
#define BGL_FORALL_OUTEDGES_T(u, e, g, G) \
  for(auto SHB_CAT(_r,__LINE__) = out_edges(u, g); SHB_CAT(_r,__LINE__).first != SHB_CAT(_r,__LINE__).second; ++SHB_CAT(_r,__LINE__).first) \
    if(bool SHB_CAT(_b,__LINE__) = false) {} else for(typename boost::graph_traits<G>::edge_descriptor e = *SHB_CAT(_r,__LINE__).first; !SHB_CAT(_b,__LINE__); SHB_CAT(_b,__LINE__) = true)
