// TEST INFRASTRUCTURE shim (boost is absent): the undirectedS tag that src/CompactUndirectedGraph.hpp names.
#pragma once
namespace boost { struct undirectedS {}; struct directedS {}; struct bidirectionalS {}; }
