# TEST INFRASTRUCTURE. Builds _ref/libshasta_ref_markergraph_edges.so: the reference's UNMODIFIED MarkerGraph.cpp,
# MultithreadedObject.cpp, SHASTA_ASSERT.cpp and touchMemory.cpp, compiled from where they lie under $(SHASTA_REF_SRC), plus
# the extern "C" glue ref_glue/ref_markergraph_edges.cpp that follows createMarkerGraphEdges, its source and target tables and
# findMarkerGraphReverseComplementEdges over them. Only when that tree exists; where it does not (the GPU machines), the
# prebuilt library is kept. No reference source is copied into this repository.
#   make -C oracle -f markergraph_edges.mk ref
SHASTA_REF_SRC ?= /root/reference/src
CXX = /usr/bin/g++

MGE_TUS = MarkerGraph MultithreadedObject SHASTA_ASSERT touchMemory
MGE_FLAGS = -std=c++20 -O3 -DNDEBUG -mcx16 -fPIC -include cstdint -include limits -I$(SHASTA_REF_SRC) -w
MGE_OBJS = $(addprefix _ref/obj_markergraph_edges/,$(addsuffix .o,$(MGE_TUS))) _ref/obj_markergraph_edges/ref_markergraph_edges.o

ref:
	@if [ -d $(SHASTA_REF_SRC) ]; then $(MAKE) -f markergraph_edges.mk _ref/libshasta_ref_markergraph_edges.so; else echo "reference tree absent: keeping prebuilt _ref"; fi

_ref/obj_markergraph_edges/%.o: $(SHASTA_REF_SRC)/%.cpp
	mkdir -p _ref/obj_markergraph_edges
	$(CXX) $(MGE_FLAGS) -c $< -o $@

_ref/obj_markergraph_edges/ref_markergraph_edges.o: ref_glue/ref_markergraph_edges.cpp
	mkdir -p _ref/obj_markergraph_edges
	$(CXX) $(MGE_FLAGS) -c $< -o $@

_ref/libshasta_ref_markergraph_edges.so: $(MGE_OBJS)
	$(CXX) -shared -Wl,-z,defs -o $@ $(MGE_OBJS) -lpthread -latomic

.PHONY: ref
