# TEST INFRASTRUCTURE. Builds _ref/libshasta_ref_markergraph.so: the reference's UNMODIFIED PeakFinder.cpp,
# compressAlignment.cpp and the header-only DisjointSets (dset64-gccAtomic.hpp), compiled from where they lie under
# $(SHASTA_REF_SRC) (with touchMemory.cpp for MemoryMapped::Vector), plus the extern "C" glue ref_glue/ref_markergraph.cpp that follows createMarkerGraphVertices and
# findMarkerGraphReverseComplementVertices over them. Only when that tree exists; where it does not (the GPU machines), the
# prebuilt library is kept. No reference source is copied into this repository.
#   make -C oracle -f markergraph.mk ref
SHASTA_REF_SRC ?= /root/reference/src
CXX = /usr/bin/g++

MG_TUS = PeakFinder compressAlignment SHASTA_ASSERT touchMemory
MG_FLAGS = -std=c++20 -O3 -DNDEBUG -mcx16 -fPIC -include cstdint -include limits -I$(SHASTA_REF_SRC) -w
MG_OBJS = $(addprefix _ref/obj_markergraph/,$(addsuffix .o,$(MG_TUS))) _ref/obj_markergraph/ref_markergraph.o

ref:
	@if [ -d $(SHASTA_REF_SRC) ]; then $(MAKE) -f markergraph.mk _ref/libshasta_ref_markergraph.so; else echo "reference tree absent: keeping prebuilt _ref"; fi

_ref/obj_markergraph/%.o: $(SHASTA_REF_SRC)/%.cpp
	mkdir -p _ref/obj_markergraph
	$(CXX) $(MG_FLAGS) -c $< -o $@

_ref/obj_markergraph/ref_markergraph.o: ref_glue/ref_markergraph.cpp
	mkdir -p _ref/obj_markergraph
	$(CXX) $(MG_FLAGS) -c $< -o $@

_ref/libshasta_ref_markergraph.so: $(MG_OBJS)
	$(CXX) -shared -Wl,-z,defs -o $@ $(MG_OBJS) -lpthread -latomic

.PHONY: ref
