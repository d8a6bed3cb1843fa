# TEST INFRASTRUCTURE. Builds _ref/libshasta_ref_readgraph_flags.so: the reference's UNMODIFIED ReadGraph.cpp (the read
# graph and ReadGraph::computeShortPath) and the translation units it links against, compiled from where they lie under
# $(SHASTA_REF_SRC) against the boost shims in ref_glue/shims, plus the extern "C" glue ref_glue/ref_readgraph_flags.cpp that
# follows flagCrossStrandReadGraphEdges1 and flagChimericReads over them. Only when that tree exists; where it does not
# (the GPU machines), the prebuilt library is kept. No reference source is copied into this repository.
#   make -C oracle -f readgraph_flags.mk ref
SHASTA_REF_SRC ?= /root/reference/src
CXX = /usr/bin/g++

RGF_TUS = ReadGraph SHASTA_ASSERT touchMemory
RGF_SHIMS = $(wildcard ref_glue/shims/*.h) $(wildcard ref_glue/shims/boost/*/*.hpp)
RGF_FLAGS = -std=c++20 -O3 -DNDEBUG -mcx16 -fPIC -include cstdint -include algorithm -I$(SHASTA_REF_SRC) -Iref_glue/shims -w
RGF_OBJS = $(addprefix _ref/obj_readgraph_flags/,$(addsuffix .o,$(RGF_TUS))) _ref/obj_readgraph_flags/ref_readgraph_flags.o

ref:
	@if [ -d $(SHASTA_REF_SRC) ]; then $(MAKE) -f readgraph_flags.mk _ref/libshasta_ref_readgraph_flags.so; else echo "reference tree absent: keeping prebuilt _ref"; fi

_ref/obj_readgraph_flags/%.o: $(SHASTA_REF_SRC)/%.cpp $(RGF_SHIMS)
	mkdir -p _ref/obj_readgraph_flags
	$(CXX) $(RGF_FLAGS) -c $< -o $@

_ref/obj_readgraph_flags/ref_readgraph_flags.o: ref_glue/ref_readgraph_flags.cpp $(RGF_SHIMS)
	mkdir -p _ref/obj_readgraph_flags
	$(CXX) $(RGF_FLAGS) -c $< -o $@

_ref/libshasta_ref_readgraph_flags.so: $(RGF_OBJS)
	$(CXX) -shared -Wl,-z,defs -o $@ $(RGF_OBJS) -lpthread -latomic

.PHONY: ref
