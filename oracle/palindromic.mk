# TEST INFRASTRUCTURE. Builds _ref/libshasta_ref_palindromic.so: the reference's UNMODIFIED AlignmentGraph.cpp (alignment
# method 0, used by flagPalindromicReads) and the translation units it links against, compiled from where they lie under
# $(SHASTA_REF_SRC), plus the extern "C" glue ref_glue/ref_palindromic.cpp. Only when that tree exists; where it does not
# (the GPU machines), the prebuilt library is kept. No reference source is copied into this repository.
#   make -C oracle -f palindromic.mk ref
SHASTA_REF_SRC ?= /root/reference/src
CXX = /usr/bin/g++

PAL_TUS = AlignmentGraph Alignment SHASTA_ASSERT
PAL_SHIMS = $(wildcard ref_glue/shims/*.h) $(wildcard ref_glue/shims/boost/graph/*.hpp)
# AlignmentGraph.cpp and CompactUndirectedGraph.hpp call std::sort and std::reverse without including <algorithm>.
PAL_FLAGS = -std=c++20 -O3 -DNDEBUG -mcx16 -fPIC -include cstdint -include algorithm -I$(SHASTA_REF_SRC) -Iref_glue/shims -w
PAL_OBJS = $(addprefix _ref/obj_palindromic/,$(addsuffix .o,$(PAL_TUS))) _ref/obj_palindromic/ref_palindromic.o

ref:
	@if [ -d $(SHASTA_REF_SRC) ]; then $(MAKE) -f palindromic.mk _ref/libshasta_ref_palindromic.so; else echo "reference tree absent: keeping prebuilt _ref"; fi

_ref/obj_palindromic/%.o: $(SHASTA_REF_SRC)/%.cpp $(PAL_SHIMS)
	mkdir -p _ref/obj_palindromic
	$(CXX) $(PAL_FLAGS) -c $< -o $@

_ref/obj_palindromic/ref_palindromic.o: ref_glue/ref_palindromic.cpp $(PAL_SHIMS)
	mkdir -p _ref/obj_palindromic
	$(CXX) $(PAL_FLAGS) -c $< -o $@

_ref/libshasta_ref_palindromic.so: $(PAL_OBJS)
	$(CXX) -shared -Wl,-z,defs -o $@ $(PAL_OBJS) -lpthread -latomic

.PHONY: ref
