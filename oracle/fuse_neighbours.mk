# The neighbour-fusion checker (test infrastructure): make -C oracle -f fuse_neighbours.mk ref
#   libfuse_neighbours_oracle.so   every pair LocalMapping::SearchInNeighbors searches, over the start-of-member state
#                                  (fuse_neighbours_oracle.cpp): Fuse's prelude written out as the reference writes it, with the host's
#                                  logf, and the reference-pinned window search orc_fuse_search of liboracle.so.  Shares nothing with
#                                  the product but the C structs of include/ccm_b200.h.
#   _ref/libfuse_neighbours_shim.so      shim/FuseNeighbours_shim.cpp on the stand-in LocalMapping / KeyFrame / MapPoint / Map of
#                                        ref_stub_fn/, next to a literal restatement of SearchInNeighbors, Fuse and Replace
#                                        (ref_fuse_neighbours_wrap.cpp); the device entry point answered by the host entry point
#                                        (ccm_fuse_neighbours_double.cpp)
#   _ref/libfuse_neighbours_shim_gpu.so  the same over the real device entry point (GPU suite)
# None of them reads the reference tree.  Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off

libfuse_neighbours_oracle.so: fuse_neighbours_oracle.cpp ../include/ccm_b200.h liboracle.so
	$(CXX) $(CXXFLAGS) -I../include -shared -o $@ fuse_neighbours_oracle.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'

REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_fn -Iref_stub_mp -Iref_stub -I../include -I../shim
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_fuse_neighbours_wrap.cpp ../shim/FuseNeighbours_shim.cpp
SHIM_DEPS = $(SHIM_SRCS) ../shim/FuseNeighbours_shim.h ../shim/MapPointDescriptor_shim.h ../include/ccm_b200.h ref_stub_fn/cslam/Mapping.h \
            $(PRODUCT)/libccm_b200.so

_ref/libfuse_neighbours_shim.so: $(SHIM_DEPS) ccm_fuse_neighbours_double.cpp
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_fuse_neighbours_double.cpp -L$(PRODUCT) -lccm_b200 \
	    -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libfuse_neighbours_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libfuse_neighbours_shim.so _ref/libfuse_neighbours_shim_gpu.so,)

# type-check the shim against the stand-in LocalMapping (each member cites the line of the real header it mirrors)
shim-check:
	$(REF_CXX) -std=c++14 -fsyntax-only -w $(STUB) ../shim/FuseNeighbours_shim.cpp

liboracle.so:
	$(MAKE) -f Makefile liboracle.so

ref: libfuse_neighbours_oracle.so $(SHIM_LIBS)

clean:
	rm -f libfuse_neighbours_oracle.so _ref/libfuse_neighbours_shim.so _ref/libfuse_neighbours_shim_gpu.so

.PHONY: ref shim-check clean
