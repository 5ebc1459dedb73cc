# The loop / merge fusion checker (test infrastructure): make -C oracle -f search_and_fuse.mk ref
#   libsearch_and_fuse_oracle.so   every (corrected keyframe, loop point) pair LoopFinder / MapMerger::SearchAndFuse searches, over the
#                                  start-of-member state (search_and_fuse_oracle.cpp): Fuse(Scw)'s prelude written out as the reference
#                                  writes it, with the host's logf, and the reference-pinned window search orc_fuse_search of
#                                  liboracle.so.  Shares nothing with the product but the C structs of include/ccm_b200.h, and does not
#                                  read the reference tree.
#   _ref/libsearch_and_fuse_shim.so      shim/SearchAndFuse_shim.cpp on the stand-in KeyFrame / MapPoint / Map / Converter of ref_stub_sf/
#                                        (g2o::Sim3 from ref_stub_sc/), next to a literal restatement of both SearchAndFuse bodies, Fuse(Scw),
#                                        Replace and ReplaceAndLock (ref_search_and_fuse_wrap.cpp); the device entry point answered by the
#                                        host entry point (ccm_search_and_fuse_double.cpp)
#   _ref/libsearch_and_fuse_shim_gpu.so  the same over the real device entry point (GPU suite)
# Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off

libsearch_and_fuse_oracle.so: search_and_fuse_oracle.cpp ../include/ccm_b200.h liboracle.so
	$(CXX) $(CXXFLAGS) -I../include -shared -o $@ search_and_fuse_oracle.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'

REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_sf -Iref_stub_sc -Iref_stub_mp -Iref_stub -I../include -I../shim
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_search_and_fuse_wrap.cpp ../shim/SearchAndFuse_shim.cpp
SHIM_DEPS = $(SHIM_SRCS) ../shim/SearchAndFuse_shim.h ../shim/Sim3Split_shim.h ../shim/Sim3Correction_shim.h ../include/ccm_b200.h \
            ref_stub_sf/cslam/KeyFrame.h ref_stub_sf/cslam/Converter.h $(PRODUCT)/libccm_b200.so

_ref/libsearch_and_fuse_shim.so: $(SHIM_DEPS) ccm_search_and_fuse_double.cpp
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_search_and_fuse_double.cpp -L$(PRODUCT) -lccm_b200 \
	    -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libsearch_and_fuse_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libsearch_and_fuse_shim.so _ref/libsearch_and_fuse_shim_gpu.so,)

# type-check the shim against the stand-ins
shim-check:
	$(REF_CXX) -std=c++14 -fsyntax-only -w $(STUB) ../shim/SearchAndFuse_shim.cpp

liboracle.so:
	$(MAKE) -f Makefile liboracle.so

ref: libsearch_and_fuse_oracle.so $(SHIM_LIBS)

clean:
	rm -f libsearch_and_fuse_oracle.so _ref/libsearch_and_fuse_shim.so _ref/libsearch_and_fuse_shim_gpu.so

.PHONY: ref shim-check clean
