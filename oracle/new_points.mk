# The new-map-point checker (test infrastructure): make -C oracle -f new_points.mk [ref | shim-check]
#   libnew_points_oracle.so   the sequential loop of LocalMapping::CreateNewMapPoints over the flat views (new_points_oracle.cpp): the
#                             oracle's reference-pinned orc_match_triangulation from liboracle.so per neighbour, then the triangulation
#                             and its gates written out as the reference writes them.  It shares one thing with the product, the 4x4
#                             decomposition of ccm_slam_b200/csrc/new_points_math.cuh, compiled here by g++ with -ffp-contract=off.
#   _ref/libnew_points_shim.so      shim/NewMapPoints_shim.cpp on the stand-in LocalMapping / KeyFrame / MapPoint / Map of ref_stub_np/, next
#                                   to a literal restatement of the reference body (ref_new_points_wrap.cpp); the device entry point
#                                   ccm_new_map_points doubled on the CPU by the oracle (ccm_new_points_double.cpp)
#   _ref/libnew_points_shim_gpu.so  the same over the real device entry point (GPU suite)
# None of them reads the reference tree.  Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off

libnew_points_oracle.so: new_points_oracle.cpp ../ccm_slam_b200/csrc/new_points_math.cuh ../include/ccm_b200.h liboracle.so
	$(CXX) $(CXXFLAGS) -Wno-unknown-pragmas -I../include -shared -o $@ new_points_oracle.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'

REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_np -Iref_stub_mp -Iref_stub -I../include
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_new_points_wrap.cpp ../shim/NewMapPoints_shim.cpp
SHIM_DEPS = $(SHIM_SRCS) ../shim/NewMapPoints_shim.h ../include/ccm_b200.h ref_stub_np/cslam/Mapping.h ../ccm_slam_b200/csrc/new_points_math.cuh \
            liboracle.so $(PRODUCT)/libccm_b200.so

_ref/libnew_points_shim.so: $(SHIM_DEPS) ccm_new_points_double.cpp libnew_points_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_new_points_double.cpp -L. -lnew_points_oracle -loracle \
	    -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libnew_points_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L. -loracle -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' \
	    -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libnew_points_shim.so _ref/libnew_points_shim_gpu.so,)

# type-check the shim against the stand-in LocalMapping (each member cites the line of the real header it mirrors)
shim-check:
	$(REF_CXX) -std=c++14 -fsyntax-only -w $(STUB) ../shim/NewMapPoints_shim.cpp

liboracle.so:
	$(MAKE) -f Makefile liboracle.so

ref: libnew_points_oracle.so $(SHIM_LIBS)

clean:
	rm -f libnew_points_oracle.so _ref/libnew_points_shim.so _ref/libnew_points_shim_gpu.so

.PHONY: ref shim-check clean
