# The map-point descriptor checker (test infrastructure): make -C oracle -f distinctive.mk [ref | shim-check]
#   libdistinctive_oracle.so          our restatement of MapPoint::ComputeDistinctiveDescriptors over the flat arrays (distinctive_oracle.cpp)
#   _ref/libdistinctive_shim.so       shim/MapPointDescriptor_shim.cpp AND shim/MapPoint_shim.cpp on the stand-in MapPoint / KeyFrame of
#                                     ref_stub_dd/, next to a literal restatement of the reference body (ref_distinctive_wrap.cpp); the
#                                     device entry points ccm_distinctive_descriptors, ccm_kfstore_distinctive_descriptors and
#                                     ccm_normal_depth doubled on the CPU by the oracles (ccm_distinctive_double.cpp,
#                                     ccm_normal_depth_double.cpp), the host entry points from libccm_b200.so
#   _ref/libdistinctive_shim_gpu.so   the same over the real device entry points (GPU suite)
# None of them reads the reference tree.  Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off
REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_dd -Iref_stub_mp -Iref_stub -I../include
SHIM_FLAGS = -O2 -fPIC -std=c++11 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_distinctive_wrap.cpp ../shim/MapPointDescriptor_shim.cpp ../shim/MapPoint_shim.cpp

libdistinctive_oracle.so: distinctive_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ distinctive_oracle.cpp

libnormal_depth_oracle.so: normal_depth_oracle.cpp
	$(MAKE) -s -f normal_depth.mk libnormal_depth_oracle.so

SHIM_DEPS = $(SHIM_SRCS) ../shim/MapPointDescriptor_shim.h ../shim/MapPoint_shim.h ../include/ccm_b200.h ref_stub_dd/cslam/MapPoint.h \
            $(PRODUCT)/libccm_b200.so

_ref/libdistinctive_shim.so: $(SHIM_DEPS) ccm_distinctive_double.cpp ccm_normal_depth_double.cpp libdistinctive_oracle.so libnormal_depth_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_distinctive_double.cpp ccm_normal_depth_double.cpp \
	    -L. -ldistinctive_oracle -lnormal_depth_oracle -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' \
	    -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libdistinctive_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libdistinctive_shim.so _ref/libdistinctive_shim_gpu.so,)
ref: libdistinctive_oracle.so $(SHIM_LIBS)

# type-check the shim against the stand-in MapPoint (each member cites the cslam/MapPoint.h line it mirrors)
shim-check:
	$(REF_CXX) -std=c++11 -fsyntax-only -w $(STUB) ../shim/MapPointDescriptor_shim.cpp

clean:
	rm -f libdistinctive_oracle.so _ref/libdistinctive_shim.so _ref/libdistinctive_shim_gpu.so

.PHONY: ref shim-check clean
