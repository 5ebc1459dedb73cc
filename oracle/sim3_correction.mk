# The Sim3 correction checker (test infrastructure): make -C oracle -f sim3_correction.mk [ref | shim-check]
#   libsim3_correction_oracle.so   our flat restatement of the Sim3 pass of LoopFinder::CorrectLoop / MapMerger::MergeMaps over the
#                                  arrays of ccm_sim3_correction (sim3_correction_oracle.cpp): the entries walked in order with a live
#                                  centre table, each point's normal from libnormal_depth_oracle.so (oracle/normal_depth.mk)
#   _ref/libsim3_correction_shim.so     shim/Sim3Correction_shim.cpp and shim/MapPoint_shim.cpp on the stand-ins of ref_stub_sc/,
#                                       next to a literal restatement of both loop bodies (ref_sim3_correction_wrap.cpp); the device entry
#                                       point ccm_sim3_correction doubled on the CPU by the oracle (ccm_sim3_correction_double.cpp)
#   _ref/libsim3_correction_shim_gpu.so the same over the real device entry point (GPU suite)
# None of them reads the reference tree.  Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off

libsim3_correction_oracle.so: sim3_correction_oracle.cpp libnormal_depth_oracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ sim3_correction_oracle.cpp -L. -lnormal_depth_oracle -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

libnormal_depth_oracle.so: normal_depth_oracle.cpp
	$(MAKE) -f normal_depth.mk libnormal_depth_oracle.so

REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_sc -Iref_stub_mp -Iref_stub -I../include -I../shim
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_sim3_correction_wrap.cpp ../shim/Sim3Correction_shim.cpp ../shim/MapPoint_shim.cpp
SHIM_DEPS = $(SHIM_SRCS) ../shim/Sim3Correction_shim.h ../shim/MapPoint_shim.h ../shim/KeyFrameConnections_shim.h ../include/ccm_b200.h \
            ref_stub_sc/cslam/KeyFrame.h ref_stub_sc/thirdparty/g2o/g2o/types/sim3.h $(PRODUCT)/libccm_b200.so

_ref/libsim3_correction_shim.so: $(SHIM_DEPS) ccm_sim3_correction_double.cpp libsim3_correction_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_sim3_correction_double.cpp -L. -lsim3_correction_oracle \
	    -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libsim3_correction_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libsim3_correction_shim.so _ref/libsim3_correction_shim_gpu.so,)
ref: libsim3_correction_oracle.so $(SHIM_LIBS)

# type-check the shim against the stand-ins (each member cites the cslam header line it mirrors)
shim-check:
	$(REF_CXX) -std=c++11 -fsyntax-only -w $(STUB) ../shim/Sim3Correction_shim.cpp

clean:
	rm -f libsim3_correction_oracle.so _ref/libsim3_correction_shim.so _ref/libsim3_correction_shim_gpu.so

.PHONY: ref shim-check clean
