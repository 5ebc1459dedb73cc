# The covisibility checker (test infrastructure): make -C oracle -f covis.mk [ref | shim-check]
#   libcovis_oracle.so        our restatement of UpdateConnections' counter and orders over the flat arrays (covis_oracle.cpp)
#   _ref/libcovis_shim.so     shim/KeyFrameConnections_shim.cpp on the stand-in KeyFrame / MapPoint of ref_stub_cv/, next to a literal
#                             restatement of the reference body and the members it calls (ref_covis_wrap.cpp); the device entry point
#                             ccm_covisibility doubled on the CPU by the oracle (ccm_covis_double.cpp), ccm_covisibility_host from
#                             libccm_b200.so
#   _ref/libcovis_shim_gpu.so the same over the real device entry point (GPU suite)
# None of them reads the reference tree.  Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off
REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_cv -Iref_stub_mp -Iref_stub -I../include
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_covis_wrap.cpp ../shim/KeyFrameConnections_shim.cpp

libcovis_oracle.so: covis_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ covis_oracle.cpp

SHIM_DEPS = $(SHIM_SRCS) ../shim/KeyFrameConnections_shim.h ../include/ccm_b200.h ref_stub_cv/cslam/KeyFrame.h $(PRODUCT)/libccm_b200.so

_ref/libcovis_shim.so: $(SHIM_DEPS) ccm_covis_double.cpp libcovis_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_covis_double.cpp -L. -lcovis_oracle -L$(PRODUCT) -lccm_b200 \
	    -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libcovis_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libcovis_shim.so _ref/libcovis_shim_gpu.so,)
ref: libcovis_oracle.so $(SHIM_LIBS)

# type-check the shim against the stand-in KeyFrame (each member cites the cslam/KeyFrame.h line it mirrors)
shim-check:
	$(REF_CXX) -std=c++14 -fsyntax-only -w $(STUB) ../shim/KeyFrameConnections_shim.cpp

clean:
	rm -f libcovis_oracle.so _ref/libcovis_shim.so _ref/libcovis_shim_gpu.so

.PHONY: ref shim-check clean
