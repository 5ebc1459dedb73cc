# The keyframe-culling checker (test infrastructure): make -C oracle -f keyframe_culling.mk [ref | shim-check]
#   libkeyframe_culling_oracle.so   our flat restatement of LocalMapping::KeyFrameCullingV3 over the arrays of ccm_keyframe_culling
#                                   (keyframe_culling_oracle.cpp): the candidates walked in order over live keyframe and point state,
#                                   with the deliberately wrong readings the tests tell apart.  Shares nothing with the product but the
#                                   C declarations of include/ccm_b200.h, and does not read the reference tree.
#   _ref/libkeyframe_culling_shim.so      shim/KeyFrameCulling_shim.cpp on the stand-in LocalMapping / KeyFrame / MapPoint / Map of
#                                         ref_stub_kc/, next to a literal restatement of the member and of the SetBadFlag /
#                                         EraseObservation paths it reaches (ref_keyframe_culling_wrap.cpp); the device entry point answered
#                                         by the host entry point (ccm_keyframe_culling_double.cpp)
#   _ref/libkeyframe_culling_shim_gpu.so  the same over the real device entry point (GPU suite)
# Shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off

libkeyframe_culling_oracle.so: keyframe_culling_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ keyframe_culling_oracle.cpp -Wl,--no-undefined

REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_kc -Iref_stub_mp -Iref_stub -I../include -I../shim
SHIM_FLAGS = -O2 -fPIC -std=c++14 -fno-fast-math -ffp-contract=off -w -pthread -shared
SHIM_SRCS = ref_keyframe_culling_wrap.cpp ../shim/KeyFrameCulling_shim.cpp
SHIM_DEPS = $(SHIM_SRCS) ../shim/KeyFrameCulling_shim.h ../include/ccm_b200.h ref_stub_kc/cslam/Mapping.h ref_stub_kc/cslam/KeyFrame.h \
            ref_stub_kc/cslam/MapPoint.h ref_stub_kc/cslam/Map.h $(PRODUCT)/libccm_b200.so

_ref/libkeyframe_culling_shim.so: $(SHIM_DEPS) ccm_keyframe_culling_double.cpp
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ $(SHIM_SRCS) ccm_keyframe_culling_double.cpp -L$(PRODUCT) -lccm_b200 \
	    -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libkeyframe_culling_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ $(SHIM_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libkeyframe_culling_shim.so _ref/libkeyframe_culling_shim_gpu.so,)

# type-check the shim against the stand-ins (each member cites the line of the real header it mirrors)
shim-check:
	$(REF_CXX) -std=c++14 -fsyntax-only -w $(STUB) ../shim/KeyFrameCulling_shim.cpp

ref: libkeyframe_culling_oracle.so $(SHIM_LIBS)

clean:
	rm -f libkeyframe_culling_oracle.so _ref/libkeyframe_culling_shim.so _ref/libkeyframe_culling_shim_gpu.so

.PHONY: ref shim-check clean
