# The map-point normal checker (test infrastructure): make -C oracle -f normal_depth.mk [ref | shim-check]
#   libnormal_depth_oracle.so        our restatement of MapPoint::UpdateNormalAndDepth over the flat arrays (normal_depth_oracle.cpp)
#   _ref/libnormal_depth_shim.so     shim/MapPoint_shim.cpp on the stand-in MapPoint / KeyFrame of ref_stub_mp/, next to a literal
#                                    restatement of the reference body (ref_normal_depth_wrap.cpp); the device entry point
#                                    ccm_normal_depth doubled on the CPU by the oracle (ccm_normal_depth_double.cpp),
#                                    ccm_normal_depth_host from libccm_b200.so
#   _ref/libnormal_depth_shim_gpu.so the same over the real device entry point (GPU suite)
#   _ref/liboptimizer_nd_shim.so     shim/Optimizer_shim.cpp AND shim/MapPoint_shim.cpp in one library, against the reference's own
#                                    cslam/Optimizer.h / Converter.cc and the stand-ins of ref_stub_opt_mp, driven by the unchanged
#                                    ref_optimizer_wrap.cpp; ref_optimizer_nd_wrap.cpp reads the normals each write-back leaves.  Device
#                                    entry points doubled on the CPU (ccm_device_double.cpp + ccm_normal_depth_double.cpp)
#   _ref/liboptimizer_nd_shim_gpu.so the same over the real device entry points (GPU suite)
# The first three do not read the reference tree: the stand-ins replace cslam/MapPoint.h, whose own includes (ROS messages, cereal, the
# communicator) do not build here.  The optimiser pair needs the reference tree and liboracle.so (pyoracle.build()).  Shim libraries are
# built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off
REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
PRODUCT ?= ../ccm_slam_b200
STUB = -Iref_stub_mp -Iref_stub -I../include
SHIM_FLAGS = -O2 -fPIC -std=c++11 -fno-fast-math -ffp-contract=off -w -pthread -shared

libnormal_depth_oracle.so: normal_depth_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ normal_depth_oracle.cpp

SHIM_DEPS = ref_normal_depth_wrap.cpp ../shim/MapPoint_shim.cpp ../shim/MapPoint_shim.h ../include/ccm_b200.h ref_stub_mp/cslam/MapPoint.h \
            ref_stub_mp/opencv_matexpr.h $(PRODUCT)/libccm_b200.so

_ref/libnormal_depth_shim.so: $(SHIM_DEPS) ccm_normal_depth_double.cpp libnormal_depth_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) -Wl,-Bsymbolic $(STUB) -o $@ ref_normal_depth_wrap.cpp ../shim/MapPoint_shim.cpp ccm_normal_depth_double.cpp \
	    -L. -lnormal_depth_oracle -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libnormal_depth_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(SHIM_FLAGS) $(STUB) -o $@ ref_normal_depth_wrap.cpp ../shim/MapPoint_shim.cpp \
	    -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

CSLAM ?= /root/reference/cslam
G2O ?= $(CSLAM)/thirdparty/g2o
OPT_FLAGS = -O2 -fPIC -std=c++11 -DCCM_SHIM_BUILD -w -pthread -shared -I. -Iref_stub_opt_mp -Iref_stub -I$(CSLAM)/include -I$(CSLAM) \
            -I$(G2O)/g2o -I../include -include ref_stub_opt/optimizer_prelude.h
OPT_SRCS = ref_optimizer_wrap.cpp ref_optimizer_nd_wrap.cpp ../shim/Optimizer_shim.cpp ../shim/MapPoint_shim.cpp $(CSLAM)/src/Converter.cc
OPT_DEPS = ref_optimizer_wrap.cpp ref_optimizer_nd_wrap.cpp ../shim/Optimizer_shim.cpp ../shim/MapPoint_shim.cpp ../shim/MapPoint_shim.h \
           ../include/ccm_b200.h ref_stub_opt_mp/cslam/Frame.h ref_stub_opt/optimizer_prelude.h $(PRODUCT)/libccm_b200.so

_ref/liboptimizer_nd_shim.so: $(OPT_DEPS) ccm_device_double.cpp ccm_normal_depth_double.cpp libnormal_depth_oracle.so
	mkdir -p _ref
	$(REF_CXX) $(OPT_FLAGS) -Wl,-Bsymbolic -o $@ $(OPT_SRCS) ccm_device_double.cpp ccm_normal_depth_double.cpp \
	    -L. -loracle -lnormal_depth_oracle -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200'

_ref/liboptimizer_nd_shim_gpu.so: $(OPT_DEPS)
	mkdir -p _ref
	$(REF_CXX) $(OPT_FLAGS) -o $@ $(OPT_SRCS) -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200'

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libnormal_depth_shim.so _ref/libnormal_depth_shim_gpu.so,)
OPT_LIBS = $(if $(and $(wildcard $(PRODUCT)/libccm_b200.so),$(wildcard $(CSLAM)/src/Converter.cc),$(wildcard liboracle.so)),_ref/liboptimizer_nd_shim.so _ref/liboptimizer_nd_shim_gpu.so,)
ref: libnormal_depth_oracle.so $(SHIM_LIBS) $(OPT_LIBS)

# type-check the shim against the stand-in MapPoint (each member cites the cslam/MapPoint.h line it mirrors), and, where the reference
# tree is present, against the optimiser-side stand-ins it is linked with next to Optimizer_shim.cpp
shim-check:
	$(REF_CXX) -std=c++11 -fsyntax-only -w $(STUB) ../shim/MapPoint_shim.cpp
	$(if $(wildcard $(CSLAM)/include/cslam/estd.h),$(REF_CXX) -std=c++11 -fsyntax-only -w $(OPT_FLAGS:-shared=) ../shim/MapPoint_shim.cpp,)

clean:
	rm -f libnormal_depth_oracle.so _ref/libnormal_depth_shim.so _ref/libnormal_depth_shim_gpu.so _ref/liboptimizer_nd_shim.so \
	      _ref/liboptimizer_nd_shim_gpu.so

.PHONY: ref shim-check clean
