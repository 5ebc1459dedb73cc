# The keyframe-database checker (test infrastructure): make -C oracle -f kfdb.mk [ref]
#   libkfdb_oracle.so    our restatement of S/Database.cpp's queries and DBoW2's scores (kfdb_oracle.cpp)
#   _ref/libkfdb_ref.so  THE REFERENCE'S OWN cslam/src/Database.cpp and DBoW2 ScoringObject.cpp / BowVector.cpp, compiled where they
#                        lie (nothing is copied) against the stand-in KeyFrame / Map / Frame / MapPoint of ref_stub_db/ and driven by
#                        ref_kfdb_wrap.cpp through the same C interface as the oracle
#   _ref/libkfdb_shim.so      this repository's shim/Database_shim.cpp in place of Database.cpp, same stand-ins, same wrapper; the
#                             device entry points doubled on the CPU by ccm_kfdb_double.cpp (the oracle's scores), ccm_kfdb_select
#                             from libccm_b200.so
#   _ref/libkfdb_shim_gpu.so  the same over the real device entry points (GPU suite)
# The shim libraries are built only where the product library exists (it needs nvcc).
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -fPIC -std=c++17 -Wall -Wextra -fno-fast-math -ffp-contract=off
REF_CXX ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)
CSLAM ?= /root/reference/cslam
DBOW2 = $(CSLAM)/thirdparty/DBoW2

libkfdb_oracle.so: kfdb_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ kfdb_oracle.cpp

_ref/libkfdb_ref.so: ref_kfdb_wrap.cpp ref_stub_db/cslam/KeyFrame.h
	mkdir -p _ref
	$(REF_CXX) -O2 -fPIC -std=c++11 -w -pthread -shared -Iref_stub_db -Iref_stub -I$(CSLAM)/include -I$(CSLAM) -I$(DBOW2) -o $@ \
	    ref_kfdb_wrap.cpp $(CSLAM)/src/Database.cpp $(DBOW2)/DBoW2/ScoringObject.cpp $(DBOW2)/DBoW2/BowVector.cpp \
	    $(DBOW2)/DBoW2/FeatureVector.cpp $(DBOW2)/DBoW2/FORB.cpp $(DBOW2)/DUtils/Random.cpp $(DBOW2)/DUtils/Timestamp.cpp -Wl,--no-undefined

PRODUCT ?= ../ccm_slam_b200
DBOW2_SRCS = $(DBOW2)/DBoW2/ScoringObject.cpp $(DBOW2)/DBoW2/BowVector.cpp $(DBOW2)/DBoW2/FeatureVector.cpp $(DBOW2)/DBoW2/FORB.cpp \
             $(DBOW2)/DUtils/Random.cpp $(DBOW2)/DUtils/Timestamp.cpp
SHIM_DEPS = ref_kfdb_wrap.cpp ../shim/Database_shim.cpp ../include/ccm_b200.h ref_stub_db/cslam/KeyFrame.h $(PRODUCT)/libccm_b200.so

_ref/libkfdb_shim.so: $(SHIM_DEPS) ccm_kfdb_double.cpp libkfdb_oracle.so
	mkdir -p _ref
	$(REF_CXX) -O2 -fPIC -std=c++11 -w -pthread -shared -Wl,-Bsymbolic -Iref_stub_db -Iref_stub -I$(CSLAM)/include -I$(CSLAM) -I$(DBOW2) \
	    -I../include -o $@ ref_kfdb_wrap.cpp ../shim/Database_shim.cpp ccm_kfdb_double.cpp $(DBOW2_SRCS) \
	    -L. -lkfdb_oracle -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/..' -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

_ref/libkfdb_shim_gpu.so: $(SHIM_DEPS)
	mkdir -p _ref
	$(REF_CXX) -O2 -fPIC -std=c++11 -w -pthread -shared -Iref_stub_db -Iref_stub -I$(CSLAM)/include -I$(CSLAM) -I$(DBOW2) \
	    -I../include -o $@ ref_kfdb_wrap.cpp ../shim/Database_shim.cpp $(DBOW2_SRCS) \
	    -L$(PRODUCT) -lccm_b200 -Wl,-rpath,'$$ORIGIN/../../ccm_slam_b200' -Wl,--no-undefined

SHIM_LIBS = $(if $(wildcard $(PRODUCT)/libccm_b200.so),_ref/libkfdb_shim.so _ref/libkfdb_shim_gpu.so,)
ref: _ref/libkfdb_ref.so $(SHIM_LIBS)

# type-check the shim against the reference's own cslam/Database.h
shim-check:
	$(REF_CXX) -std=c++11 -fsyntax-only -w -Iref_stub_db -Iref_stub -I$(CSLAM)/include -I$(CSLAM) -I$(DBOW2) -I../include ../shim/Database_shim.cpp

clean:
	rm -f libkfdb_oracle.so _ref/libkfdb_ref.so _ref/libkfdb_shim.so _ref/libkfdb_shim_gpu.so

.PHONY: ref shim-check clean
