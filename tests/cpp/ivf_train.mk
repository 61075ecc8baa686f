# TEST INFRASTRUCTURE: builds tests/cpp/_build/dropin_ivf_train_check (IvfIndex's training upsert and RebuildCentroids through
# GpuIvfMap::TrainAndFill) with the flags and objects of the Makefile next to it, where /root/reference (headers + oracle/_ref objects) exists.
include Makefile

.PHONY: ivf_train
ivf_train: _build/dropin_ivf_train_check
_build/dropin_ivf_train_check: dropin_ivf_train_check.cc $(TOP)/reindexer_b200/host/gpu_ivf.h $(TOP)/include/rxgpu.h
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -fopenmp -DFAISS_WITH_OPENMP=1 -c dropin_ivf_train_check.cc -o _build/dropin_ivf_train_check.o
	$(CXX) -pthread -o $@ _build/dropin_ivf_train_check.o $(FAISS_OBJS) $(OBJ)/ref_ivf_facade.o $(OBJ)/l2_dist.o $(OBJ)/ip_dist.o \
	  $(OBJ)/normalize.o $(OBJ)/cpucheck.o $(OBJ)/bruteforce.o $(OBJ)/ref_shim.o -L$(TOP)/reindexer_b200 -lrxgpu -l:libgomp.so.1 \
	  -Wl,-rpath,'$$ORIGIN/../../../reindexer_b200'
