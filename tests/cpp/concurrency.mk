# TEST INFRASTRUCTURE: builds tests/cpp/_build/dropin_concurrency_check (the drop-in adapters' searches from many reader threads under a
# shared lock, a writer between rounds) with the flags and objects of the Makefile next to it, where the reference tree exists.
include Makefile

.PHONY: concurrency
concurrency: _build/dropin_concurrency_check
_build/dropin_concurrency_check: dropin_concurrency_check.cc $(TOP)/reindexer_b200/host/gpu_bruteforce.h $(TOP)/reindexer_b200/host/gpu_hnsw.h \
  $(TOP)/reindexer_b200/host/gpu_ivf.h $(TOP)/include/rxgpu.h $(OBJ)/hnsw.o
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -fopenmp -DFAISS_WITH_OPENMP=1 -c dropin_concurrency_check.cc -o _build/dropin_concurrency_check.o
	$(CXX) -pthread -o $@ _build/dropin_concurrency_check.o $(FAISS_OBJS) $(OBJ)/ref_ivf_facade.o $(OBJ)/hnsw.o $(OBJ)/l2_dist.o \
	  $(OBJ)/ip_dist.o $(OBJ)/normalize.o $(OBJ)/cpucheck.o $(OBJ)/bruteforce.o $(OBJ)/ref_shim.o -L$(TOP)/reindexer_b200 -lrxgpu \
	  -L$(TOP)/oracle -loracle_port -l:libgomp.so.1 -Wl,-rpath,'$$ORIGIN/../../../reindexer_b200' -Wl,-rpath,'$$ORIGIN/../../../oracle'
