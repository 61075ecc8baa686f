# TEST INFRASTRUCTURE: builds tests/cpp/_build/dropin_ivf_many_centroids_check (the IVF adapter over 20 000 centroids) with the flags
# and objects of the Makefile next to it, where /root/reference (headers + oracle/_ref objects) exists.
include Makefile

.PHONY: ivf_many_centroids
ivf_many_centroids: _build/dropin_ivf_many_centroids_check
_build/dropin_ivf_many_centroids_check: dropin_ivf_many_centroids_check.cc $(TOP)/reindexer_b200/host/gpu_ivf.h $(TOP)/include/rxgpu.h
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -fopenmp -DFAISS_WITH_OPENMP=1 -c dropin_ivf_many_centroids_check.cc -o _build/dropin_ivf_many_centroids_check.o
	$(CXX) -pthread -o $@ _build/dropin_ivf_many_centroids_check.o $(FAISS_OBJS) $(OBJ)/ref_ivf_facade.o $(OBJ)/l2_dist.o $(OBJ)/ip_dist.o \
	  $(OBJ)/normalize.o $(OBJ)/cpucheck.o $(OBJ)/bruteforce.o $(OBJ)/ref_shim.o -L$(TOP)/reindexer_b200 -lrxgpu -l:libgomp.so.1 \
	  -Wl,-rpath,'$$ORIGIN/../../../reindexer_b200'
