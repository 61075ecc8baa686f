# TEST INFRASTRUCTURE: builds tests/cpp/_build/dropin_hnsw_build_check (GpuHnsw<OnInsertions> with device building: concurrent inserts
# staged and built by rxgpu_hnsw_build) with the flags and objects of the Makefile next to it, where /root/reference exists.
include Makefile

.PHONY: hnsw_build
hnsw_build: _build/dropin_hnsw_build_check
_build/dropin_hnsw_build_check: dropin_hnsw_build_check.cc $(TOP)/reindexer_b200/host/gpu_hnsw.h $(TOP)/include/rxgpu.h $(OBJ)/hnsw.o
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -o $@ dropin_hnsw_build_check.cc $(OBJ)/hnsw.o $(OBJ)/l2_dist.o $(OBJ)/ip_dist.o $(OBJ)/normalize.o $(OBJ)/cpucheck.o \
	  $(OBJ)/ref_shim.o -L$(TOP)/reindexer_b200 -lrxgpu -L$(TOP)/oracle -loracle_port \
	  -Wl,-rpath,'$$ORIGIN/../../../reindexer_b200' -Wl,-rpath,'$$ORIGIN/../../../oracle'
