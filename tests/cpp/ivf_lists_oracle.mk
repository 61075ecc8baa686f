# TEST INFRASTRUCTURE: builds tests/cpp/_build/libivf_lists_oracle.so (FAISS' IndexIVFFlat over given centroids and lists, no k-means)
# against the reference's vendored FAISS in oracle/_ref/liboracle_ref_ivf.so, where /root/reference exists.
include Makefile

.PHONY: ivf_lists_oracle
ivf_lists_oracle: _build/libivf_lists_oracle.so
_build/libivf_lists_oracle.so: ivf_lists_oracle.cc $(TOP)/oracle/_ref/liboracle_ref_ivf.so
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -fPIC -fopenmp -DFAISS_WITH_OPENMP=1 -c ivf_lists_oracle.cc -o _build/ivf_lists_oracle.o
	$(CXX) -shared -pthread -o $@ _build/ivf_lists_oracle.o -L$(TOP)/oracle/_ref -l:liboracle_ref_ivf.so -l:libgomp.so.1 \
	  -Wl,-rpath,'$$ORIGIN/../../../oracle/_ref'
