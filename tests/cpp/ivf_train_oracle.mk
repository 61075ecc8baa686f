# TEST INFRASTRUCTURE: builds tests/cpp/_build/libivf_train_oracle.so (FAISS's IVF k-means as IvfIndex::trainIdx runs it) against the
# reference's vendored FAISS in oracle/_ref/liboracle_ref_ivf.so, where /root/reference exists.
include Makefile

.PHONY: ivf_train_oracle
ivf_train_oracle: _build/libivf_train_oracle.so
_build/libivf_train_oracle.so: ivf_train_oracle.cc $(TOP)/oracle/_ref/liboracle_ref_ivf.so
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -fPIC -fopenmp -DFAISS_WITH_OPENMP=1 -c ivf_train_oracle.cc -o _build/ivf_train_oracle.o
	$(CXX) -shared -pthread -o $@ _build/ivf_train_oracle.o -L$(TOP)/oracle/_ref -l:liboracle_ref_ivf.so -l:libgomp.so.1 \
	  -Wl,-rpath,'$$ORIGIN/../../../oracle/_ref'
