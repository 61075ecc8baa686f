# TEST INFRASTRUCTURE: builds tests/cpp/_build/dropin_ft_areas_check (the highlight-area side of the ft_fast adapter) with the flags
# and objects of the Makefile next to it, where /root/reference (headers + oracle/_ref objects) exists.
include Makefile

.PHONY: areas
areas: _build/dropin_ft_areas_check
_build/dropin_ft_areas_check: dropin_ft_areas_check.cc dropin_ft_check.cc $(TOP)/reindexer_b200/host/gpu_ft_merge.h $(TOP)/include/rxgpu.h
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -o $@ dropin_ft_areas_check.cc $(OBJ)/idrelset.o $(OBJ)/ref_shim_ft.o -L$(TOP)/reindexer_b200 -lrxgpu \
	  -Wl,-rpath,'$$ORIGIN/../../../reindexer_b200'
