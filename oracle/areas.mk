# ORACLE / TEST INFRASTRUCTURE ONLY.
#
#   make -f areas.mk ref_areas -> oracle/_ref/liboracle_ref_ft_areas.so: the reference's ft::Merger with MergeDataAreas<Area>
#                                 (ref_ft_areas_facade.cc) on the objects and flags of the Makefile's full-text oracle.
include Makefile

.PHONY: ref_areas
ref_areas: $(OUT)/liboracle_ref_ft_areas.so
$(OUT)/obj/ref_ft_areas_facade.o: ref_ft_areas_facade.cc ref_ft_facade.cc ft_problem.h | $(OUT)/obj
	$(CXX) $(REFFLAGS) -I. -c $< -o $@
$(OUT)/liboracle_ref_ft_areas.so: $(FT_REF_OBJS) $(OUT)/obj/ref_shim_ft.o $(OUT)/obj/ref_ft_areas_facade.o
	$(CXX) -shared -pthread -o $@ $^
