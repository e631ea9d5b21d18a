# ORACLE build (test infrastructure): oracle/_ref/libdropin_bow.so = oracle/_ref/libdropin.so's ingredients (the recipe of ./Makefile, included
# here unchanged) with the reference's own src/Frame.cpp and src/KeyFrame.cpp compiled with ComputeBoW renamed away (INTEGRATION.md §2), plus
# dropin/ComputeBoW_b200.cpp, dropin/ComputeBoW_cpu_forward.cpp and the harness bow_dropin_api.cpp. libdropin.so and libref.so keep the
# unrenamed objects. Built by __graft_entry__.build() where the reference tree exists:  make -C oracle -f bow_dropin.mk _ref/libdropin_bow.so
include Makefile

BOW_RENAME := -DComputeBoW=ComputeBoW_cpu
BOW_OBJ := $(filter-out _ref/obj/Frame.o _ref/obj/KeyFrame.o,$(DROPIN_OBJ)) _ref/obj_bow/Frame_cpu.o _ref/obj_bow/KeyFrame_cpu.o \
           _ref/obj_bow/ComputeBoW_cpu_forward.o _ref/obj_bow/ComputeBoW_b200.o _ref/obj_bow/bow_dropin_api.o

_ref/obj_bow/Frame_cpu.o _ref/obj_bow/KeyFrame_cpu.o: _ref/obj_bow/%_cpu.o: $(REF)/src/%.cpp cvshim/cvshim.h bow_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_bow
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) $(BOW_RENAME) -c $< -o $@
_ref/obj_bow/ComputeBoW_cpu_forward.o: ../dropin/ComputeBoW_cpu_forward.cpp cvshim/cvshim.h bow_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_bow
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) $(BOW_RENAME) -c $< -o $@
_ref/obj_bow/ComputeBoW_b200.o: ../dropin/ComputeBoW_b200.cpp ../include/cubemap_b200.h cvshim/cvshim.h bow_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_bow
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -I../include -c $< -o $@
_ref/obj_bow/bow_dropin_api.o: bow_dropin_api.cpp ref_scene.h cvshim/cvshim.h bow_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_bow
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -c $< -o $@
_ref/libdropin_bow.so: $(BOW_OBJ) ../cubemapslam_b200/libcubemap_b200.so
	$(REFCXX) -shared -pthread -o $@ $(BOW_OBJ) -L../cubemapslam_b200 -lcubemap_b200 -Wl,-rpath,'$$ORIGIN/../../cubemapslam_b200' -ldl
