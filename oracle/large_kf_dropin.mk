# ORACLE build (test infrastructure): oracle/_ref/libdropin_large.so = oracle/_ref/libdropin.so's ingredients (the recipe of ./Makefile, included
# here unchanged) plus the harness large_kf_api.cpp: SearchByBoW in both forms on reference objects, through the drop-in and through the
# reference's CPU body. Built by __graft_entry__.build() where the reference tree exists:  make -C oracle -f large_kf_dropin.mk _ref/libdropin_large.so
include Makefile

LARGE_OBJ := $(DROPIN_OBJ) _ref/obj_large/large_kf_api.o

# the drop-ins include ../dropin/FeatureVector_csr_b200.h, which ./Makefile's rule for them does not list
$(filter _ref/obj_dropin/%_b200.o,$(DROPIN_OBJ)): ../dropin/FeatureVector_csr_b200.h

_ref/obj_large/large_kf_api.o: large_kf_api.cpp ref_scene.h cvshim/cvshim.h large_kf_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_large
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -c $< -o $@
_ref/libdropin_large.so: $(LARGE_OBJ) ../cubemapslam_b200/libcubemap_b200.so
	$(REFCXX) -shared -pthread -o $@ $(LARGE_OBJ) -L../cubemapslam_b200 -lcubemap_b200 -Wl,-rpath,'$$ORIGIN/../../cubemapslam_b200' -ldl
