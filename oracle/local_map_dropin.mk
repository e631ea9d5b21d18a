# ORACLE build (test infrastructure): oracle/_ref/libdropin_local_map.so = oracle/_ref/libdropin.so's ingredients (the recipe of ./Makefile, with
# the drop-in header dependency of large_kf_dropin.mk, both included unchanged) plus the harness local_map_api.cpp: the local-map
# SearchByProjection on reference objects, through the drop-in and through the reference's CPU body. Built by __graft_entry__.build() where the
# reference tree exists:  make -C oracle -f local_map_dropin.mk _ref/libdropin_local_map.so
include large_kf_dropin.mk

LOCAL_MAP_OBJ := $(DROPIN_OBJ) _ref/obj_local_map/local_map_api.o

_ref/obj_local_map/local_map_api.o: local_map_api.cpp ref_scene.h cvshim/cvshim.h local_map_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_local_map
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -c $< -o $@
_ref/libdropin_local_map.so: $(LOCAL_MAP_OBJ) ../cubemapslam_b200/libcubemap_b200.so
	$(REFCXX) -shared -pthread -o $@ $(LOCAL_MAP_OBJ) -L../cubemapslam_b200 -lcubemap_b200 -Wl,-rpath,'$$ORIGIN/../../cubemapslam_b200' -ldl
