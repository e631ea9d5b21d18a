# ORACLE build (test infrastructure) for SearchForInitialization. Three libraries:
#   liboracle_init.so       the oracle's restatement (init_search.h, entries init_search_oracle.cpp); needs only a C++ compiler.
#   _ref/libref_init.so     the reference's own objects of libref.so (./Makefile's recipe, unchanged) with ref_scene.cpp and init_search_ref_api.cpp:
#                           the reference's SearchForInitialization and GetFeaturesInArea on Frames of given key points. No GPU library.
#   _ref/libdropin_init.so  libdropin.so's ingredients (./Makefile, with the drop-in header dependency of large_kf_dropin.mk, both unchanged),
#                           except that the reference's src/ORBMatcher.cpp and dropin/ORBMatcher_cpu_forward.cpp are compiled again with
#                           SearchForInitialization renamed away too, plus the drop-in dropin/ORBMatcher_init_b200.cpp and the harness
#                           init_search_api.cpp: the drop-in and the reference's CPU body on the same reference Frames.
# Built by __graft_entry__.build(): liboracle_init.so always, the two _ref libraries where the reference tree exists:
#   make -C oracle -f init_search_dropin.mk liboracle_init.so _ref/libref_init.so _ref/libdropin_init.so
include large_kf_dropin.mk

liboracle_init.so: init_search_oracle.cpp init_search.h frame_index.h orb_extractor.h orb_matcher.h cvprim.h init_search_dropin.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ init_search_oracle.cpp

INIT_RENAME := $(RENAME) -DSearchForInitialization=SearchForInitialization_cpu
INIT_REPLACED := _ref/obj_dropin/ORBMatcher_cpu.o _ref/obj_dropin/ORBMatcher_cpu_forward.o
INIT_OBJ := $(filter-out $(INIT_REPLACED),$(DROPIN_OBJ)) _ref/obj_init/ORBMatcher_cpu.o _ref/obj_init/ORBMatcher_cpu_forward.o _ref/obj_init/ORBMatcher_init_b200.o \
            _ref/obj_init/init_search_api.o

_ref/obj_init/ORBMatcher_cpu.o: $(REF)/src/ORBMatcher.cpp cvshim/cvshim.h init_search_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_init
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) $(INIT_RENAME) -c $< -o $@
_ref/obj_init/ORBMatcher_cpu_forward.o: ../dropin/ORBMatcher_cpu_forward.cpp cvshim/cvshim.h init_search_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_init
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) $(INIT_RENAME) -c $< -o $@
_ref/obj_init/ORBMatcher_init_b200.o: ../dropin/ORBMatcher_init_b200.cpp ../include/cubemap_b200.h cvshim/cvshim.h init_search_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_init
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -I../include -c $< -o $@
_ref/obj_init/%.o: %.cpp ref_scene.h cvshim/cvshim.h init_search_dropin.mk $(REF_STAMP)
	@mkdir -p _ref/obj_init
	$(REFCXX) $(REF_FLAGS) -ffp-contract=off $(REF_INC) -c $< -o $@

_ref/libref_init.so: $(REF_OBJ) _ref/obj/ref_scene.o _ref/obj_init/init_search_ref_api.o
	$(REFCXX) -shared -pthread -Wl,-Bsymbolic -o $@ $^ -ldl
_ref/libdropin_init.so: $(INIT_OBJ) ../cubemapslam_b200/libcubemap_b200.so
	$(REFCXX) -shared -pthread -o $@ $(INIT_OBJ) -L../cubemapslam_b200 -lcubemap_b200 -Wl,-rpath,'$$ORIGIN/../../cubemapslam_b200' -ldl
