# TEST INFRASTRUCTURE. DO_LIGHT_SAMPLING 0 (Config.h:24) builds of the oracles, next to what Makefile builds:
#   _ref/libtoyref_nolight.so               the reference with DO_LIGHT_SAMPLING 0 (46 spheres); only if $(REF) exists
#   _ref/libtoyref_small_mitsuba_nolight.so the same with DO_BIG_SCENE 0 and DO_MITSUBA_COMPARE 1
#   _ref/liboracle_nolight.so               the CPU restatement (restate.cpp) with the switch off
#   _ref/librefgpu_nolight.so               the restatement of the GPU shader (refgpu_restate.cpp) with the switch off
# Usage: make -C oracle -f nolight.mk all
# Every variant is compiled from an edited COPY in a mktemp directory that is deleted afterwards (the pattern of
# Makefile's build_variant); only the .so lands in _ref/. The edits mirror the reference's two `#if DO_LIGHT_SAMPLING`
# blocks: the light loop of Lambert Scatter (Test.cpp:95-133, ComputeShader.hlsl:200) and the doMaterialE suppression in
# Trace (Test.cpp:209-215, ComputeShader.hlsl:314). Each edit is checked with grep, so a source that no longer matches
# fails the build instead of silently building the stock oracle.
REF ?= /root/reference/Cpp/Source
CXX ?= g++
FLAGS = -O2 -std=c++11 -msse4.1 -ffp-contract=off -DNDEBUG -w -fPIC

all: _ref/liboracle_nolight.so _ref/librefgpu_nolight.so ref

ref:
	@if [ -d $(REF) ]; then $(MAKE) -f nolight.mk _ref/libtoyref_nolight.so _ref/libtoyref_small_mitsuba_nolight.so; else echo "reference sources absent; using prebuilt _ref/libtoyref*_nolight.so if any"; fi

# $(1) DO_MITSUBA_COMPARE, $(2) DO_BIG_SCENE; DO_LIGHT_SAMPLING is 0
define build_ref_nolight
	mkdir -p _ref
	T=$$(mktemp -d) && cp -r $(REF)/. $$T/ && chmod -R u+w $$T && \
	sed -i 's/^#define DO_MITSUBA_COMPARE 0/#define DO_MITSUBA_COMPARE $(1)/' $$T/Config.h && \
	sed -i 's/^#define DO_BIG_SCENE 1/#define DO_BIG_SCENE $(2)/' $$T/Test.cpp && \
	sed -i 's/^#define DO_LIGHT_SAMPLING 1/#define DO_LIGHT_SAMPLING 0/' $$T/Config.h && \
	grep -q '^#define DO_MITSUBA_COMPARE $(1)' $$T/Config.h && grep -q '^#define DO_BIG_SCENE $(2)' $$T/Test.cpp && \
	grep -q '^#define DO_LIGHT_SAMPLING 0' $$T/Config.h && \
	$(CXX) $(FLAGS) -include string.h -I$$T -shared -o $@ ref_harness.cpp \
	    $$T/Test.cpp $$T/Maths.cpp $$T/enkiTS/TaskScheduler.cpp $$T/enkiTS/TaskScheduler_c.cpp -lpthread; \
	rc=$$?; rm -rf $$T; exit $$rc
endef
_ref/libtoyref_nolight.so: ref_harness.cpp $(REF)/Test.cpp $(REF)/Maths.cpp $(REF)/Config.h
	$(call build_ref_nolight,0,1)
_ref/libtoyref_small_mitsuba_nolight.so: ref_harness.cpp $(REF)/Test.cpp $(REF)/Maths.cpp $(REF)/Config.h
	$(call build_ref_nolight,1,0)

# $(1) source, $(2) its emissive-list member: the light loop's condition becomes false, the suppression line goes
define build_restatement_nolight
	mkdir -p _ref
	T=$$(mktemp -d) && cp $(1) $$T/src.cpp && \
	sed -i 's/for (size_t j = 0; j < sc\.$(2)\.size(); ++j)/for (size_t j = 0; false \&\& j < sc.$(2).size(); ++j)/' $$T/src.cpp && \
	sed -i '/^ *if (!doMaterialE) matE = mk(0, 0, 0);$$/d' $$T/src.cpp && \
	test $$(grep -c 'false && j < sc\.$(2)\.size()' $$T/src.cpp) -eq 1 && ! grep -q 'if (!doMaterialE)' $$T/src.cpp && \
	$(CXX) $(FLAGS) -shared -o $@ $$T/src.cpp -lpthread -lm; \
	rc=$$?; rm -rf $$T; exit $$rc
endef
_ref/liboracle_nolight.so: restate.cpp
	$(call build_restatement_nolight,restate.cpp,emissive)
_ref/librefgpu_nolight.so: refgpu_restate.cpp
	$(call build_restatement_nolight,refgpu_restate.cpp,emissives)
