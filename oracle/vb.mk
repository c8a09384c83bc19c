# TEST INFRASTRUCTURE ONLY. Builds
#   _ref/libref_vb.so   the UNMODIFIED reference variational Bayes header (core/models/genotype/variational_bayes_mixture_model.hpp)
#                       with its real utils/maths.hpp and lib/fmath.hpp, behind ref_vb_driver.cpp; compiled from the octopus
#                       checkout REF (-O2, no -ffast-math; -DNDEBUG as a release build; SSE2 on, so fast_exp / fast_log are fmath's).
#                       Headers resolve to ref_shim_vb/ first, then the checkout, then ref_shim/ (boost/optional.hpp).
#                       Usage: make -f vb.mk REF=<checkout>
REF ?=
CXX ?= g++

_ref/libref_vb.so: ref_vb_driver.cpp $(wildcard ref_shim_vb/*/*.hpp ref_shim_vb/*/*/*.hpp ref_shim_vb/*/*/*/*.hpp ref_shim_vb/*/*.h)
	@mkdir -p _ref
	$(CXX) -std=c++17 -O2 -DNDEBUG -fPIC -shared -pthread -msse4.1 -Wno-ignored-attributes \
	    -Iref_shim_vb -I$(REF)/src -I$(REF)/lib -Iref_shim -o $@ ref_vb_driver.cpp

.PHONY: clean
clean:
	rm -f _ref/libref_vb.so
