# TEST INFRASTRUCTURE ONLY. Builds
#   _ref/libref_vbmm.so  the UNMODIFIED reference core/models/genotype/variational_bayes_mixture_mixture_model.cpp with its real
#                        utils/maths.hpp, behind ref_vbmm_driver.cpp; compiled from the octopus checkout REF (-O2, no
#                        -ffast-math; -DNDEBUG as a release build). Headers resolve as for vb.mk: ref_shim_vb/ first, then the
#                        checkout, then ref_shim/.
#                        Usage: make -f vbmm.mk REF=<checkout>
REF ?=
CXX ?= g++

_ref/libref_vbmm.so: ref_vbmm_driver.cpp $(REF)/src/core/models/genotype/variational_bayes_mixture_mixture_model.cpp \
                     $(wildcard ref_shim_vb/*/*.hpp ref_shim_vb/*/*/*.hpp ref_shim_vb/*/*/*/*.hpp ref_shim_vb/*/*.h)
	@mkdir -p _ref
	$(CXX) -std=c++17 -O2 -DNDEBUG -fPIC -shared -pthread -msse4.1 -Wno-ignored-attributes -Wl,--no-undefined \
	    -Iref_shim_vb -I$(REF)/src -I$(REF)/lib -Iref_shim -o $@ ref_vbmm_driver.cpp \
	    $(REF)/src/core/models/genotype/variational_bayes_mixture_mixture_model.cpp

.PHONY: clean
clean:
	rm -f _ref/libref_vbmm.so
