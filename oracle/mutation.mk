# TEST INFRASTRUCTURE ONLY. Builds
#   _ref/libref_mutation.so   the UNMODIFIED reference mutation model (indel_mutation_model.cpp, denovo_model.cpp) with the repeat
#                             finder it calls (lib/tandem + libdivsufsort), behind ref_mutation_driver.cpp; compiled from the octopus
#                             checkout REF like _ref/libref_errmodel.so (-O2, no -ffast-math; -DNDEBUG as a release build). Its
#                             headers' dependencies resolve to ref_shim_mutation/, then ref_shim/. Usage: make -f mutation.mk REF=<checkout>
REF ?=
CXX ?= g++
CC  ?= gcc
MUT    = $(REF)/src/core/models/mutation
DIVSUF = $(REF)/lib/tandem/libdivsufsort
REF_MUT_SRCS = $(MUT)/indel_mutation_model.cpp $(MUT)/denovo_model.cpp $(REF)/lib/tandem/tandem.cpp

_ref/libref_mutation.so: ref_mutation_driver.cpp $(wildcard ref_shim_mutation/*/*.hpp ref_shim_mutation/*/*/*.hpp ref_shim/*/*.hpp ref_shim/*/*/*.hpp)
	@mkdir -p _ref/obj_mutation
	for f in divsufsort sssort trsort utils; do $(CC) -O2 -fPIC -DHAVE_CONFIG_H -I$(DIVSUF) -c $(DIVSUF)/$$f.c -o _ref/obj_mutation/$$f.o || exit 1; done
	$(CXX) -std=c++17 -O2 -DNDEBUG -fPIC -shared -pthread -msse4.1 -include immintrin.h -include iterator -Wno-ignored-attributes \
	    -Iref_shim_mutation -Iref_shim -I$(REF)/src -I$(REF)/lib -I$(DIVSUF) -o $@ ref_mutation_driver.cpp $(REF_MUT_SRCS) \
	    _ref/obj_mutation/divsufsort.o _ref/obj_mutation/sssort.o _ref/obj_mutation/trsort.o _ref/obj_mutation/utils.o

.PHONY: clean
clean:
	rm -rf _ref/libref_mutation.so _ref/obj_mutation
