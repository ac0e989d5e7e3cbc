# Compiles the reference's native code into _ref/ (test infrastructure only): the
# birth-death-mutation simulator elfi/examples/cpp/bdm.cpp of the checkout named by
# ELFI_REFERENCE_ROOT, the oracle of tests/test_bdm_host.py and tests/golden/gen_golden_bdm.py.
# Nothing from the reference is copied into this repository.  Without that checkout there is
# nothing to build, and a _ref/bdm built elsewhere is left as it is.
#
#     ELFI_REFERENCE_ROOT=<reference checkout> make -C oracle -f ref_bins.mk
CXX ?= g++

BDM_SRC := $(if $(ELFI_REFERENCE_ROOT),$(wildcard $(ELFI_REFERENCE_ROOT)/elfi/examples/cpp/bdm.cpp))

ifneq ($(BDM_SRC),)
all: _ref/bdm
else
all:
endif

_ref/bdm: $(BDM_SRC)
	mkdir -p _ref
	$(CXX) -std=c++11 -O2 -o $@ $<

.PHONY: all
