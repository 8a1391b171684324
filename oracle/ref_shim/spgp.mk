# oracle/ref_shim/spgp.mk — SPGP test binaries built from the reference's OWN headers (REF = the src/ directory of a
# resibots/limbo checkout; __graft_entry__.build() passes it) against the Eigen stand-in extended for spgp.hpp:
#     make -C oracle/ref_shim -f spgp.mk REF=... all spgp_dropin
# Outputs (git-ignored) under oracle/_ref/:
#   libref_spgp.so     spgp_driver.cpp: the reference's experimental::model::SPGP _likelihood, _compute and _predict behind a C
#                      entry (oracle/ref_spgp.py, tests/golden/make_golden_spgp.py, tests/test_spgp_host.py)
#   spgp_dropin_test   tests/cpp/spgp_dropin_test.cpp: the reference's SPGP next to limbo_b200::model::SPGP
#                      (run by tests/test_gpu_spgp.py; needs limbo_b200/lib/liblimbo_b200.so)
# Both compile against spgp_eigen/ (the stand-in plus the members spgp.hpp needs) before ./Eigen.
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
OUT := ../_ref/libref_spgp.so
SPGP_DROPIN := ../_ref/spgp_dropin_test
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fno-fast-math -ffp-contract=off -DNDEBUG -w

all: $(OUT)

$(OUT): spgp_driver.cpp spgp_eigen/Eigen/Core boost/optional.hpp
	mkdir -p ../_ref
	$(CXX) $(CXXFLAGS) -Ispgp_eigen -I. -I$(REF) -shared -o $@ spgp_driver.cpp -pthread

spgp_dropin: $(SPGP_DROPIN)

$(SPGP_DROPIN): $(ROOT)/tests/cpp/spgp_dropin_test.cpp $(ROOT)/include/limbo_b200/model/spgp.hpp $(ROOT)/include/limbo_b200.h spgp_eigen/Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -DNDEBUG -ffp-contract=off -Ispgp_eigen -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/spgp_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib' -pthread

.PHONY: all spgp_dropin
