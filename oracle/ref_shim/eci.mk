# oracle/ref_shim/eci.mk — constrained-BO test binaries built from the reference's OWN headers (REF = the src/ directory of a
# resibots/limbo checkout; __graft_entry__.build() passes it) against the Eigen/Boost stand-in in this directory:
#     make -C oracle/ref_shim -f eci.mk REF=... all eci_dropin
# Outputs (git-ignored) under oracle/_ref/:
#   libref_eci.so    eci_driver.cpp: the reference's experimental::acqui::ECI behind a C entry (oracle/ref_eci.py,
#                    tests/golden/make_golden_eci.py, tests/test_eci_host.py)
#   eci_dropin_test  tests/cpp/eci_dropin_test.cpp: the reference's ECI over limbo_b200::model::GP pairs and limbo_b200::acqui::ECI
#                    (run by tests/test_gpu_eci.py; needs limbo_b200/lib/liblimbo_b200.so)
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
OUT := ../_ref/libref_eci.so
ECI_DROPIN := ../_ref/eci_dropin_test
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fno-fast-math -ffp-contract=off -DNDEBUG -w

all: $(OUT)

$(OUT): eci_driver.cpp Eigen/Core boost/optional.hpp
	mkdir -p ../_ref
	$(CXX) $(CXXFLAGS) -I. -I$(REF) -shared -o $@ eci_driver.cpp -pthread

eci_dropin: $(ECI_DROPIN)

$(ECI_DROPIN): $(ROOT)/tests/cpp/eci_dropin_test.cpp $(ROOT)/include/limbo_b200/opt/batched_random.hpp $(ROOT)/include/limbo_b200/model/gp.hpp $(ROOT)/include/limbo_b200.h Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -DNDEBUG -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/eci_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib'

.PHONY: all eci_dropin
