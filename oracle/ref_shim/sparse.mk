# oracle/ref_shim/sparse.mk — sparsification test binaries built from the reference's OWN headers (REF = the src/ directory of a
# resibots/limbo checkout; __graft_entry__.build() passes it) against the Eigen/Boost stand-in in this directory:
#     make -C oracle/ref_shim -f sparse.mk REF=... all sparse_dropin
# Outputs (git-ignored) under oracle/_ref/:
#   libref_sparse.so     sparse_driver.cpp: the reference's model::SparsifiedGP::_sparsify behind a C entry (oracle/ref_sparse.py,
#                        tests/golden/make_golden_sparsify.py, tests/test_sparsify_host.py)
#   sparse_dropin_test   tests/cpp/sparsified_dropin_test.cpp: the reference's SparsifiedGP next to limbo_b200::model::SparsifiedGP
#                        (run by tests/test_gpu_sparsify.py; needs limbo_b200/lib/liblimbo_b200.so)
# Both compile against sparse_eigen/ (the stand-in plus the writable VectorXd::Map that sparsified_gp.hpp needs) before ./Eigen.
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
OUT := ../_ref/libref_sparse.so
SPARSE_DROPIN := ../_ref/sparse_dropin_test
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -fno-fast-math -ffp-contract=off -DNDEBUG -w

all: $(OUT)

$(OUT): sparse_driver.cpp sparse_eigen/Eigen/Core Eigen/Core boost/optional.hpp
	mkdir -p ../_ref
	$(CXX) $(CXXFLAGS) -Isparse_eigen -I. -I$(REF) -shared -o $@ sparse_driver.cpp -pthread

sparse_dropin: $(SPARSE_DROPIN)

$(SPARSE_DROPIN): $(ROOT)/tests/cpp/sparsified_dropin_test.cpp $(ROOT)/include/limbo_b200/model/sparsified_gp.hpp $(ROOT)/include/limbo_b200/model/gp.hpp $(ROOT)/include/limbo_b200.h sparse_eigen/Eigen/Core Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -DNDEBUG -ffp-contract=off -Isparse_eigen -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/sparsified_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib' -pthread

.PHONY: all sparse_dropin
