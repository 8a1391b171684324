# oracle/ref_shim/spgp_grad.mk — the SPGP candidate-gradient drop-in test, built from the reference's OWN headers (REF = the src/
# directory of a resibots/limbo checkout; __graft_entry__.build() passes it) against the Eigen stand-in extended for spgp.hpp:
#     make -C oracle/ref_shim -f spgp_grad.mk REF=... spgp_grad_dropin
# Output (git-ignored): oracle/_ref/spgp_grad_dropin_test, tests/cpp/spgp_grad_dropin_test.cpp: limbo_b200::acqui::UCB / EI over
# limbo_b200::model::SPGP under BatchedRandom's and BatchedGradient's requests, against the reference's experimental::model::SPGP
# (run by tests/test_gpu_spgp_grad.py; needs limbo_b200/lib/liblimbo_b200.so).  Compiles against spgp_eigen/ before ./Eigen, as
# spgp.mk's spgp_dropin_test does.
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
SPGP_GRAD_DROPIN := ../_ref/spgp_grad_dropin_test

spgp_grad_dropin: $(SPGP_GRAD_DROPIN)

$(SPGP_GRAD_DROPIN): $(ROOT)/tests/cpp/spgp_grad_dropin_test.cpp $(ROOT)/include/limbo_b200/model/spgp.hpp $(ROOT)/include/limbo_b200/model/mean_traits.hpp $(ROOT)/include/limbo_b200/opt/batched_gradient.hpp $(ROOT)/include/limbo_b200/opt/batched_random.hpp $(ROOT)/include/limbo_b200.h spgp_eigen/Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -DNDEBUG -ffp-contract=off -Ispgp_eigen -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/spgp_grad_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib' -pthread

.PHONY: spgp_grad_dropin
