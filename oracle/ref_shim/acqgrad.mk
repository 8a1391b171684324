# oracle/ref_shim/acqgrad.mk — the candidate-gradient drop-in test built against the reference's OWN headers (REF = the src/
# directory of a resibots/limbo checkout; __graft_entry__.build() passes it) and the Eigen/Boost stand-in in this directory:
#     make -C oracle/ref_shim -f acqgrad.mk REF=... acqgrad_dropin
# Output (git-ignored): oracle/_ref/acq_grad_dropin_test, tests/cpp/acq_grad_dropin_test.cpp: limbo_b200::acqui::UCB / EI gradients
# (lb_acq_grad) against central differences and the batched answer, the reference's opt::GradientAscent and opt::Adam over them,
# and limbo_b200::opt::BatchedGradient (run by tests/test_gpu_acq_grad.py; needs limbo_b200/lib/liblimbo_b200.so)
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
ACQGRAD_DROPIN := ../_ref/acq_grad_dropin_test

acqgrad_dropin: $(ACQGRAD_DROPIN)

$(ACQGRAD_DROPIN): $(ROOT)/tests/cpp/acq_grad_dropin_test.cpp $(ROOT)/include/limbo_b200/opt/batched_gradient.hpp $(ROOT)/include/limbo_b200/opt/batched_random.hpp $(ROOT)/include/limbo_b200/model/gp.hpp $(ROOT)/include/limbo_b200.h Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/acq_grad_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib'

.PHONY: acqgrad_dropin
