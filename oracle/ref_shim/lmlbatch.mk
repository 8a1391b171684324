# oracle/ref_shim/lmlbatch.mk — the batched hyper-parameter fit drop-in test built against the reference's OWN headers (REF = the
# src/ directory of a resibots/limbo checkout; __graft_entry__.build() passes it) and the Eigen/Boost stand-in in this directory:
#     make -C oracle/ref_shim -f lmlbatch.mk REF=... lmlbatch_dropin
# Output (git-ignored): oracle/_ref/lml_batch_dropin_test, tests/cpp/lml_batch_dropin_test.cpp: limbo_b200::model::GP::lml_grad_batch
# against the reference GP, limbo_b200::opt::BatchedRprop against the reference's opt::Rprop, and a GP typedef with
# limbo_b200::model::gp::BatchedKernelLFOpt (run by tests/test_gpu_lml_batch.py; needs limbo_b200/lib/liblimbo_b200.so)
CXX ?= g++
REF ?= ../../../reference/src
ROOT := ../..
LMLBATCH_DROPIN := ../_ref/lml_batch_dropin_test

lmlbatch_dropin: $(LMLBATCH_DROPIN)

$(LMLBATCH_DROPIN): $(ROOT)/tests/cpp/lml_batch_dropin_test.cpp $(ROOT)/include/limbo_b200/opt/batched_rprop.hpp $(ROOT)/include/limbo_b200/model/gp.hpp $(ROOT)/include/limbo_b200.h Eigen/Core
	mkdir -p ../_ref
	$(CXX) -O2 -std=c++17 -w -I. -I$(REF) -I$(ROOT)/include $(ROOT)/tests/cpp/lml_batch_dropin_test.cpp -o $@ \
	  -L$(ROOT)/limbo_b200/lib -llimbo_b200 -Wl,-rpath,'$$ORIGIN/../../limbo_b200/lib'

.PHONY: lmlbatch_dropin
