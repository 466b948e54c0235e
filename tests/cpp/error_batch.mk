# Builds error_batch_test (SfmAligner::EvaluateErrorBatch through the facade) against libdfk.so.
#   make -C tests/cpp -f error_batch.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: error_batch_test
error_batch_test: error_batch_test.cpp $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/df/dfk_standins.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ error_batch_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f error_batch_test
