# Builds depth_prior_test (df::DepthPriorFactor + WindowSystem::AddDepthPrior) against libdfk.so.
#   make -C tests/cpp -f depth_prior.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: depth_prior_test
depth_prior_test: depth_prior_test.cpp $(ROOT)/include/df/dfk_factor.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/df/dfk_standins.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ depth_prior_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f depth_prior_test
