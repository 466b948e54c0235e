# Builds match_test (df::ReprojectionMatcher of df/dfk_matching.h against the C matching calls) against libdfk.so.
#   make -C tests/cpp -f match.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: match_test
match_test: match_test.cpp $(ROOT)/include/df/dfk_matching.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ match_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f match_test
