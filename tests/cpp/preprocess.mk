# Builds preprocess_test (df::FramePreprocessor of df/dfk_preprocess.h against dfk_preprocess_batch) against libdfk.so.
#   make -C tests/cpp -f preprocess.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: preprocess_test
preprocess_test: preprocess_test.cpp $(ROOT)/include/df/dfk_preprocess.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ preprocess_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f preprocess_test
