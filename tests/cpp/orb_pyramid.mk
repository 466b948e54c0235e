# Builds orb_pyramid_test (df::OrbPyramidDetector of df/dfk_matching.h against dfk_orb_detect_pyramid_batch) against libdfk.so.
#   make -C tests/cpp -f orb_pyramid.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: orb_pyramid_test
orb_pyramid_test: orb_pyramid_test.cpp $(ROOT)/include/df/dfk_matching.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ orb_pyramid_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f orb_pyramid_test
