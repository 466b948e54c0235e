# Builds window_solve_test (dfk_window_solve vs a host Cholesky of df::WindowSystem) against libdfk.so.
#   make -C tests/cpp -f window_solve.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: window_solve_test
window_solve_test: window_solve_test.cpp $(ROOT)/include/df/dfk_factor.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/df/dfk_standins.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ window_solve_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f window_solve_test
