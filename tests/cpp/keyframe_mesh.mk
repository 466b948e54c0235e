# Builds keyframe_mesh_test (df::KeyframeMesher of df/dfk_mesh.h against dfk_keyframe_mesh_batch) against libdfk.so.
#   make -C tests/cpp -f keyframe_mesh.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: keyframe_mesh_test
keyframe_mesh_test: keyframe_mesh_test.cpp $(ROOT)/include/df/dfk_mesh.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ keyframe_mesh_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f keyframe_mesh_test
