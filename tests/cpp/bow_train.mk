# Builds bow_train_test (df::BowVocabulary's training constructor, Export and BowVocabularyData::SaveText of
# df/dfk_bow.h against the dfk_bow_vocabulary_train / _export calls) against libdfk.so.
#   make -C tests/cpp -f bow_train.mk
CXX := /usr/bin/g++
ROOT := ../..
CUDA ?= /usr/local/cuda
all: bow_train_test
bow_train_test: bow_train_test.cpp $(ROOT)/include/df/dfk_bow.h $(ROOT)/include/df/dfk_facade.h $(ROOT)/include/dfk.h
	$(CXX) -std=c++17 -O2 -Wall -I$(ROOT)/include -I$(CUDA)/include -o $@ bow_train_test.cpp \
	  -L$(ROOT)/deepfactors_b200 -ldfk -L$(CUDA)/lib64 -lcudart \
	  -Wl,-rpath,'$$ORIGIN/../../deepfactors_b200' -Wl,-rpath,$(CUDA)/lib64
clean:
	rm -f bow_train_test
