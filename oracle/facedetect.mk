# TEST INFRASTRUCTURE.  Builds oracle/_ref/libref_facedetect.so: the UNMODIFIED image.libfacedetection sources compiled IN
# PLACE from $(REF) (only when $(REF) exists) with R's -O2 and the -fopenmp its Makevars asks for, plus
# oracle/ref_wrap_facedetect.cpp (facedetect_cnn and a layer driver over the reference's own functions).  The convolution
# loops it parallelises write disjoint outputs, so the build is deterministic.
#   make -f oracle/facedetect.mk
REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
FSRC := $(REF)/image.libfacedetection/src

ifneq ($(wildcard $(FSRC)/facedetectcnn.cpp),)
ref: $(OUT)/libref_facedetect.so
else
ref:
	@echo "reference tree $(REF) absent: using prebuilt oracle/_ref/libref_facedetect.so (if any)"
endif

$(OUT)/fd_int8data.o: $(FSRC)/facedetectcnn-int8data.cpp $(HERE)stubs_facedetect/Rcpp.h
	mkdir -p $(OUT)
	$(CXX) -O2 -fPIC -fopenmp -I$(HERE)stubs_facedetect -I$(FSRC) -c -o $@ $<

$(OUT)/libref_facedetect.so: $(HERE)ref_wrap_facedetect.cpp $(HERE)stubs_facedetect/Rcpp.h $(OUT)/fd_int8data.o
	$(CXX) -O2 -fPIC -shared -fopenmp -I$(HERE)stubs_facedetect -I$(FSRC) -o $@ $(HERE)ref_wrap_facedetect.cpp \
	  $(FSRC)/facedetectcnn.cpp $(FSRC)/facedetectcnn-model.cpp $(OUT)/fd_int8data.o -lm

.PHONY: ref
