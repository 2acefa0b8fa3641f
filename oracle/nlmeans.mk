# TEST INFRASTRUCTURE.  Builds oracle/_ref/libref_nlmeans.so: the UNMODIFIED image.DenoiseNLMeans sources compiled IN
# PLACE from $(REF) (only when $(REF) exists), with R's -O2 but WITHOUT -fopenmp although its Makevars asks for it: the
# parallel loop of nlmeans_ipol races on the output rows, so the serial order is the reference (DESIGN.md §5).
#   make -f oracle/nlmeans.mk
REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CC := $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo gcc)
NSRC := $(REF)/image.DenoiseNLMeans/src

ifneq ($(wildcard $(NSRC)/libdenoising.cpp),)
ref: $(OUT)/libref_nlmeans.so
else
ref:
	@echo "reference tree $(REF) absent: using prebuilt oracle/_ref/libref_nlmeans.so (if any)"
endif

$(OUT)/libref_nlmeans.so: $(HERE)ref_wrap_nlmeans.cpp $(HERE)stubs_nlmeans/Rcpp.h $(HERE)stubs/Rcpp.h
	mkdir -p $(OUT)
	$(CC) -O2 -fPIC -c -I$(NSRC) -o $(OUT)/mt19937ar.o $(NSRC)/mt19937ar.c
	$(CXX) -O2 -fPIC -shared -I$(HERE)stubs_nlmeans -I$(HERE)stubs -I$(NSRC) -o $@ $(HERE)ref_wrap_nlmeans.cpp \
	  $(NSRC)/rcpp_denoisenlmeans.cpp $(NSRC)/libdenoising.cpp $(NSRC)/libauxiliar.cpp $(OUT)/mt19937ar.o -lm

.PHONY: ref
