# TEST INFRASTRUCTURE.  For the R shim test (tests/test_darknet_rshim_gpu.py), next to oracle/darknet.mk's build:
#   oracle/_ref/libref_darknet_rapi.so  the package's own R glue (src/__R_API_detector.c, src/__R_API_classifier.c,
#                                       unmodified) compiled against the R stubs of oracle/stubs/ and linked with
#                                       libref_darknet.so: the reference image_b200/rshim/darknet_r_api.c is compared with;
#   oracle/_ref/darknet/include/        the package's headers, which the shim is compiled against;
#   oracle/_ref/darknet/data/labels/    the label glyphs draw_detections reads.
# Only when $(REF) exists; run after oracle/darknet.mk.
#   make -f oracle/darknet_rapi.mk
REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
CC := $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo gcc)
PKG := $(REF)/image.darknet
DSRC := $(PKG)/src
DINC := $(PKG)/inst/include/darknet
FILES := $(patsubst $(DINC)/data/labels/%,$(OUT)/darknet/data/labels/%,$(wildcard $(DINC)/data/labels/*.png)) \
         $(patsubst $(DSRC)/%,$(OUT)/darknet/include/%,$(wildcard $(DSRC)/*.h))

ifneq ($(wildcard $(DSRC)/__R_API_detector.c),)
ref: $(OUT)/libref_darknet_rapi.so $(FILES)
else
ref:
	@echo "reference tree $(REF) absent: using prebuilt oracle/_ref/libref_darknet_rapi.so (if any)"
endif

$(OUT)/libref_darknet_rapi.so: $(DSRC)/__R_API_detector.c $(DSRC)/__R_API_classifier.c $(OUT)/libref_darknet.so $(HERE)stubs/Rinternals.h $(HERE)stubs/Rdefines.h
	$(CC) -O2 -fPIC -shared -w -I$(DSRC) -I$(HERE)stubs -o $@ $(DSRC)/__R_API_detector.c $(DSRC)/__R_API_classifier.c \
	  -L$(OUT) -lref_darknet -Wl,-rpath,'$$ORIGIN' -lm
$(OUT)/darknet/data/labels/%: $(DINC)/data/labels/%
	@mkdir -p $(OUT)/darknet/data/labels
	cp $< $@
$(OUT)/darknet/include/%: $(DSRC)/%
	@mkdir -p $(OUT)/darknet/include
	cp $< $@

.PHONY: ref
