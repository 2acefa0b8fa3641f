# TEST INFRASTRUCTURE.  Builds oracle/_ref/libref_darknet.so: the UNMODIFIED image.darknet sources compiled IN PLACE from
# $(REF) (only when $(REF) exists) with R's -O2, every src/*.c except darknet.c (its main) and the two __R_API_*.c glue
# files, plus oracle/ref_wrap_darknet.c (a driver over the reference's own parser, network_predict, region boxes, NMS and
# top_k).  It also copies the model files the tests run (the two default cfgs and weights, the label lists, the other
# supported cfgs and the package's sample images) into oracle/_ref/darknet/.
#   make -f oracle/darknet.mk
REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
CC := $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo gcc)
PKG := $(REF)/image.darknet
DSRC := $(PKG)/src
DINC := $(PKG)/inst/include/darknet
SRCS := $(filter-out $(DSRC)/darknet.c $(DSRC)/__R_API_detector.c $(DSRC)/__R_API_classifier.c,$(wildcard $(DSRC)/*.c))
OBJS := $(patsubst $(DSRC)/%.c,$(OUT)/darknet_obj/%.o,$(SRCS))
CFGS := tiny-yolo-voc tiny darknet darknet19 darknet19_448 extraction tiny-yolo yolo-voc yolo alexnet vgg-16
FILES := $(OUT)/darknet/tiny-yolo-voc.weights $(OUT)/darknet/tiny.weights $(OUT)/darknet/voc.names \
         $(OUT)/darknet/imagenet.shortnames.list $(OUT)/darknet/coco.names \
         $(patsubst %,$(OUT)/darknet/%.cfg,$(CFGS)) \
         $(patsubst $(DINC)/data/%,$(OUT)/darknet/%,$(wildcard $(DINC)/data/*.jpg))

ifneq ($(wildcard $(DSRC)/network.c),)
ref: $(OUT)/libref_darknet.so $(FILES)
else
ref:
	@echo "reference tree $(REF) absent: using prebuilt oracle/_ref/libref_darknet.so (if any)"
endif

$(OUT)/darknet_obj/%.o: $(DSRC)/%.c
	@mkdir -p $(OUT)/darknet_obj
	$(CC) -O2 -fPIC -w -I$(DSRC) -c -o $@ $<

$(OUT)/libref_darknet.so: $(HERE)ref_wrap_darknet.c $(OBJS)
	$(CC) -O2 -fPIC -shared -w -I$(DSRC) -o $@ $(HERE)ref_wrap_darknet.c $(OBJS) -lm -lpthread

$(OUT)/darknet/%.weights: $(PKG)/inst/models/%.weights
	@mkdir -p $(OUT)/darknet
	cp $< $@
$(OUT)/darknet/%.cfg: $(DINC)/cfg/%.cfg
	@mkdir -p $(OUT)/darknet
	cp $< $@
$(OUT)/darknet/%: $(DINC)/data/%
	@mkdir -p $(OUT)/darknet
	cp $< $@

.PHONY: ref
