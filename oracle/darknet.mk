# The YOLO detector's CPU oracle (test infrastructure only; never linked into the product).
#   _ref/libdarknet.so      the reference's vendored darknet built for the CPU as its own Makefile does with
#                           GPU=0 CUDNN=0 OPENCV=0 OPENMP=0, but -O2 -ffp-contract=off in place of OPTS=-Ofast:
#                           no reassociation and no FMA contraction, so every sum runs in source order
#   _ref/libyolo_oracle.so  yolo_harness.c (repo code) on top of it
#   _ref/yolo_cfg/          the six network cfgs the reference ships
# Without the reference checkout nothing is built; the tests that need the oracle then report it missing.
REFERENCE ?= /root/reference
DN  := $(REFERENCE)/darknet
R   := _ref
OBJ := $(R)/darknet_obj
# the C objects of darknet's OBJ list with GPU=0 and OPENCV=0 (image_opencv.cpp compiles to nothing without OPENCV)
DN_SRC := gemm utils cuda deconvolutional_layer convolutional_layer list image activations im2col col2im blas crop_layer \
          dropout_layer maxpool_layer softmax_layer data matrix network connected_layer cost_layer parser option_list \
          detection_layer route_layer upsample_layer box normalization_layer avgpool_layer layer local_layer shortcut_layer \
          logistic_layer activation_layer rnn_layer gru_layer crnn_layer demo batchnorm_layer region_layer reorg_layer tree \
          lstm_layer l2norm_layer yolo_layer iseg_layer
DN_CFLAGS := -Wall -Wno-unused-result -Wno-unknown-pragmas -fPIC -O2 -ffp-contract=off -I$(DN)/include -I$(DN)/src
CFGS := yolov2-tiny yolov2-tiny-voc yolov2 yolov2-voc yolov3 yolov3-voc

ifeq ($(wildcard $(DN)/src/network.c),)
all:
	@echo "darknet.mk: no darknet sources under $(DN); the YOLO oracle is not built"
else
all: $(R)/libdarknet.so $(R)/libyolo_oracle.so $(addprefix $(R)/yolo_cfg/,$(addsuffix .cfg,$(CFGS)))
$(OBJ)/%.o: $(DN)/src/%.c
	@mkdir -p $(OBJ); gcc $(DN_CFLAGS) -c $< -o $@
$(R)/libdarknet.so: $(addprefix $(OBJ)/,$(addsuffix .o,$(DN_SRC)))
	gcc -shared -o $@ $^ -lm -pthread
$(R)/libyolo_oracle.so: yolo_harness.c $(R)/libdarknet.so
	gcc -O2 -ffp-contract=off -shared -fPIC -I$(DN)/include -o $@ $< -L$(R) -ldarknet -Wl,-rpath,'$$ORIGIN' -lm
$(R)/yolo_cfg/%.cfg: $(REFERENCE)/vins_estimator/yolo_network_config/cfg/%.cfg
	@mkdir -p $(R)/yolo_cfg; cp $< $@
endif
.PHONY: all
