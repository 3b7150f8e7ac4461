# _ref/libyolo_heads.so: yolo_heads.c (repo code, test infrastructure only) on top of darknet.mk's libyolo_oracle.so and
# libdarknet.so, with the same flags.  Built after darknet.mk; without the reference checkout nothing is built.
REFERENCE ?= /root/reference
DN := $(REFERENCE)/darknet
R  := _ref

ifeq ($(wildcard $(DN)/src/network.c),)
all:
	@echo "yolo_heads.mk: no darknet sources under $(DN); the YOLO heads oracle is not built"
else
all: $(R)/libyolo_heads.so
$(R)/libyolo_heads.so: yolo_heads.c $(R)/libyolo_oracle.so $(R)/libdarknet.so
	gcc -O2 -ffp-contract=off -shared -fPIC -I$(DN)/include -o $@ $< -L$(R) -lyolo_oracle -ldarknet -Wl,-rpath,'$$ORIGIN' -lm
endif
.PHONY: all
