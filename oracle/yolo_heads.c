/* yolo_heads.c -- test-only addition to the YOLO oracle: darknet's decoding of given head outputs.  yh_detect_from_heads copies
 * the [region] / [yolo] outputs a caller supplies (e.g. the GPU detector's, in its TF32 mode) into the darknet network's head
 * layers and runs yolo_harness.c's yh_detect on them: get_network_boxes(w, h, thresh, 0.5, 0, 1) and do_nms_obj(0.4).  So the
 * decoding, NMS and extraction can be checked bit for bit whatever arithmetic produced the heads. */
#include <string.h>

#include "darknet.h"

int yh_detect(network* net, int w, int h, float thresh, float* bbox, float* obj, float* prob, int n_max);

/* heads[i] holds layer layer_idx[i]'s outputs ([region] or [yolo], l.outputs floats); returns yh_detect's count, or -1 when a
 * named layer is not a head */
int yh_detect_from_heads(network* net, int n_heads, const int* layer_idx, const float* const* heads, int w, int h, float thresh,
                         float* bbox, float* obj, float* prob, int n_max)
{
    for (int i = 0; i < n_heads; ++i) {
        if (layer_idx[i] < 0 || layer_idx[i] >= net->n) return -1;
        layer* l = &net->layers[layer_idx[i]];
        if (l->type != REGION && l->type != YOLO) return -1;
        memcpy(l->output, heads[i], sizeof(float) * l->outputs);
    }
    return yh_detect(net, w, h, thresh, bbox, obj, prob, n_max);
}
