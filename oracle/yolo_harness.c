/* yolo_harness.c -- the YOLO detector's CPU oracle: darknet (libdarknet.so, built by darknet.mk) driven the way the
 * darknet_ros node drives it for one frame (YoloObjectDetector.cpp fetchInThread + detectInThread with avg_frames = 1):
 *   BGR8 frame -> planar float image / 255 with OpenCV's channel order (the node's mat_to_image, restated here because darknet's
 *   copy needs OpenCV, including the rgbgr_image it ends with) -> rgbgr_image -> letterbox_image at the net size
 *   -> network_predict -> get_network_boxes(w, h, thresh, 0.5, 0, 1) -> do_nms_obj(0.4).
 * Everything is exposed through plain arrays for ctypes (tests/yolo_ref.py); the box extraction darknet_ros does after NMS
 * is restated in Python there. */
#include <stdlib.h>
#include <string.h>

#include "darknet.h"

char* get_layer_string(LAYER_TYPE a);

network* yh_load(char* cfg, char* weights)
{
    network* net = load_network(cfg, weights, 0);
    set_batch_network(net, 1);
    return net;
}

int yh_n_layers(network* net) { return net->n; }
int yh_net_size(network* net, int* whc)
{
    whc[0] = net->w; whc[1] = net->h; whc[2] = net->c;
    return 0;
}

/* type string into name (>= 32 bytes); v = w h c out_w out_h out_c outputs n size stride pad batch_normalize activation
 * classes nweights */
int yh_layer_info(network* net, int i, char* name, int* v)
{
    layer l = net->layers[i];
    strncpy(name, get_layer_string(l.type), 31);
    name[31] = 0;
    int a[15] = {l.w, l.h, l.c, l.out_w, l.out_h, l.out_c, l.outputs, l.n, l.size, l.stride, l.pad, l.batch_normalize,
                 (int)l.activation, l.classes, l.nweights};
    memcpy(v, a, sizeof(a));
    return 0;
}

/* a convolutional layer's parameters as load_weights left them: biases, scales, rolling mean, rolling variance (n each; the last
 * three only with batch_normalize) and the weights (nweights) */
int yh_conv_params(network* net, int i, float* biases, float* scales, float* mean, float* var, float* weights)
{
    layer l = net->layers[i];
    if (l.type != CONVOLUTIONAL) return -1;
    memcpy(biases, l.biases, sizeof(float) * l.n);
    if (l.batch_normalize) {
        memcpy(scales, l.scales, sizeof(float) * l.n);
        memcpy(mean, l.rolling_mean, sizeof(float) * l.n);
        memcpy(var, l.rolling_variance, sizeof(float) * l.n);
    }
    memcpy(weights, l.weights, sizeof(float) * l.nweights);
    return 0;
}

/* the node's input image: planar [3][net h][net w] */
int yh_letterbox(network* net, const unsigned char* bgr, int pitch, int w, int h, float* out)
{
    image im = make_image(w, h, 3);
    for (int y = 0; y < h; ++y)
        for (int k = 0; k < 3; ++k)
            for (int x = 0; x < w; ++x) im.data[k * w * h + y * w + x] = bgr[(size_t)y * pitch + 3 * x + k] / 255.;
    rgbgr_image(im);           /* the end of mat_to_image */
    rgbgr_image(im);           /* fetchInThread */
    image boxed = letterbox_image(im, net->w, net->h);
    memcpy(out, boxed.data, sizeof(float) * net->w * net->h * 3);
    free_image(boxed);
    free_image(im);
    return 0;
}

int yh_predict(network* net, float* input)
{
    network_predict(net, input);
    return 0;
}

int yh_layer_output(network* net, int i, float* out)
{
    memcpy(out, net->layers[i].output, sizeof(float) * net->layers[i].outputs);
    return 0;
}

/* after yh_predict: the detections of the frame (w x h) after NMS, in darknet's order.  n_max rows of bbox[4], objectness[1],
 * probs[classes]; returns the count (all of them, even past n_max) */
int yh_detect(network* net, int w, int h, float thresh, float* bbox, float* obj, float* prob, int n_max)
{
    layer last = net->layers[net->n - 1];
    int nboxes = 0;
    detection* dets = get_network_boxes(net, w, h, thresh, .5, 0, 1, &nboxes);
    do_nms_obj(dets, nboxes, last.classes, .4);
    for (int i = 0; i < nboxes && i < n_max; ++i) {
        bbox[4 * i + 0] = dets[i].bbox.x; bbox[4 * i + 1] = dets[i].bbox.y;
        bbox[4 * i + 2] = dets[i].bbox.w; bbox[4 * i + 3] = dets[i].bbox.h;
        obj[i] = dets[i].objectness;
        memcpy(prob + (size_t)i * last.classes, dets[i].prob, sizeof(float) * last.classes);
    }
    free_detections(dets, nboxes);
    return nboxes;
}

void yh_free(network* net) { free_network(net); }
