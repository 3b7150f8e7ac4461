// yolo_forward.cpp -- the gf_detector_* / gf_stage_letterbox entry points of libgf_b200.so: host-only forwarders to
// libgf_yolo.so (csrc/yolo_detector.cu), the library next to this one, opened on the first call.  libgf_b200.so so exports the
// whole C ABI of include/gf_b200.h while carrying none of the detector's device code; a process that never detects never loads
// it.  A failing call also copies the detector's error text into gf_last_error().
#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

#include "../../include/gf_b200.h"

namespace gf {
extern thread_local char g_err[512];
}

namespace {

void* yolo_handle()
{
    static void* h = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        Dl_info info;
        if (!dladdr((void*)&yolo_handle, &info) || !info.dli_fname) return;
        std::string p(info.dli_fname);
        const size_t slash = p.rfind('/');
        p = (slash == std::string::npos ? std::string() : p.substr(0, slash + 1)) + "libgf_yolo.so";
        h = dlopen(p.c_str(), RTLD_NOW | RTLD_LOCAL);
    });
    return h;
}

template <typename F>
F yolo_fn(const char* name)
{
    void* h = yolo_handle();
    return h ? (F)dlsym(h, name) : nullptr;
}

int missing()
{
    snprintf(gf::g_err, sizeof(gf::g_err), "libgf_yolo.so (the YOLO detector) could not be loaded next to libgf_b200.so: %s",
             dlerror() ? "not found" : "missing symbol");
    return GF_ERR_UNSUPPORTED;
}

int copy_err(int rc)
{
    if (rc != GF_OK) {
        auto e = yolo_fn<const char* (*)(void)>("gf_detector_last_error");
        if (e) snprintf(gf::g_err, sizeof(gf::g_err), "%s", e());
    }
    return rc;
}

}  // namespace

#define GF_FORWARD(name, params, args)                                             \
    int name params                                                                \
    {                                                                              \
        static auto f = yolo_fn<int(*) params>(#name);                             \
        return f ? copy_err(f args) : missing();                                   \
    }

extern "C" {

const char* gf_detector_last_error(void)
{
    static auto f = yolo_fn<const char* (*)(void)>("gf_detector_last_error");
    return f ? f() : "libgf_yolo.so not loaded";
}

GF_FORWARD(gf_detector_create, (gf_detector** det, int device, const char* cfg, const char* weights, float thresh),
           (det, device, cfg, weights, thresh))
GF_FORWARD(gf_detector_info, (gf_detector* det, int* net_wh, int* n_layers, int* classes), (det, net_wh, n_layers, classes))
GF_FORWARD(gf_detector_detect, (gf_detector* det, const void* bgr, size_t pitch, int w, int h, int on_device, gf_box* boxes,
                                int* class_ids, float* probs, int cap, int* n_out),
           (det, bgr, pitch, w, h, on_device, boxes, class_ids, probs, cap, n_out))
GF_FORWARD(gf_detector_last_device_ms, (gf_detector* det, float* ms), (det, ms))
GF_FORWARD(gf_detector_layer_shape, (gf_detector* det, int layer, int* whc), (det, layer, whc))
GF_FORWARD(gf_detector_layer_output, (gf_detector* det, int layer, float* out, size_t n), (det, layer, out, n))
GF_FORWARD(gf_detector_layer_times, (gf_detector* det, int reps, float* ms), (det, reps, ms))
GF_FORWARD(gf_stage_letterbox, (int device, const void* bgr, size_t pitch, int w, int h, int on_device, int net_w, int net_h,
                                float* out),
           (device, bgr, pitch, w, h, on_device, net_w, net_h, out))
GF_FORWARD(gf_detector_set_precision, (gf_detector* det, int precision), (det, precision))
GF_FORWARD(gf_detector_get_precision, (gf_detector* det, int* precision), (det, precision))
GF_FORWARD(gf_detector_set_max_batch, (gf_detector* det, int max_batch), (det, max_batch))
GF_FORWARD(gf_detector_detect_batch, (gf_detector* det, int n, const void* const* bgr, const size_t* pitch, const int* w,
                                      const int* h, int on_device, gf_box* boxes, int* class_ids, float* probs, int cap,
                                      int* box_start),
           (det, n, bgr, pitch, w, h, on_device, boxes, class_ids, probs, cap, box_start))
GF_FORWARD(gf_detector_member_layer_output, (gf_detector* det, int member, int layer, float* out, size_t n),
           (det, member, layer, out, n))
GF_FORWARD(gf_stage_yolo_conv, (int device, int precision, const int* shape, const float* in, const float* w, const float* bias,
                                const float* scale, const float* mean, const float* var, float* out),
           (device, precision, shape, in, w, bias, scale, mean, var, out))

void gf_detector_destroy(gf_detector* det)
{
    static auto f = yolo_fn<void (*)(gf_detector*)>("gf_detector_destroy");
    if (f) f(det);
}

}  // extern "C"
