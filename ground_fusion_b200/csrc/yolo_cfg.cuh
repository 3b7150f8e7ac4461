// yolo_cfg.cuh -- host side of gf_detector: darknet's cfg format and .weights format, read into a network description.
// Written from the file formats darknet documents by use (section headers "[type]", "key=value" lines, '#' and ';' comments,
// whitespace removed anywhere in a line; weights: an int32 major / minor / revision header, the images-seen counter in 8 bytes
// when major * 10 + minor >= 2 and in 4 otherwise, then per convolutional layer biases[n], with batch_normalize scales[n],
// rolling_mean[n], rolling_variance[n], then weights[n][c][size][size], all float32).
// The shapes follow darknet's layer constructors for the networks the reference ships (DESIGN.md "YOLO detector"): anything
// else -- a layer type, an activation or a key value whose inference darknet would run differently -- is refused by name.
#pragma once
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace gfy {

enum LayerType { L_CONV, L_MAXPOOL, L_ROUTE, L_REORG, L_SHORTCUT, L_UPSAMPLE, L_REGION, L_YOLO };
enum Act { A_LINEAR = 0, A_LEAKY = 1 };

struct Layer {
    int type = 0;
    int w = 0, h = 0, c = 0;             // input
    int ow = 0, oh = 0, oc = 0;          // output
    long outputs = 0;
    // convolutional
    int n = 0, size = 0, stride = 1, pad = 0, bn = 0, act = A_LINEAR;
    std::vector<float> biases, scales, mean, var, weights;
    // maxpool: size, stride, pad (darknet's `padding`)
    // route
    std::vector<int> in;
    // shortcut (from = in[0]), with its input dims in w/h/c; alpha, beta; act
    float alpha = 1.f, beta = 1.f;
    // upsample: stride, scale
    float scale = 1.f;
    // region / yolo
    int classes = 0, coords = 4, num = 0, softmax = 0, background = 0;
    std::vector<int> mask;
    std::vector<float> anchors;
};

struct Net {
    int w = 0, h = 0, c = 0;
    std::vector<Layer> layers;
};

struct Section {
    std::string type;
    std::vector<std::pair<std::string, std::string>> kv;
    const char* find(const char* k) const
    {
        for (auto& p : kv) if (p.first == k) return p.second.c_str();
        return nullptr;
    }
    int geti(const char* k, int def) const { const char* v = find(k); return v ? atoi(v) : def; }
    float getf(const char* k, float def) const { const char* v = find(k); return v ? (float)atof(v) : def; }
};

inline bool read_sections(const char* path, std::vector<Section>& out, std::string& err)
{
    FILE* f = fopen(path, "r");
    if (!f) { err = std::string("cannot open cfg ") + path; return false; }
    char buf[8192];
    while (fgets(buf, sizeof(buf), f)) {
        std::string s;
        for (char* p = buf; *p; p++) if (*p != ' ' && *p != '\t' && *p != '\n' && *p != '\r') s += *p;
        if (s.empty() || s[0] == '#' || s[0] == ';') continue;
        if (s[0] == '[') { out.push_back(Section{s.substr(1, s.find(']') == std::string::npos ? std::string::npos : s.find(']') - 1), {}}); continue; }
        const size_t eq = s.find('=');
        if (out.empty() || eq == std::string::npos) { fclose(f); err = "bad cfg line: " + s; return false; }
        out.back().kv.push_back({s.substr(0, eq), s.substr(eq + 1)});
    }
    fclose(f);
    if (out.empty() || (out[0].type != "net" && out[0].type != "network")) { err = "cfg must start with [net]"; return false; }
    return true;
}

inline std::vector<float> parse_floats(const char* a)
{
    std::vector<float> v;
    while (a && *a) {
        v.push_back((float)atof(a));
        a = strchr(a, ',');
        if (a) a++;
    }
    return v;
}

inline bool parse_act(const Section& s, const char* def, int& act, std::string& err)
{
    const char* a = s.find("activation");
    std::string v = a ? a : def;
    if (v == "leaky") act = A_LEAKY;
    else if (v == "linear") act = A_LINEAR;
    else { err = "unsupported activation '" + v + "' in [" + s.type + "] (leaky and linear only)"; return false; }
    return true;
}

#define GFY_REFUSE(cond, msg) do { if (cond) { err = std::string("[") + s.type + "] layer " + std::to_string(i) + ": " + (msg); return false; } } while (0)

inline bool parse_net(const char* path, Net& net, std::string& err)
{
    std::vector<Section> secs;
    if (!read_sections(path, secs, err)) return false;
    const Section& ns = secs[0];
    net.w = ns.geti("width", 0); net.h = ns.geti("height", 0); net.c = ns.geti("channels", 0);
    if (net.c != 3) { err = "[net] channels must be 3 (a BGR frame)"; return false; }
    if (net.w < 1 || net.h < 1 || net.w > 8192 || net.h > 8192) { err = "[net] width / height must be in [1, 8192]"; return false; }
    int w = net.w, h = net.h, c = net.c;
    for (size_t si = 1; si < secs.size(); si++) {
        const Section& s = secs[si];
        const int i = (int)si - 1;
        Layer l;
        l.w = w; l.h = h; l.c = c;
        GFY_REFUSE(!(w && h && c), "the layer before must output an image");
        if (s.type == "convolutional" || s.type == "conv") {
            l.type = L_CONV;
            l.n = s.geti("filters", 1); l.size = s.geti("size", 1); l.stride = s.geti("stride", 1);
            const int pad = s.geti("pad", 0);
            l.pad = pad ? l.size / 2 : s.geti("padding", 0);
            l.bn = s.geti("batch_normalize", 0);
            GFY_REFUSE(s.geti("groups", 1) != 1, "groups other than 1 are not supported");
            GFY_REFUSE(s.geti("binary", 0) || s.geti("xnor", 0), "binary / xnor convolutions are not supported");
            GFY_REFUSE(s.geti("flipped", 0), "flipped weights are not supported");
            GFY_REFUSE(l.n < 1 || l.size < 1 || l.stride < 1 || l.pad < 0, "bad filters / size / stride / padding");
            if (!parse_act(s, "logistic", l.act, err)) return false;
            l.ow = (w + 2 * l.pad - l.size) / l.stride + 1;
            l.oh = (h + 2 * l.pad - l.size) / l.stride + 1;
            l.oc = l.n;
        } else if (s.type == "maxpool" || s.type == "max") {
            l.type = L_MAXPOOL;
            l.stride = s.geti("stride", 1); l.size = s.geti("size", l.stride); l.pad = s.geti("padding", l.size - 1);
            GFY_REFUSE(l.stride < 1 || l.size < 1 || l.pad < 0, "bad size / stride / padding");
            l.ow = (w + l.pad - l.size) / l.stride + 1;
            l.oh = (h + l.pad - l.size) / l.stride + 1;
            l.oc = c;
        } else if (s.type == "route") {
            l.type = L_ROUTE;
            const char* a = s.find("layers");
            GFY_REFUSE(!a, "route needs layers=");
            for (const char* p = a; p && *p;) {
                int k = atoi(p);
                if (k < 0) k = i + k;
                GFY_REFUSE(k < 0 || k >= i, "route input out of range");
                l.in.push_back(k);
                p = strchr(p, ',');
                if (p) p++;
            }
            const Layer& f = net.layers[l.in[0]];
            l.ow = f.ow; l.oh = f.oh; l.oc = 0;
            for (int k : l.in) {
                const Layer& g = net.layers[k];
                GFY_REFUSE(g.ow != f.ow || g.oh != f.oh, "route inputs of different sizes are not supported");
                l.oc += g.oc;
            }
        } else if (s.type == "reorg") {
            l.type = L_REORG;
            l.stride = s.geti("stride", 1);
            GFY_REFUSE(s.geti("reverse", 0) || s.geti("flatten", 0) || s.geti("extra", 0), "reverse / flatten / extra reorg is not supported");
            GFY_REFUSE(l.stride < 1 || w % l.stride || h % l.stride, "reorg stride must divide the input");
            l.ow = w / l.stride; l.oh = h / l.stride; l.oc = c * l.stride * l.stride;
        } else if (s.type == "shortcut") {
            l.type = L_SHORTCUT;
            const char* a = s.find("from");
            GFY_REFUSE(!a, "shortcut needs from=");
            int k = atoi(a);
            if (k < 0) k = i + k;
            GFY_REFUSE(k < 0 || k >= i, "shortcut input out of range");
            l.in.push_back(k);
            const Layer& f = net.layers[k];
            l.w = f.ow; l.h = f.oh; l.c = f.oc;            // darknet keeps the added layer's dims in w / h / c
            l.ow = w; l.oh = h; l.oc = c;
            const int st = l.w / l.ow, sa = l.ow / l.w;
            GFY_REFUSE(st != l.h / l.oh || sa != l.oh / l.h, "shortcut sizes must scale alike in x and y");
            if (!parse_act(s, "linear", l.act, err)) return false;
            l.alpha = s.getf("alpha", 1.f); l.beta = s.getf("beta", 1.f);
        } else if (s.type == "upsample") {
            l.type = L_UPSAMPLE;
            l.stride = s.geti("stride", 2);
            GFY_REFUSE(l.stride < 1, "reverse (negative stride) upsample is not supported");
            l.scale = s.getf("scale", 1.f);
            l.ow = w * l.stride; l.oh = h * l.stride; l.oc = c;
        } else if (s.type == "region") {
            l.type = L_REGION;
            l.coords = s.geti("coords", 4); l.classes = s.geti("classes", 20); l.num = s.geti("num", 1);
            l.softmax = s.geti("softmax", 0); l.background = s.geti("background", 0);
            GFY_REFUSE(l.coords != 4, "coords other than 4 are not supported");
            GFY_REFUSE(l.background, "background is not supported");
            GFY_REFUSE(s.find("tree") || s.find("map"), "softmax trees and class maps are not supported");
            GFY_REFUSE(l.classes < 1 || l.num < 1, "bad classes / num");
            GFY_REFUSE(c != l.num * (l.classes + l.coords + 1), "input channels must equal num * (classes + coords + 1)");
            l.anchors = parse_floats(s.find("anchors"));
            GFY_REFUSE((int)l.anchors.size() < 2 * l.num, "fewer than 2 * num anchors");
            l.ow = w; l.oh = h; l.oc = c;
        } else if (s.type == "yolo") {
            l.type = L_YOLO;
            l.classes = s.geti("classes", 20);
            const int total = s.geti("num", 1);
            const char* m = s.find("mask");
            if (m) { for (float v : parse_floats(m)) l.mask.push_back((int)v); }
            else for (int k = 0; k < total; k++) l.mask.push_back(k);
            l.num = (int)l.mask.size();
            GFY_REFUSE(s.find("map"), "class maps are not supported");
            GFY_REFUSE(l.classes < 1 || total < 1, "bad classes / num");
            l.anchors = parse_floats(s.find("anchors"));
            for (int k : l.mask) GFY_REFUSE(k < 0 || 2 * k + 1 >= (int)l.anchors.size() || k >= total, "mask entry without an anchor");
            GFY_REFUSE(c != l.num * (l.classes + 4 + 1), "input channels must equal the mask count * (classes + 5)");
            l.ow = w; l.oh = h; l.oc = c;
        } else {
            err = "unsupported layer type [" + s.type + "] (layer " + std::to_string(i) + ")";
            return false;
        }
        GFY_REFUSE(l.ow < 1 || l.oh < 1 || l.oc < 1, "the output is empty at this input size");
        l.outputs = (long)l.ow * l.oh * l.oc;
        GFY_REFUSE(l.outputs > (1l << 30), "the output is too large");
        w = l.ow; h = l.oh; c = l.oc;
        net.layers.push_back(l);
    }
    if (net.layers.empty()) { err = "the network has no layers"; return false; }
    const int lt = net.layers.back().type;
    if (lt != L_REGION && lt != L_YOLO) { err = "the last layer must be [region] or [yolo]"; return false; }
    for (const Layer& l : net.layers)
        if ((l.type == L_REGION || l.type == L_YOLO) && l.classes != net.layers.back().classes) {
            err = "every [region] / [yolo] layer must have the last layer's classes"; return false;
        }
    return true;
}
#undef GFY_REFUSE

inline bool load_weights(const char* path, Net& net, std::string& err)
{
    FILE* f = fopen(path, "rb");
    if (!f) { err = std::string("cannot open weights ") + path; return false; }
    int32_t hdr[3];
    bool ok = fread(hdr, 4, 3, f) == 3;
    if (ok) {
        const int seen_bytes = (hdr[0] * 10 + hdr[1] >= 2 && hdr[0] < 1000 && hdr[1] < 1000) ? 8 : 4;
        char seen[8];
        ok = fread(seen, 1, seen_bytes, f) == (size_t)seen_bytes;
    }
    for (size_t i = 0; ok && i < net.layers.size(); i++) {
        Layer& l = net.layers[i];
        if (l.type != L_CONV) continue;
        auto rd = [&](std::vector<float>& v, size_t n) { v.resize(n); return fread(v.data(), 4, n, f) == n; };
        ok = rd(l.biases, l.n);
        if (ok && l.bn) ok = rd(l.scales, l.n) && rd(l.mean, l.n) && rd(l.var, l.n);
        if (ok) ok = rd(l.weights, (size_t)l.n * l.c * l.size * l.size);
        if (!ok) err = "weights file ends inside layer " + std::to_string(i);
    }
    if (!ok && err.empty()) err = "weights file header is truncated";
    fclose(f);
    return ok;
}

}  // namespace gfy
