/*
 * tests/clahe_restate.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Plain-C restatement of cv::CLAHE::apply for CV_8UC1 (cv::createCLAHE(clip_limit, Size(tiles_x, tiles_y))), the call the
 * reference makes on every camera image when the config key `equalize` is set (rosNodeTest.cpp:256-261).  Pinned bit for
 * bit against cv2 4.13.0 by tests/test_clahe_oracle.py; the CUDA kernels of ground_fusion_b200/csrc/fe_clahe.cuh follow it
 * operation by operation.
 *
 * Build: gcc -O2 -ffp-contract=off -msse2 -mfpmath=sse -shared -fPIC.  Every float op must round on its own.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define GF_EXPORT __attribute__((visibility("default")))

static inline int reflect101(int i, int n)
{
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;
}

static inline uint8_t sat_u8(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
static inline int cv_round_f(float v) { return (int)lrintf(v); }      /* round half to even */
static inline int cv_floor_f(float v) { int i = (int)v; return i - (i > v); }

/* Tile geometry and clip limit as CLAHE_Impl::apply derives them.  stats (nullable, 4 ints): tiles that clipped, tiles
 * with a non-zero residual, 1 if the histogram source was padded, the integer clip limit. */
GF_EXPORT void gfo_clahe(const uint8_t* src, int w, int h, double clip_limit, int tiles_x, int tiles_y, uint8_t* dst, int* stats)
{
    /* padding: when EITHER dimension does not divide, copyMakeBorder(0, ty - h % ty, 0, tx - w % tx, REFLECT_101), so a
     * dimension that divides still gains a whole tile row / column */
    const int padded = (w % tiles_x != 0) || (h % tiles_y != 0);
    const int ext_w = padded ? w + tiles_x - w % tiles_x : w, ext_h = padded ? h + tiles_y - h % tiles_y : h;
    const int tw = ext_w / tiles_x, th = ext_h / tiles_y, area = tw * th;
    const float lut_scale = 255.f / (float)area;
    int limit = 0;
    if (clip_limit > 0.0) {
        limit = (int)(clip_limit * area / 256);
        if (limit < 1) limit = 1;
    }
    if (stats) { stats[0] = stats[1] = 0; stats[2] = padded; stats[3] = limit; }
    uint8_t* lut = (uint8_t*)malloc((size_t)tiles_x * tiles_y * 256);
    for (int ty = 0; ty < tiles_y; ty++)
        for (int tx = 0; tx < tiles_x; tx++) {
            int hist[256];
            memset(hist, 0, sizeof(hist));
            for (int r = 0; r < th; r++) {
                const uint8_t* row = src + (size_t)reflect101(ty * th + r, h) * w;
                for (int c = 0; c < tw; c++) hist[row[reflect101(tx * tw + c, w)]]++;
            }
            if (limit > 0) {
                int excess = 0;
                for (int i = 0; i < 256; i++)
                    if (hist[i] > limit) { excess += hist[i] - limit; hist[i] = limit; }
                const int batch = excess / 256, residual = excess - 256 * batch;
                for (int i = 0; i < 256; i++) hist[i] += batch;
                if (residual) {
                    const int step = 256 / residual > 1 ? 256 / residual : 1;
                    for (int i = 0, left = residual; i < 256 && left > 0; i += step, left--) hist[i]++;
                }
                if (stats) { stats[0] += excess > 0; stats[1] += residual != 0; }
            }
            uint8_t* L = lut + ((size_t)ty * tiles_x + tx) * 256;
            int sum = 0;
            for (int i = 0; i < 256; i++) {
                sum += hist[i];
                L[i] = sat_u8(cv_round_f((float)sum * lut_scale));
            }
        }
    const float inv_tw = 1.f / (float)tw, inv_th = 1.f / (float)th;
    for (int y = 0; y < h; y++) {
        const float tyf = (float)y * inv_th - 0.5f;
        int ty1 = cv_floor_f(tyf), ty2 = ty1 + 1;
        const float ya = tyf - (float)ty1, ya1 = 1.f - ya;
        if (ty1 < 0) ty1 = 0;
        if (ty2 > tiles_y - 1) ty2 = tiles_y - 1;
        const uint8_t* L1 = lut + (size_t)ty1 * tiles_x * 256;
        const uint8_t* L2 = lut + (size_t)ty2 * tiles_x * 256;
        for (int x = 0; x < w; x++) {
            const float txf = (float)x * inv_tw - 0.5f;
            int tx1 = cv_floor_f(txf), tx2 = tx1 + 1;
            const float xa = txf - (float)tx1, xa1 = 1.f - xa;
            if (tx1 < 0) tx1 = 0;
            if (tx2 > tiles_x - 1) tx2 = tiles_x - 1;
            const int v = src[(size_t)y * w + x];
            const float res = ((float)L1[tx1 * 256 + v] * xa1 + (float)L1[tx2 * 256 + v] * xa) * ya1 +
                              ((float)L2[tx1 * 256 + v] * xa1 + (float)L2[tx2 * 256 + v] * xa) * ya;
            dst[(size_t)y * w + x] = sat_u8(cv_round_f(res));
        }
    }
    free(lut);
}
