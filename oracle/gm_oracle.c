/* gm_oracle.c -- TEST AND MEASUREMENT INFRASTRUCTURE ONLY.  A sequential restatement of the reference's grid_mapping tool
 * (support_files/grid_mapping: main.cpp:114-119, grid_mapper.cpp, grid_map.cpp), one point and one ray step at a time, with no
 * shortcut.  Built -O3 -ffp-contract=off -msse2 -mfpmath=sse: every double operation rounds once, as the tool's -O2 x86-64 build.
 *
 * mode 0 (libm): the tool's arithmetic on this host (glibc log / exp).  mode 1 (shared): the log / exp of
 * ground_fusion_b200/csrc/gm_math.h, which the GPU grid (gm_grid.cu) uses; the GPU equals this mode bit for bit. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../ground_fusion_b200/csrc/gm_math.h"

#define Z_LO 0.1                                  /* main.cpp:117: kept iff !(z > 0.5 || z < 0.1) */
#define Z_HI 0.5

typedef struct {
    int sx, sy, ix, iy, shared;
    double cs, p[3], c[3];                        /* p, log(p / (1 - p)) by kind: 0 free, 1 occupied, 2 prior */
    double ric[9], tic[3];
    double* bel;                                  /* column-major bel(x, y) at x + sx * y */
    int n_kf, cap_kf;
    double* poses;                                /* [n_kf][12]: R row-major, P */
    int* kf_off;                                  /* keyframe k's points are [kf_off[k], kf_off[k + 1]) */
    float* pts;                                   /* [n][3] camera-frame points */
    int n_pts, cap_pts;
} gmo;

static double gmo_lg(const gmo* g, double x) { return g->shared ? gm_log(x) : log(x); }
static double gmo_ex(const gmo* g, double x) { return g->shared ? gm_exp(x) : exp(x); }

double gmo_log(double x) { return gm_log(x); }
double gmo_exp(double x) { return gm_exp(x); }

static void mv3(const double* M, const double* x, double* y)
{
    const double y0 = M[0] * x[0] + M[1] * x[1] + M[2] * x[2];
    const double y1 = M[3] * x[0] + M[4] * x[1] + M[5] * x[2];
    const double y2 = M[6] * x[0] + M[7] * x[1] + M[8] * x[2];
    y[0] = y0; y[1] = y1; y[2] = y2;
}

gmo* gmo_create(int sx, int sy, int ix, int iy, double cs, double p_occ, double p_free, double p_prior, const double* ric,
                const double* tic, int shared)
{
    gmo* g = (gmo*)calloc(1, sizeof(gmo));
    g->sx = sx; g->sy = sy; g->ix = ix; g->iy = iy; g->cs = cs; g->shared = shared;
    g->p[0] = p_free; g->p[1] = p_occ; g->p[2] = p_prior;
    for (int k = 0; k < 3; k++) g->c[k] = gmo_lg(g, g->p[k] / (1.0 - g->p[k]));
    memcpy(g->ric, ric, sizeof(g->ric)); memcpy(g->tic, tic, sizeof(g->tic));
    g->bel = (double*)malloc(sizeof(double) * (size_t)sx * sy);
    for (size_t i = 0; i < (size_t)sx * sy; i++) g->bel[i] = 0.5;
    g->cap_kf = 16;
    g->poses = (double*)malloc(sizeof(double) * 12 * g->cap_kf);
    g->kf_off = (int*)malloc(sizeof(int) * (g->cap_kf + 1));
    g->kf_off[0] = 0;
    return g;
}

void gmo_destroy(gmo* g)
{
    if (!g) return;
    free(g->bel); free(g->poses); free(g->kf_off); free(g->pts); free(g);
}

/* GridMap::getIdx (grid_map.cpp:19-32) with GridMapper::updateGrid (grid_mapper.cpp:38-46) */
static void gmo_update(gmo* g, double x, double y, int kind)
{
    const double fx = floor(x / g->cs), fy = floor(y / g->cs);
    if (!(fx >= -(double)g->ix && fx < (double)(g->sx - g->ix) && fy >= -(double)g->iy && fy < (double)(g->sy - g->iy))) return;
    double* b = g->bel + ((size_t)((int)fx + g->ix) + (size_t)g->sx * (size_t)((int)fy + g->iy));
    double l = gmo_lg(g, *b / (1.0 - *b));
    l += g->c[kind];
    *b = 1.0 - 1.0 / (1 + gmo_ex(g, l));
}

/* GridMapper::updateMap (grid_mapper.cpp:12-36) from the body position (T0, T1) to the world point (px, py) */
static void gmo_ray(gmo* g, double px, double py, double T0, double T1)
{
    const double cs = g->cs;
    const double dx = px - T0, dy = py - T1;
    const double z = sqrt(dy * dy + dx * dx);
    const double cosz = dx / z, sinz = dy / z;
    double lx = -1.0, ly = -1.0;                  /* Eigen::Infinity is the integer -1 */
    for (double r = 0; r < z + cs; r += cs) {
        const double wx = r * cosz + T0, wy = r * sinz + T1;
        if (wx == lx && wy == ly) continue;
        const int kind = r < (z - 0.5 * cs) ? 0 : (r > (z + 0.5 * cs) ? 2 : 1);      /* laserInvModel, :48-57 */
        gmo_update(g, wx, wy, kind);
        lx = wx; ly = wy;
    }
}

/* main.cpp:114-120 over one keyframe's points */
static void gmo_apply(gmo* g, int k)
{
    const double* T = g->poses + 12 * (size_t)k;
    for (int i = g->kf_off[k]; i < g->kf_off[k + 1]; i++) {
        const float* l = g->pts + 3 * (size_t)i;
        const double p[3] = {(double)l[0], (double)l[1], (double)l[2]};
        double a[3], b[3], w[3];
        mv3(g->ric, p, a);
        for (int j = 0; j < 3; j++) a[j] = a[j] + g->tic[j];
        mv3(T, a, b);
        for (int j = 0; j < 3; j++) w[j] = b[j] + T[9 + j];
        if (w[2] > Z_HI || w[2] < Z_LO) continue;
        gmo_ray(g, w[0], w[1], T[9], T[10]);
    }
}

/* pts: n rows of stride floats, x y z first */
int gmo_add_keyframe(gmo* g, const double* R, const double* P, const float* pts, int n, int stride)
{
    if (g->n_kf == g->cap_kf) {
        g->cap_kf *= 2;
        g->poses = (double*)realloc(g->poses, sizeof(double) * 12 * g->cap_kf);
        g->kf_off = (int*)realloc(g->kf_off, sizeof(int) * (g->cap_kf + 1));
    }
    if (g->n_pts + n > g->cap_pts) {
        g->cap_pts = 2 * (g->n_pts + n) + 16;
        g->pts = (float*)realloc(g->pts, sizeof(float) * 3 * (size_t)g->cap_pts);
    }
    for (int i = 0; i < n; i++)
        for (int j = 0; j < 3; j++) g->pts[3 * (size_t)(g->n_pts + i) + j] = pts[(size_t)stride * i + j];
    g->n_pts += n;
    memcpy(g->poses + 12 * (size_t)g->n_kf, R, 9 * sizeof(double));
    memcpy(g->poses + 12 * (size_t)g->n_kf + 9, P, 3 * sizeof(double));
    g->kf_off[g->n_kf + 1] = g->n_pts;
    g->n_kf++;
    gmo_apply(g, g->n_kf - 1);
    return 0;
}

/* a fresh grid at 0.5, every keyframe applied again in order with its new pose */
int gmo_update_poses(gmo* g, int n, const double* R, const double* P)
{
    if (n != g->n_kf) return -1;
    for (int k = 0; k < n; k++) {
        memcpy(g->poses + 12 * (size_t)k, R + 9 * (size_t)k, 9 * sizeof(double));
        memcpy(g->poses + 12 * (size_t)k + 9, P + 3 * (size_t)k, 3 * sizeof(double));
    }
    for (size_t i = 0; i < (size_t)g->sx * g->sy; i++) g->bel[i] = 0.5;
    for (int k = 0; k < n; k++) gmo_apply(g, k);
    return 0;
}

int gmo_n_keyframes(const gmo* g) { return g->n_kf; }

void gmo_read_bel(const gmo* g, double* out) { memcpy(out, g->bel, sizeof(double) * (size_t)g->sx * g->sy); }

/* GridMap::saveMap (grid_map.cpp:74-87, 113-118): m = 1 - bel, eigen2cv (rows = x), flip (rows reversed), * 255, and imwrite's
 * conversion of the double image to 8 bits (round half to even, saturate).  out: (sx, sy) row-major. */
static uint8_t gmo_pixel(double bel)
{
    const double v = rint((1.0 - bel) * 255.0);
    return v <= 0 ? 0 : (v >= 255 ? 255 : (uint8_t)v);
}
void gmo_image(const gmo* g, uint8_t* out)
{
    for (int x = 0; x < g->sx; x++)
        for (int y = 0; y < g->sy; y++) out[(size_t)(g->sx - 1 - x) * g->sy + y] = gmo_pixel(g->bel[x + (size_t)g->sx * y]);
}

/* pose_graph_node.cpp:865-899 over the pixels saveMap wrote: flip back, convertTo(CV_32F, 1 / 255.0), value = 1 - v in double;
 * -1 unless |value - 0.5| > 0.005, else (signed char)(value * 100) at data[sx * y + x] */
void gmo_occupancy(const gmo* g, int8_t* out)
{
    const float s = (float)(1 / 255.0);
    for (size_t i = 0; i < (size_t)g->sx * g->sy; i++) {
        const float v = (float)gmo_pixel(g->bel[i]) * s;
        const double value = 1.0 - 1.0 * v;
        out[i] = fabs(value - 0.5) > 0.005 ? (int8_t)(value * 100) : -1;
    }
}
