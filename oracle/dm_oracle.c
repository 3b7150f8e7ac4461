/* dm_oracle.c -- sequential restatement of dense_map's colour map (test and measurement infrastructure only):
 *   pose_graph_node.cpp:598-623  keyframe point sampling
 *   pose_graph.cpp:191-221       insertion: z band, OctreePointCloudDensity(0.01) gate < 3, keyframe list compacted
 *   pose_graph.cpp:228-239       RadiusOutlierRemoval(0.8, 10)
 *   pose_graph.cpp:997-1058      updatePath: fresh octree over the wider box, gate < 5, no z band, filter again
 * One point at a time in the reference's order.  PCL is not vendored; the octree box anchoring, the density and the radius
 * filter are stated from PCL 1.10 (unverified) in dmo_anchor, the voxel hash and dmo_radius_filter.
 * Built with -ffp-contract=off: every double and float operation rounds separately, as the reference does without FMA. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define VOXEL 0.01
#define EMPTY_KEY (~0ull)

typedef struct { uint64_t* key; int* val; size_t mask; size_t n; } hmap;

static size_t hh(uint64_t k, size_t mask)
{
    k ^= k >> 31; k *= 0x9e3779b97f4a7c15ull; k ^= k >> 29;
    return (size_t)k & mask;
}
static void hm_init(hmap* h, size_t cap)
{
    size_t c = 64;
    while (c < 2 * cap) c <<= 1;
    h->key = malloc(8 * c); h->val = malloc(4 * c); h->mask = c - 1; h->n = 0;
    memset(h->key, 0xff, 8 * c);
}
static void hm_free(hmap* h) { free(h->key); free(h->val); memset(h, 0, sizeof(*h)); }
static int* hm_get(hmap* h, uint64_t k, int insert)
{
    if (insert && 2 * (h->n + 1) > h->mask + 1) {          /* grow */
        hmap g; hm_init(&g, 2 * (h->mask + 1));
        for (size_t s = 0; s <= h->mask; s++) if (h->key[s] != EMPTY_KEY) { *hm_get(&g, h->key[s], 1) = h->val[s]; }
        hm_free(h); *h = g;
    }
    for (size_t s = hh(k, h->mask);; s = (s + 1) & h->mask) {
        if (h->key[s] == k) return &h->val[s];
        if (h->key[s] == EMPTY_KEY) {
            if (!insert) return NULL;
            h->key[s] = k; h->val[s] = 0; h->n++;
            return &h->val[s];
        }
    }
}

/* PCL 1.10 OctreePointCloud::getKeyBitSize on an empty tree: the box is widened symmetrically to 2^depth voxels per axis */
void dmo_anchor(int rebuild, double* mn, double* mx)
{
    const double lo[3] = {-10000, rebuild ? -10000 : -1000, -10000}, hi[3] = {10000, 10000, 10000};
    const float min_value = FLT_EPSILON;
    unsigned mk[3], mv = 2;
    for (int a = 0; a < 3; a++) { mk[a] = (unsigned)ceil((hi[a] - lo[a] - min_value) / VOXEL); if (mk[a] > mv) mv = mk[a]; }
    unsigned depth = (unsigned)ceil(log2((double)mv) - min_value);
    if (depth > 32) depth = 32;
    const double side = (double)(1ull << depth) * VOXEL;
    for (int a = 0; a < 3; a++) { const double o = (side - (hi[a] - lo[a])) / 2.0; mn[a] = lo[a] - o; mx[a] = hi[a] + o; }
}

typedef struct {
    int w, h, dd, db;
    double cam[8]; int nodist;
    double ric[9], tic[3];
    double mn[3], mx[3];
    hmap vox;
    /* cloud */
    float* cxyz; uint8_t* crgb; uint8_t* keep; int n, cap;
    /* keyframes: kept local points (x y z r g b) */
    float* kp; int* kid; int nk, kcap; int* koff; int nkf, kfcap;
} dm_oracle;

static void lift(const dm_oracle* m, double u, double v, double* ox, double* oy)
{   /* PinholeCamera::liftProjective (recursive distortion, n = 8) */
    const double fx = m->cam[0], fy = m->cam[1], cx = m->cam[2], cy = m->cam[3], k1 = m->cam[4], k2 = m->cam[5], p1 = m->cam[6], p2 = m->cam[7];
    const double mx_d = (1.0 / fx) * u + (-cx / fx), my_d = (1.0 / fy) * v + (-cy / fy);
    if (m->nodist) { *ox = mx_d; *oy = my_d; return; }
    double x = mx_d, y = my_d;
    for (int i = 0; i < 8; i++) {
        const double mx2 = x * x, my2 = y * y, mxy = x * y, rho2 = mx2 + my2, rad = k1 * rho2 + k2 * rho2 * rho2;
        const double dx = x * rad + 2.0 * p1 * mxy + p2 * (rho2 + 2.0 * mx2), dy = y * rad + 2.0 * p2 * mxy + p1 * (rho2 + 2.0 * my2);
        x = mx_d - dx; y = my_d - dy;
    }
    *ox = x; *oy = y;
}
static void world(const dm_oracle* m, const double* R, const double* P, const float* l, double* w)
{   /* R * (qic * point + tic) + P, Eigen's 3x3 products without FMA */
    const double p[3] = {l[0], l[1], l[2]};
    double a[3];
    for (int i = 0; i < 3; i++) a[i] = (m->ric[3 * i] * p[0] + m->ric[3 * i + 1] * p[1] + m->ric[3 * i + 2] * p[2]) + m->tic[i];
    for (int i = 0; i < 3; i++) w[i] = (R[3 * i] * a[0] + R[3 * i + 1] * a[1] + R[3 * i + 2] * a[2]) + P[i];
}
/* voxel key of a float point; -1 when outside the anchored box */
static int vkey(const dm_oracle* m, const float* f, uint64_t* key)
{
    uint64_t k = 0;
    for (int a = 0; a < 3; a++) {
        const double x = f[a];
        if (!(x >= m->mn[a] && x < m->mx[a])) return -1;
        k = (k << 21) | (uint64_t)(unsigned)((x - m->mn[a]) / VOXEL);
    }
    *key = k;
    return 0;
}
static void cloud_push(dm_oracle* m, const float* f, const uint8_t* c)
{
    if (m->n == m->cap) {
        m->cap = m->cap ? 2 * m->cap : 4096;
        m->cxyz = realloc(m->cxyz, 12 * (size_t)m->cap); m->crgb = realloc(m->crgb, 3 * (size_t)m->cap); m->keep = realloc(m->keep, m->cap);
    }
    memcpy(m->cxyz + 3 * (size_t)m->n, f, 12); memcpy(m->crgb + 3 * (size_t)m->n, c, 3);
    m->n++;
}

dm_oracle* dmo_create(int w, int h, const double* pinhole, int depth_dist, int depth_boundary, const double* ric, const double* tic)
{
    dm_oracle* m = calloc(1, sizeof(dm_oracle));
    m->w = w; m->h = h; m->dd = depth_dist; m->db = depth_boundary;
    memcpy(m->cam, pinhole, 64); memcpy(m->ric, ric, 72); memcpy(m->tic, tic, 24);
    m->nodist = pinhole[4] == 0.0 && pinhole[5] == 0.0 && pinhole[6] == 0.0 && pinhole[7] == 0.0;
    dmo_anchor(0, m->mn, m->mx);
    hm_init(&m->vox, 1024);
    m->koff = malloc(sizeof(int) * 16); m->kfcap = 16; m->koff[0] = 0;
    return m;
}
void dmo_destroy(dm_oracle* m)
{
    if (!m) return;
    hm_free(&m->vox);
    free(m->cxyz); free(m->crgb); free(m->keep); free(m->kp); free(m->kid); free(m->koff); free(m);
}

/* RadiusOutlierRemoval (PCL 1.10, unverified): keep iff more than min_pts points (itself and duplicates included) lie at
 * FLANN's float distance ((dx*dx) + dy*dy) + dz*dz < float(radius^2).  Exact count over a grid of 1 m cells (>= radius). */
typedef struct { uint64_t k; int i; } cell_ent;
static int cmp_cell(const void* a, const void* b)
{
    const cell_ent *x = a, *y = b;
    return x->k < y->k ? -1 : x->k > y->k ? 1 : x->i - y->i;
}
static uint64_t ckey(long cx, long cy, long cz) { return ((uint64_t)(cx + (1 << 20)) << 42) | ((uint64_t)(cy + (1 << 20)) << 21) | (uint64_t)(cz + (1 << 20)); }
void dmo_radius_filter(const float* xyz, int n, double radius, int min_pts, uint8_t* keep)
{
    if (n <= 0) return;
    const double cell = radius > 1.0 ? radius * 1.25 : 1.0;
    const float r2 = (float)(radius * radius);
    cell_ent* e = malloc(sizeof(cell_ent) * (size_t)n);
    for (int i = 0; i < n; i++)
        e[i].k = ckey((long)floor(xyz[3 * i] / cell), (long)floor(xyz[3 * i + 1] / cell), (long)floor(xyz[3 * i + 2] / cell)), e[i].i = i;
    qsort(e, n, sizeof(cell_ent), cmp_cell);
    hmap start; hm_init(&start, n);
    for (int j = 0; j < n; j++) if (j == 0 || e[j].k != e[j - 1].k) *hm_get(&start, e[j].k, 1) = j;
    for (int i = 0; i < n; i++) {
        const float* q = xyz + 3 * (size_t)i;
        const long cx = (long)floor(q[0] / cell), cy = (long)floor(q[1] / cell), cz = (long)floor(q[2] / cell);
        int cnt = 0;
        for (long a = -1; a <= 1; a++) for (long b = -1; b <= 1; b++) for (long c = -1; c <= 1; c++) {
            const uint64_t k = ckey(cx + a, cy + b, cz + c);
            const int* s = hm_get(&start, k, 0);
            if (!s) continue;
            for (int j = *s; j < n && e[j].k == k; j++) {
                const float* p = xyz + 3 * (size_t)e[j].i;
                const float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
                if ((dx * dx + dy * dy) + dz * dz < r2 && ++cnt > min_pts) goto counted;     /* the search's cap: min_pts + 1 */
            }
        }
    counted:
        keep[i] = cnt > min_pts;
    }
    hm_free(&start);
    free(e);
}

/* one keyframe; returns the number of points inserted, -1 when a point falls outside the octree's box (nothing changed).
 * filter = 0 skips the filter (the filter of a cloud depends on the cloud alone; dmo_filter runs it later). */
int dmo_add_keyframe(dm_oracle* m, const double* R, const double* P, const uint8_t* rgb, size_t rgb_pitch, const uint16_t* depth, size_t depth_pitch, int filter)
{
    int ins = 0;
    /* pass 0 checks the box so that a failing keyframe changes nothing, pass 1 inserts */
    for (int pass = 0; pass < 2; pass++)
        for (int v = m->db; v < m->h - m->db; v += m->dd)
            for (int u = m->db; u < m->w - m->db; u += m->dd) {
                const uint8_t* c = rgb + (size_t)v * rgb_pitch + 3 * (size_t)u;
                float d = (float)(int)*(const uint16_t*)((const uint8_t*)depth + (size_t)v * depth_pitch + 2 * (size_t)u);
                d = d / 1000;
                const float r = c[0], g = c[1], b = c[2];
                if (r > 240 && g > 240 && b > 240) continue;
                if (d < 0.1 || d >= 7.0) continue;
                double ax, ay;
                lift(m, u, v, &ax, &ay);
                const float l[3] = {(float)(ax * d), (float)(ay * d), d};
                double w[3];
                world(m, R, P, l, w);
                if (w[2] > 2 || w[2] < -0.5) continue;
                const float f[3] = {(float)w[0], (float)w[1], (float)w[2]};
                uint64_t k;
                if (vkey(m, f, &k)) { if (pass == 0) return -1; continue; }
                if (pass == 0) continue;
                int* cnt = hm_get(&m->vox, k, 1);
                if (*cnt < 3) {
                    (*cnt)++;
                    cloud_push(m, f, c);
                    if (m->nk == m->kcap) { m->kcap = m->kcap ? 2 * m->kcap : 4096; m->kp = realloc(m->kp, 24 * (size_t)m->kcap); m->kid = realloc(m->kid, 4 * (size_t)m->kcap); }
                    float* o = m->kp + 6 * (size_t)m->nk;
                    o[0] = l[0]; o[1] = l[1]; o[2] = l[2]; o[3] = r; o[4] = g; o[5] = b;
                    m->kid[m->nk++] = m->nkf;
                    ins++;
                }
            }
    if (m->nkf + 2 > m->kfcap) { m->kfcap *= 2; m->koff = realloc(m->koff, sizeof(int) * (size_t)m->kfcap); }
    m->koff[++m->nkf] = m->nk;
    if (filter) dmo_radius_filter(m->cxyz, m->n, 0.8, 10, m->keep);
    return ins;
}

void dmo_filter(dm_oracle* m) { dmo_radius_filter(m->cxyz, m->n, 0.8, 10, m->keep); }

/* updatePath; returns the cloud size, -1 when a point falls outside the box or n differs from the keyframe count (nothing changed) */
int dmo_update_poses(dm_oracle* m, int n, const double* R, const double* P, int filter)
{
    if (n != m->nkf) return -1;
    dm_oracle t = *m;
    dmo_anchor(1, t.mn, t.mx);
    for (int i = 0; i < m->nk; i++) {
        double w[3];
        world(&t, R + 9 * (size_t)m->kid[i], P + 3 * (size_t)m->kid[i], m->kp + 6 * (size_t)i, w);
        const float f[3] = {(float)w[0], (float)w[1], (float)w[2]};
        uint64_t k;
        if (vkey(&t, f, &k)) return -1;
    }
    memcpy(m->mn, t.mn, sizeof(m->mn)); memcpy(m->mx, t.mx, sizeof(m->mx));
    hm_free(&m->vox); hm_init(&m->vox, 1024);
    m->n = 0;
    for (int i = 0; i < m->nk; i++) {
        const float* l = m->kp + 6 * (size_t)i;
        double w[3];
        world(m, R + 9 * (size_t)m->kid[i], P + 3 * (size_t)m->kid[i], l, w);
        const float f[3] = {(float)w[0], (float)w[1], (float)w[2]};
        uint64_t k;
        vkey(m, f, &k);
        int* cnt = hm_get(&m->vox, k, 1);
        if (*cnt < 5) {
            (*cnt)++;
            const uint8_t c[3] = {(uint8_t)l[3], (uint8_t)l[4], (uint8_t)l[5]};
            cloud_push(m, f, c);
        }
    }
    if (filter) dmo_filter(m);
    return m->n;
}

void dmo_size(const dm_oracle* m, int* n_cloud, int* n_filtered, int* n_kf)
{
    int f = 0;
    for (int i = 0; i < m->n; i++) f += m->keep[i];
    *n_cloud = m->n; *n_filtered = f; *n_kf = m->nkf;
}
void dmo_read(const dm_oracle* m, float* xyz, uint8_t* rgb, uint8_t* keep)
{
    if (!m->n) return;
    memcpy(xyz, m->cxyz, 12 * (size_t)m->n); memcpy(rgb, m->crgb, 3 * (size_t)m->n); memcpy(keep, m->keep, m->n);
}
int dmo_keyframe_points(const dm_oracle* m, int k, float* out6)
{
    if (k < 0 || k >= m->nkf) return -1;
    const int c = m->koff[k + 1] - m->koff[k];
    if (out6 && c) memcpy(out6, m->kp + 6 * (size_t)m->koff[k], 24 * (size_t)c);
    return c;
}
