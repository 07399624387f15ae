/*
 * TEST INFRASTRUCTURE ONLY -- CPU restatement of the exact 3-nearest-neighbour mean distance that
 * `simple_knn._C.distCUDA2` returns (contract: include/gh_rasterizer.h, DESIGN §14), used to CHECK
 * gaussianhaircut_b200/csrc/gh_knn.cu.  Compiled with -ffp-contract=off (oracle/knn_oracle.py): every float32
 * operation is rounded on its own, as in the kernels.
 *
 * The neighbour search is a k-d tree over the finite points, independent of the product's Morton-ordered box tree:
 * median splits on the widest axis down to buckets of at most 8 points, nearest side first.  The far side of a split
 * at value v is skipped only when fl(d*d) >= b2 with d = fl(p - v): every point q beyond the plane has
 * |fl(q - p)| >= |d| (rounding is monotone and symmetric), so its float32 squared distance is >= fl(d*d) >= b2 and it
 * cannot be among the three smallest (a value equal to b2 never changes them).  Exact by construction.
 */
#include <math.h>
#include <stdlib.h>

typedef struct {
    float c[3];
    int idx;
} KPt;

typedef struct {
    int lo, hi;          /* bucket [lo, hi) of the point array (leaves) */
    int axis;            /* -1: leaf */
    float split;
    int left, right;
} KNode;

typedef struct {
    KPt* pts;
    KNode* nodes;
    int n_nodes;
} KTree;

#define KNN_BUCKET 8

static float knn_dist2(const float* p, const float* q)
{
    const float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
    return (dx * dx + dy * dy) + dz * dz;
}

static void knn_insert(float s, float* b)
{
    if (s < b[2]) {
        if (s < b[1]) {
            b[2] = b[1];
            if (s < b[0]) { b[1] = b[0]; b[0] = s; } else { b[1] = s; }
        } else {
            b[2] = s;
        }
    }
}

static void knn_swap(KPt* a, int i, int j)
{
    const KPt t = a[i]; a[i] = a[j]; a[j] = t;
}

static float knn_median3(float a, float b, float c)
{
    if (a > b) { const float t = a; a = b; b = t; }
    if (b > c) b = c;
    return a > b ? a : b;
}

/* a[k] becomes the k-th smallest of a[lo, hi) on `ax`, smaller-or-equal before it and greater-or-equal after it.
 * Three-way partitions keep runs of equal coordinates (lattices, duplicates) linear. */
static void knn_select(KPt* a, int lo, int hi, int k, int ax)
{
    while (hi - lo > 1) {
        const float pv = knn_median3(a[lo].c[ax], a[lo + (hi - lo) / 2].c[ax], a[hi - 1].c[ax]);
        int lt = lo, i = lo, gt = hi;
        while (i < gt) {
            const float v = a[i].c[ax];
            if (v < pv) knn_swap(a, lt++, i++);
            else if (v > pv) knn_swap(a, i, --gt);
            else i++;
        }
        if (k < lt) hi = lt;
        else if (k >= gt) lo = gt;
        else return;
    }
}

static int knn_build(KTree* t, int lo, int hi)
{
    const int id = t->n_nodes++;
    KNode* n = &t->nodes[id];
    n->lo = lo; n->hi = hi; n->axis = -1; n->left = n->right = -1; n->split = 0.f;
    if (hi - lo <= KNN_BUCKET) return id;
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = lo; i < hi; i++)
        for (int k = 0; k < 3; k++) {
            const float v = t->pts[i].c[k];
            if (v < mn[k]) mn[k] = v;
            if (v > mx[k]) mx[k] = v;
        }
    int ax = 0;
    double best = (double)mx[0] - (double)mn[0];
    for (int k = 1; k < 3; k++)
        if ((double)mx[k] - (double)mn[k] > best) { best = (double)mx[k] - (double)mn[k]; ax = k; }
    const int mid = lo + (hi - lo) / 2;
    knn_select(t->pts, lo, hi, mid, ax);
    const float split = t->pts[mid].c[ax];
    const int left = knn_build(t, lo, mid);
    const int right = knn_build(t, mid, hi);
    n = &t->nodes[id];              /* (the array does not move: sized up front) */
    n->axis = ax; n->split = split; n->left = left; n->right = right;
    return id;
}

static void knn_query(const KTree* t, int id, const float* p, int self, float* b)
{
    const KNode* n = &t->nodes[id];
    if (n->axis < 0) {
        for (int j = n->lo; j < n->hi; j++)
            if (t->pts[j].idx != self) knn_insert(knn_dist2(p, t->pts[j].c), b);
        return;
    }
    const float d = p[n->axis] - n->split;
    const int near = d < 0.f ? n->left : n->right, far = d < 0.f ? n->right : n->left;
    knn_query(t, near, p, self, b);
    if (b[2] == 0.f) return;
    if (d * d < b[2]) knn_query(t, far, p, self, b);
}

/* out[i] for i < P; returns 0, or -1 when memory runs out. */
int gho_knn_mean_dist3(long long P, const float* points, float* out)
{
    int nf = 0;
    for (long long i = 0; i < P; i++)
        if (isfinite(points[3 * i]) && isfinite(points[3 * i + 1]) && isfinite(points[3 * i + 2])) nf++;
    KTree t;
    t.n_nodes = 0;
    t.pts = (KPt*)malloc(sizeof(KPt) * (size_t)(nf > 0 ? nf : 1));
    t.nodes = (KNode*)malloc(sizeof(KNode) * (size_t)(2 * (nf / (KNN_BUCKET / 2) + 1) + 1));
    if (!t.pts || !t.nodes) { free(t.pts); free(t.nodes); return -1; }
    int m = 0;
    for (long long i = 0; i < P; i++) {
        const float* q = points + 3 * i;
        if (isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2])) {
            t.pts[m].c[0] = q[0]; t.pts[m].c[1] = q[1]; t.pts[m].c[2] = q[2]; t.pts[m].idx = (int)i;
            m++;
        } else {
            out[i] = NAN;
        }
    }
    if (nf > 0) knn_build(&t, 0, nf);
#pragma omp parallel for schedule(dynamic, 4096)
    for (int k = 0; k < nf; k++) {
        float b[3] = {INFINITY, INFINITY, INFINITY};
        knn_query(&t, 0, t.pts[k].c, t.pts[k].idx, b);
        out[t.pts[k].idx] = ((b[0] + b[1]) + b[2]) / 3.0f;
    }
    free(t.pts);
    free(t.nodes);
    return 0;
}
