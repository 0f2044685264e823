// Delaunay adjacency of a point set by per-cell Voronoi clipping in fp64 (rfb_delaunay_count / rfb_delaunay_write).
//
// Definition (include/radfoam_b200.h): {i, j} is an edge iff the face F_ij = { x in B : |x - p_i| = |x - p_j| <=
// |x - p_k| for all k } has positive area.  Each cell C_i = B ∩ (half-spaces of its neighbours' bisector planes) is
// built on its own, relative to p_i, as a list of face planes plus the vertices of their polygons:
//   * a face's polygon = a square on its plane, clipped by the box and by every other face plane (clip_polygon);
//   * a candidate q (sorted points, nearest first) is added as a face plane only when some current vertex lies
//     beyond its bisector; the polygons are rebuilt every few additions, and planes whose polygon vanished dropped;
//   * stop rule: once the next candidate is farther than 2R, R the largest distance from p_i to a vertex of the
//     current cell, no later candidate can cut the cell (its bisector is more than R from p_i).  Candidate order and
//     the k of the first k-nearest query change only the speed.
// The fast kernel runs a thread per cell with fixed capacities; a cell that exceeds one of them (hull cells bounded
// only by B see every point within 2R, hubs have many faces) goes to the overflow kernel, a warp per cell with its
// face and vertex lists in a per-warp slice of global scratch.  A face is kept when its polygon's area exceeds
// kDelFaceArea |p_i - p_j|^2: zero-area faces at co-spherical ties may be found from one end and not the other, and
// the assembly takes the union of both ends' findings, so the graph is symmetric whatever each end decided.
#pragma once

namespace rfb {

constexpr int kDelLeaf = 8;            // points per leaf of the implicit tree
constexpr int kDelKnn = 32;            // fast kernel: candidates per round, the next k nearest
constexpr int kDelRounds = 4;          // fast kernel: nearest-first rounds before the vertex-ball walk
constexpr int kDelFaces = 48;          // fast kernel: face planes of a cell at once
constexpr int kDelVerts = 256;         // fast kernel: vertices of the current cell (per face polygon, so repeated)
constexpr int kDelPolyVerts = 32;      // fast kernel: vertices of one polygon while it is clipped
constexpr int kDelOvfPolyVerts = 96;   // overflow kernel: the same
constexpr int kDelOvfFaces = 4096;     // overflow kernel: face planes per cell (per-warp scratch)
constexpr int kDelOvfVerts = 12288;    // overflow kernel: vertices per cell (per-warp scratch)
constexpr int kDelOvfWarps = 512;      // overflow kernel: at most this many warps (4 per SM), one scratch slice each
constexpr int kDelOvfPointsPerWarp = 1024; // overflow kernel: one warp (and slice) per this many points, up to the cap
constexpr int kDelOvfBatch = 16;       // overflow kernel: face planes added between polygon rebuilds
constexpr int kDelBlock = 128;
constexpr int kDelRebuild = 4;         // fast kernel: face planes added between polygon rebuilds
constexpr double kDelFaceArea = 1e-10; // a face is kept when area > kDelFaceArea |p_i - p_j|^2
constexpr double kDelSlack = 1e-9;     // relative slack of the stop rule (vertices carry fp64 rounding)
constexpr double kDelCutMargin = 1e-12; // a vertex within kDelCutMargin R |q| of a bisector counts as beyond it
constexpr uint32_t kDelBoxPlane = 0xFFFFFFF0u; // plane ids kDelBoxPlane + c, c < 6: x_c <= hi_c (c < 3), x_c >= lo_c
constexpr uint32_t kDelNone = 0xFFFFFFFFu;

// totals[] of a build (uint64): [0] entries added from one end only, [1] edges E (both written by the scan),
// [2] face entries the cells need in the pool, [3] cells sent to the overflow kernel, [4] duplicate points found,
// [5] non-finite points, [6] cells over the overflow kernel's capacity, [7] entries of `order` that are out of range
// or repeated (not a permutation).
enum { kDelOneSided = 0, kDelEdges = 1, kDelPoolNeed = 2, kDelOverflow = 3, kDelDuplicate = 4, kDelNonFinite = 5,
       kDelOverCapacity = 6, kDelBadOrder = 7, kDelTotals = 8 };

struct DelaunayParams {
    const float *points;   // [N][3] in the locality order
    const float *tree;     // [2 P][6] node boxes (lo, hi); node 1 is the root, node P + l is leaf l
    uint32_t n, pow2;      // N, P = leaf count rounded up to a power of two
    float lo[3], hi[3];    // the box B
};

// ---------------------------------------------------------------------------------------------- order and tree
// `seen` (N u32, zeroed) checks that order is a permutation.
__global__ void __launch_bounds__(kDelBlock) delaunay_gather_kernel(const float *__restrict__ points,
                                                                    const uint32_t *__restrict__ order, uint32_t n,
                                                                    float *__restrict__ sorted,
                                                                    uint32_t *__restrict__ seen,
                                                                    unsigned long long *__restrict__ totals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const uint32_t s = order[i];
    if (s >= n || atomicExch(seen + s, 1u) != 0u)
        atomicAdd(totals + kDelBadOrder, 1ull);
    bool finite = true;
    for (int c = 0; c < 3; ++c) {
        const float x = s < n ? points[3 * (uint64_t)s + c] : 0.0f;
        finite = finite && isfinite(x);
        sorted[3 * (uint64_t)i + c] = x;
    }
    if (!finite)
        atomicAdd(totals + kDelNonFinite, 1ull);
}

// Leaf l covers the sorted points [l L, min((l + 1) L, N)); leaves past the points get an empty box (lo > hi).
__global__ void __launch_bounds__(kDelBlock) delaunay_leaf_kernel(const float *__restrict__ sorted, uint32_t n,
                                                                  uint32_t pow2, float *__restrict__ tree) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= pow2)
        return;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    const uint64_t b = (uint64_t)l * kDelLeaf, e = b + kDelLeaf < n ? b + kDelLeaf : n;
    for (uint64_t k = b; k < e; ++k)
        for (int c = 0; c < 3; ++c) {
            lo[c] = fminf(lo[c], sorted[3 * k + c]);
            hi[c] = fmaxf(hi[c], sorted[3 * k + c]);
        }
    float *node = tree + 6 * ((uint64_t)pow2 + l);
    for (int c = 0; c < 3; ++c) {
        node[c] = lo[c];
        node[3 + c] = hi[c];
    }
}

// Internal nodes [first, 2 first): the union of their two children (one launch per level, bottom-up).
__global__ void __launch_bounds__(kDelBlock) delaunay_level_kernel(uint32_t first, float *__restrict__ tree) {
    const uint32_t k = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= 2 * first)
        return;
    const float *a = tree + 6 * (2 * (uint64_t)k), *b = a + 6;
    float *node = tree + 6 * (uint64_t)k;
    for (int c = 0; c < 3; ++c) {
        node[c] = fminf(a[c], b[c]);
        node[3 + c] = fmaxf(a[3 + c], b[3 + c]);
    }
}

// ---------------------------------------------------------------------------------------------- geometry
__device__ __forceinline__ void del_point(const DelaunayParams &P, uint32_t j, const double *pi, double *q) {
    for (int c = 0; c < 3; ++c)
        q[c] = (double)__ldg(P.points + 3 * (uint64_t)j + c) - pi[c];
}

__device__ __forceinline__ double del_box_dist2(const DelaunayParams &P, uint32_t node, const double *pi) {
    const float *b = P.tree + 6 * (uint64_t)node;
    double d2 = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double lo = __ldg(b + c), hi = __ldg(b + 3 + c);
        if (!(lo <= hi))
            return INFINITY; // empty leaf
        const double d = pi[c] < lo ? lo - pi[c] : (pi[c] > hi ? pi[c] - hi : 0.0);
        d2 += d * d;
    }
    return d2;
}

// Plane `id` relative to p_i as clip_polygon takes it, { x : (x - m).nrm <= 0 }: a box side, or the bisector of
// (p_i, p_id), whose nrm = q = p_id - p_i and m = q / 2.
__device__ __forceinline__ void del_plane(const DelaunayParams &P, const double *pi, uint32_t id, double *nrm,
                                          double *m) {
    if (id >= kDelBoxPlane) {
        const int c = (int)(id - kDelBoxPlane), a = c % 3;
        for (int k = 0; k < 3; ++k)
            nrm[k] = m[k] = 0.0;
        nrm[a] = c < 3 ? 1.0 : -1.0;
        m[a] = (c < 3 ? (double)P.hi[a] : (double)P.lo[a]) - pi[a];
        return;
    }
    del_point(P, id, pi, nrm);
    for (int k = 0; k < 3; ++k)
        m[k] = 0.5 * nrm[k];
}

// The polygon of plane `self` on the cell bounded by the box and the planes faces[0, nf): a square of half-width w
// around the plane's closest point to p_i, clipped by all of them.  w must exceed the cell's radius.  Returns the
// vertex count (0 when it vanished, -1 over PV) and points *poly at the vertices.
template <int PV>
__device__ int del_face_polygon(const DelaunayParams &P, const double *pi, uint32_t self, const uint32_t *faces,
                                int nf, double w, double (*a)[3], double (*b)[3], double (**poly)[3]) {
    double nrm[3], m[3];
    del_plane(P, pi, self, nrm, m);
    const double nn2 = nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2];
    const double t = (nrm[0] * m[0] + nrm[1] * m[1] + nrm[2] * m[2]) / nn2;
    const double nn = sqrt(nn2);
    const double ax = fabs(nrm[0]), ay = fabs(nrm[1]), az = fabs(nrm[2]);
    const int s = ax <= ay && ax <= az ? 0 : (ay <= az ? 1 : 2);
    double u[3] = {0.0, 0.0, 0.0};
    u[(s + 1) % 3] = nrm[(s + 2) % 3];
    u[(s + 2) % 3] = -nrm[(s + 1) % 3];
    const double un = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    for (int c = 0; c < 3; ++c)
        u[c] /= un;
    const double v[3] = {(nrm[1] * u[2] - nrm[2] * u[1]) / nn, (nrm[2] * u[0] - nrm[0] * u[2]) / nn,
                         (nrm[0] * u[1] - nrm[1] * u[0]) / nn};
    const double su[4] = {1.0, -1.0, -1.0, 1.0}, sv[4] = {1.0, 1.0, -1.0, -1.0};
    for (int k = 0; k < 4; ++k)
        for (int c = 0; c < 3; ++c)
            a[k][c] = t * nrm[c] + w * (su[k] * u[c] + sv[k] * v[c]);
    int n = 4;
    double(*cur)[3] = a, (*nxt)[3] = b;
    for (int k = -6; k < nf && n > 0; ++k) {
        const uint32_t id = k < 0 ? kDelBoxPlane + (uint32_t)(k + 6) : faces[k];
        if (id == self)
            continue;
        double pn[3], pm[3];
        del_plane(P, pi, id, pn, pm);
        n = clip_polygon<PV>(cur, n, nxt, pn, pm);
        double(*tmp)[3] = cur;
        cur = nxt;
        nxt = tmp;
    }
    *poly = cur;
    return n;
}

__device__ __forceinline__ double del_area(const double (*v)[3], int n) {
    double s[3] = {0.0, 0.0, 0.0};
    for (int k = 1; k + 1 < n; ++k) {
        double e1[3], e2[3];
        for (int c = 0; c < 3; ++c) {
            e1[c] = v[k][c] - v[0][c];
            e2[c] = v[k + 1][c] - v[0][c];
        }
        s[0] += e1[1] * e2[2] - e1[2] * e2[1];
        s[1] += e1[2] * e2[0] - e1[0] * e2[2];
        s[2] += e1[0] * e2[1] - e1[1] * e2[0];
    }
    return 0.5 * sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
}

// Does the bisector of q cut the cell whose vertices are vtx[0, nv)?  Conservative: a vertex within the margin of
// the plane counts as beyond it (a plane added needlessly is dropped at the next rebuild).
__device__ __forceinline__ bool del_cuts(const double (*vtx)[3], int nv, const double *q, double q2, double r) {
    const double lim = 0.5 * q2 - kDelCutMargin * r * sqrt(q2);
    for (int k = 0; k < nv; ++k)
        if (vtx[k][0] * q[0] + vtx[k][1] * q[1] + vtx[k][2] * q[2] > lim)
            return true;
    return false;
}

// del_cuts with the vertices shared among the lanes of a warp, which vote (every lane calls it with the same q).
__device__ __forceinline__ bool del_cuts_warp(const double (*vtx)[3], int nv, const double *q, double q2, double r) {
    const double lim = 0.5 * q2 - kDelCutMargin * r * sqrt(q2);
    bool cut = false;
    for (int k = (int)(threadIdx.x & 31u); k < nv && !cut; k += 32)
        cut = vtx[k][0] * q[0] + vtx[k][1] * q[1] + vtx[k][2] * q[2] > lim;
    return __any_sync(0xffffffffu, cut) != 0;
}

// The box's corners relative to p_i: the vertices of the cell before any bisector.
__device__ __forceinline__ double del_box_corners(const DelaunayParams &P, const double *pi, double (*vtx)[3]) {
    double r2 = 0.0;
    for (int k = 0; k < 8; ++k) {
        double d2 = 0.0;
        for (int c = 0; c < 3; ++c) {
            vtx[k][c] = (double)((k >> c) & 1 ? P.hi[c] : P.lo[c]) - pi[c];
            d2 += vtx[k][c] * vtx[k][c];
        }
        r2 = fmax(r2, d2);
    }
    return r2;
}

// Can a point of the node's box lie in the ball of some vertex v (centre v, radius |v|, p_i at the origin)?  Only a
// point inside such a ball has its bisector beyond v, so the union of the balls is exactly where the points that
// cut the cell lie -- a far tighter region than the ball of radius 2R for cells that reach the box.  Warp: the lanes
// share the vertices and vote (every lane must call it with the same arguments).
template <bool Warp>
__device__ __forceinline__ bool del_node_near_vertex(const DelaunayParams &P, uint32_t node, const double *pi,
                                                     const double (*vtx)[3], int nv) {
    const float *b = P.tree + 6 * (uint64_t)node;
    double lo[3], hi[3];
    for (int c = 0; c < 3; ++c) {
        lo[c] = (double)__ldg(b + c) - pi[c];
        hi[c] = (double)__ldg(b + 3 + c) - pi[c];
    }
    bool near = false;
    for (int k = Warp ? (int)(threadIdx.x & 31u) : 0; k < nv && !near; k += Warp ? 32 : 1) {
        double d2 = 0.0, v2 = 0.0;
        for (int c = 0; c < 3; ++c) {
            const double x = vtx[k][c], d = x < lo[c] ? lo[c] - x : (x > hi[c] ? x - hi[c] : 0.0);
            d2 += d * d;
            v2 += x * x;
        }
        near = d2 <= v2 * (1.0 + kDelSlack);
    }
    return Warp ? __any_sync(0xffffffffu, near) != 0 : near;
}

// Resumable depth-first query over the tree: next() returns the next point j != self with |p_j - p_i|^2 <= r2 whose
// leaf box meets a vertex ball of the cell (del_node_near_vertex), nearer subtrees first, or kDelNone.  r2 and the
// vertices may change between calls (the cell only shrinks).
struct DelBallIter {
    uint32_t stack[64];
    int sp;
    uint32_t pos, end;
    __device__ void init() {
        stack[0] = 1;
        sp = 1;
        pos = end = 0;
    }
    template <bool Warp>
    __device__ uint32_t next(const DelaunayParams &P, const double *pi, uint32_t self, double r2,
                             const double (*vtx)[3], int nv, double *d2) {
        for (;;) {
            while (pos < end) {
                const uint32_t j = pos++;
                if (j == self)
                    continue;
                double q[3];
                del_point(P, j, pi, q);
                const double dd = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
                if (dd <= r2) {
                    *d2 = dd;
                    return j;
                }
            }
            if (sp == 0)
                return kDelNone;
            const uint32_t node = stack[--sp];
            if (del_box_dist2(P, node, pi) > r2 || !del_node_near_vertex<Warp>(P, node, pi, vtx, nv))
                continue;
            if (node >= P.pow2) {
                pos = (node - P.pow2) * kDelLeaf;
                end = min(P.n, pos + kDelLeaf);
            } else { // the nearer child first, so that the cell shrinks early and r2 with it
                const double dl = del_box_dist2(P, 2 * node, pi), dr = del_box_dist2(P, 2 * node + 1, pi);
                stack[sp++] = dl <= dr ? 2 * node + 1 : 2 * node;
                stack[sp++] = dl <= dr ? 2 * node : 2 * node + 1;
            }
        }
    }
};

__device__ __forceinline__ bool del_before(double da, uint32_t a, double db, uint32_t b) {
    return da < db || (da == db && a < b);
}

// The k nearest points to p_i (not i itself) after (after_d2, after_id), ascending in (distance, index); returns how
// many were found.  A point at distance 0 is a duplicate of p_i.
template <int K>
__device__ int del_knn(const DelaunayParams &P, const double *pi, uint32_t self, double after_d2, uint32_t after_id,
                       uint32_t *ids, double *d2, bool *dup) {
    int cnt = 0;
    uint32_t stack[64];
    int sp = 1;
    stack[0] = 1;
    while (sp) {
        const uint32_t node = stack[--sp];
        const double worst = cnt == K ? d2[K - 1] : INFINITY;
        if (del_box_dist2(P, node, pi) > worst)
            continue;
        if (node >= P.pow2) {
            const uint32_t b = (node - P.pow2) * kDelLeaf, e = min(P.n, b + kDelLeaf);
            for (uint32_t j = b; j < e; ++j) {
                if (j == self)
                    continue;
                double q[3];
                del_point(P, j, pi, q);
                const double dd = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
                if (dd == 0.0)
                    *dup = true;
                if (!del_before(after_d2, after_id, dd, j))
                    continue;
                if (cnt == K && !del_before(dd, j, d2[K - 1], ids[K - 1]))
                    continue;
                int at = cnt < K ? cnt++ : K - 1;
                while (at > 0 && del_before(dd, j, d2[at - 1], ids[at - 1])) {
                    d2[at] = d2[at - 1];
                    ids[at] = ids[at - 1];
                    --at;
                }
                d2[at] = dd;
                ids[at] = j;
            }
        } else {
            const double dl = del_box_dist2(P, 2 * node, pi), dr = del_box_dist2(P, 2 * node + 1, pi);
            stack[sp++] = dl <= dr ? 2 * node + 1 : 2 * node; // the nearer child is visited first
            stack[sp++] = dl <= dr ? 2 * node : 2 * node + 1;
        }
    }
    return cnt;
}

// ---------------------------------------------------------------------------------------------- fast kernel
struct DelFastCell {
    uint32_t faces[kDelFaces];
    int nf;
    double vtx[kDelVerts][3];
    int nv;
    double r2; // squared radius: an upper bound on the cell's largest vertex distance
};

// Rebuild every polygon of the cell: drops planes whose polygon vanished, refreshes the vertices and the radius.
// final: keep only the faces whose area exceeds the threshold.  Returns false when a capacity is exceeded.
__device__ bool del_rebuild_fast(const DelaunayParams &P, const double *pi, DelFastCell &cell, bool final) {
    double a[kDelPolyVerts][3], b[kDelPolyVerts][3];
    const double w = 2.0 * sqrt(cell.r2) * (1.0 + kDelSlack);
    const double rlim = cell.r2 * (1.0 + kDelSlack);
    uint64_t keep = 0;
    int nv = 0;
    double r2 = 0.0;
    for (int k = -6; k < cell.nf; ++k) {
        const uint32_t id = k < 0 ? kDelBoxPlane + (uint32_t)(k + 6) : cell.faces[k];
        double nrm[3], m[3];
        del_plane(P, pi, id, nrm, m);
        const double h = nrm[0] * m[0] + nrm[1] * m[1] + nrm[2] * m[2], nn2 = nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2];
        if (h > 0.0 && h * h > rlim * nn2) // the plane is farther from p_i than the cell reaches
            continue;
        double(*poly)[3];
        const int n = del_face_polygon<kDelPolyVerts>(P, pi, id, cell.faces, cell.nf, w, a, b, &poly);
        if (n < 0 || nv + n > kDelVerts)
            return false;
        if (n < 3)
            continue;
        if (k >= 0 && (!final || del_area(poly, n) > kDelFaceArea * nn2))
            keep |= 1ull << k;
        for (int v = 0; v < n; ++v) {
            for (int c = 0; c < 3; ++c)
                cell.vtx[nv][c] = poly[v][c];
            r2 = fmax(r2, poly[v][0] * poly[v][0] + poly[v][1] * poly[v][1] + poly[v][2] * poly[v][2]);
            ++nv;
        }
    }
    int nf = 0;
    for (int k = 0; k < cell.nf; ++k)
        if (keep >> k & 1)
            cell.faces[nf++] = cell.faces[k];
    cell.nf = nf;
    cell.nv = nv;
    cell.r2 = r2;
    return true;
}

// One candidate in the fast kernel: 1 = stop (the stop rule holds; candidates come nearest first), 0 = go on,
// -1 = over capacity.  Unsorted candidates beyond 2R are skipped instead.
__device__ __forceinline__ int del_visit_fast(const DelaunayParams &P, const double *pi, DelFastCell &cell,
                                              int &pending, uint32_t j, double q2, bool sorted) {
    if (q2 > 4.0 * cell.r2 * (1.0 + kDelSlack))
        return sorted ? 1 : 0;
    double q[3];
    del_point(P, j, pi, q);
    if (!del_cuts(cell.vtx, cell.nv, q, q2, sqrt(cell.r2)))
        return 0;
    if (cell.nf == kDelFaces) {
        if (!del_rebuild_fast(P, pi, cell, false) || cell.nf == kDelFaces)
            return -1;
        pending = 0;
    }
    cell.faces[cell.nf++] = j;
    if (++pending == kDelRebuild) {
        if (!del_rebuild_fast(P, pi, cell, false))
            return -1;
        pending = 0;
    }
    return 0;
}

// Thread per cell (sorted index i): its faces go to pool[start[i], start[i] + count[i]) as sorted indices, or the
// cell goes to the overflow list.
__global__ void __launch_bounds__(kDelBlock) delaunay_clip_kernel(const DelaunayParams P, uint32_t *__restrict__ pool,
                                                                  uint32_t pool_capacity, uint32_t *__restrict__ start,
                                                                  uint32_t *__restrict__ count,
                                                                  uint32_t *__restrict__ overflow,
                                                                  unsigned long long *__restrict__ totals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n)
        return;
    start[i] = 0;
    count[i] = 0;
    double pi[3];
    bool finite = true;
    for (int c = 0; c < 3; ++c) {
        pi[c] = (double)__ldg(P.points + 3 * (uint64_t)i + c);
        finite = finite && isfinite(pi[c]);
    }
    if (!finite)
        return; // counted by the gather; the call fails
    DelFastCell cell;
    cell.nf = 0;
    cell.nv = 8;
    cell.r2 = del_box_corners(P, pi, cell.vtx);
    // candidates nearest first, kDelKnn per round, until the stop rule holds or every point has been visited
    uint32_t ids[kDelKnn];
    double d2[kDelKnn];
    bool dup = false;
    int pending = 0, rc = 0, round = 0;
    double after_d2 = -1.0;
    uint32_t after_id = 0;
    for (; round < kDelRounds; ++round) {
        const int k = del_knn<kDelKnn>(P, pi, i, after_d2, after_id, ids, d2, &dup);
        for (int c = 0; c < k && rc == 0; ++c)
            rc = del_visit_fast(P, pi, cell, pending, ids[c], d2[c], true);
        if (rc != 0 || k < kDelKnn)
            break;
        after_d2 = d2[kDelKnn - 1];
        after_id = ids[kDelKnn - 1];
    }
    if (dup)
        atomicAdd(totals + kDelDuplicate, 1ull);
    if (round == kDelRounds && rc == 0) {
        // still open after kDelRounds * kDelKnn candidates (cells that reach the box, flat cells): walk the tree for
        // the points inside the vertex balls of the cell, skipping those the rounds visited
        if (pending && !del_rebuild_fast(P, pi, cell, false))
            rc = -1;
        pending = 0;
        DelBallIter it;
        it.init();
        double dd;
        for (uint32_t j; rc == 0 && (j = it.next<false>(P, pi, i, 4.0 * cell.r2 * (1.0 + kDelSlack), cell.vtx,
                                                        cell.nv, &dd)) != kDelNone;)
            if (del_before(after_d2, after_id, dd, j))
                rc = del_visit_fast(P, pi, cell, pending, j, dd, false);
    }
    if (rc >= 0 && !del_rebuild_fast(P, pi, cell, true))
        rc = -1;
    if (rc < 0) {
        overflow[atomicAdd(totals + kDelOverflow, 1ull)] = i;
        return;
    }
    const unsigned long long base = atomicAdd(totals + kDelPoolNeed, (unsigned long long)cell.nf);
    count[i] = (uint32_t)cell.nf;
    if (base + cell.nf > pool_capacity) {
        start[i] = kDelNone; // the pool is too small: the caller grows it and builds again
        return;
    }
    start[i] = (uint32_t)base;
    for (int f = 0; f < cell.nf; ++f)
        pool[base + f] = cell.faces[f];
}

// ---------------------------------------------------------------------------------------------- overflow kernel
// Per-warp scratch slice: two face lists and two vertex lists (current, next), and a vertex cursor.
constexpr uint64_t kDelOvfSliceBytes = 2ull * kDelOvfFaces * 4 + 2ull * kDelOvfVerts * 24 + 16;

__device__ __forceinline__ double del_warp_max(double v) {
    for (int o = 16; o > 0; o >>= 1)
        v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Warp-wide rebuild of the cell in the slice: the lanes take the planes in turn.  Face order is kept (it fixes the
// clipping order, so the result does not depend on the schedule); vertex order does not matter.
__device__ bool del_rebuild_warp(const DelaunayParams &P, const double *pi, uint32_t *&faces, uint32_t *&faces_next,
                                 int &nf, double (*&vtx)[3], double (*&vtx_next)[3], int &nv, double &r2,
                                 unsigned int *vcursor, bool final) {
    const uint32_t lane = threadIdx.x & 31u;
    double a[kDelOvfPolyVerts][3], b[kDelOvfPolyVerts][3];
    const double w = 2.0 * sqrt(r2) * (1.0 + kDelSlack), rlim = r2 * (1.0 + kDelSlack);
    if (lane == 0)
        *vcursor = 0;
    __syncwarp();
    bool ok = true;
    double my_r2 = 0.0;
    int kept = 0;
    for (int base = -6; base < nf; base += 32) {
        const int k = base + (int)lane;
        bool keep = false;
        if (k < nf) {
            const uint32_t id = k < 0 ? kDelBoxPlane + (uint32_t)(k + 6) : faces[k];
            double nrm[3], m[3];
            del_plane(P, pi, id, nrm, m);
            const double h = nrm[0] * m[0] + nrm[1] * m[1] + nrm[2] * m[2];
            const double nn2 = nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2];
            if (!(h > 0.0 && h * h > rlim * nn2)) {
                double(*poly)[3];
                const int n = del_face_polygon<kDelOvfPolyVerts>(P, pi, id, faces, nf, w, a, b, &poly);
                if (n < 0) {
                    ok = false;
                } else if (n >= 3) {
                    keep = k >= 0 && (!final || del_area(poly, n) > kDelFaceArea * nn2);
                    const unsigned int at = atomicAdd(vcursor, (unsigned int)n);
                    if (at + n > (unsigned int)kDelOvfVerts) {
                        ok = false;
                    } else {
                        for (int v = 0; v < n; ++v) {
                            for (int c = 0; c < 3; ++c)
                                vtx_next[at + v][c] = poly[v][c];
                            my_r2 = fmax(my_r2, poly[v][0] * poly[v][0] + poly[v][1] * poly[v][1] +
                                                    poly[v][2] * poly[v][2]);
                        }
                    }
                }
            }
        }
        const unsigned int bal = __ballot_sync(0xffffffffu, keep);
        if (keep)
            faces_next[kept + __popc(bal & ((1u << lane) - 1u))] = faces[k];
        kept += __popc(bal);
    }
    __syncwarp();
    ok = __ballot_sync(0xffffffffu, !ok) == 0u;
    nv = (int)min(*vcursor, (unsigned int)kDelOvfVerts);
    __syncwarp();
    r2 = del_warp_max(my_r2);
    nf = kept;
    uint32_t *tf = faces;
    faces = faces_next;
    faces_next = tf;
    double(*tv)[3] = vtx;
    vtx = vtx_next;
    vtx_next = tv;
    return ok;
}

// Warp per overflowed cell (grid-stride over the overflow list; cells over the clip kernel's capacities).  The cell
// starts as the box cut by the kDelKnn nearest points, then the warp walks the tree for the points inside its vertex
// balls (nearer subtrees first).  Every lane follows the same walk; the work per node and per point -- the tests
// against every vertex of the cell -- is split across the lanes, and the polygon rebuilds take the planes in turn.
__global__ void __launch_bounds__(kDelBlock) delaunay_overflow_kernel(const DelaunayParams P,
                                                                      const uint32_t *__restrict__ overflow,
                                                                      char *__restrict__ slices,
                                                                      uint32_t *__restrict__ pool,
                                                                      uint32_t pool_capacity,
                                                                      uint32_t *__restrict__ start,
                                                                      uint32_t *__restrict__ count,
                                                                      unsigned long long *__restrict__ totals) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    char *slice = slices + (uint64_t)warp * kDelOvfSliceBytes;
    uint32_t *faces_a = reinterpret_cast<uint32_t *>(slice), *faces_b = faces_a + kDelOvfFaces;
    double(*vtx_a)[3] = reinterpret_cast<double(*)[3]>(faces_b + kDelOvfFaces);
    double(*vtx_b)[3] = vtx_a + kDelOvfVerts;
    unsigned int *vcursor = reinterpret_cast<unsigned int *>(vtx_b + kDelOvfVerts);
    const uint64_t cells = totals[kDelOverflow];
    for (uint64_t w = warp; w < cells; w += warps) {
        const uint32_t i = overflow[w];
        double pi[3];
        for (int c = 0; c < 3; ++c)
            pi[c] = (double)__ldg(P.points + 3 * (uint64_t)i + c);
        uint32_t *faces = faces_a, *faces_next = faces_b;
        double(*vtx)[3] = vtx_a, (*vtx_next)[3] = vtx_b;
        double r2 = 0.0;
        for (int k = 0; k < 8; ++k) {
            const double x = (double)((k & 1) ? P.hi[0] : P.lo[0]) - pi[0];
            const double y = (double)((k & 2) ? P.hi[1] : P.lo[1]) - pi[1];
            const double z = (double)((k & 4) ? P.hi[2] : P.lo[2]) - pi[2];
            r2 = fmax(r2, x * x + y * y + z * z);
        }
        // seed: the nearest points as face planes (the rebuild drops those that bound nothing)
        uint32_t ids[kDelKnn];
        double d2[kDelKnn];
        bool dup = false;
        const int k0 = del_knn<kDelKnn>(P, pi, i, -1.0, 0u, ids, d2, &dup);
        for (int f = (int)lane; f < k0; f += 32)
            faces[f] = ids[f];
        int nf = k0, nv = 0;
        __syncwarp();
        bool ok = del_rebuild_warp(P, pi, faces, faces_next, nf, vtx, vtx_next, nv, r2, vcursor, false);
        DelBallIter it;
        it.init();
        int pending = 0;
        double dd;
        for (uint32_t j; ok && (j = it.next<true>(P, pi, i, 4.0 * r2 * (1.0 + kDelSlack), vtx, nv, &dd)) != kDelNone;) {
            if (k0 > 0 && !del_before(d2[k0 - 1], ids[k0 - 1], dd, j))
                continue; // a seed: already a face plane, or dropped as bounding nothing
            double q[3];
            del_point(P, j, pi, q);
            if (!del_cuts_warp(vtx, nv, q, dd, sqrt(r2)))
                continue;
            if (nf == kDelOvfFaces) {
                ok = false;
                break;
            }
            if (lane == 0)
                faces[nf] = j;
            ++nf;
            if (++pending == kDelOvfBatch) {
                __syncwarp();
                ok = del_rebuild_warp(P, pi, faces, faces_next, nf, vtx, vtx_next, nv, r2, vcursor, false);
                pending = 0;
            }
        }
        __syncwarp();
        if (ok)
            ok = del_rebuild_warp(P, pi, faces, faces_next, nf, vtx, vtx_next, nv, r2, vcursor, true);
        if (!ok) {
            if (lane == 0) {
                atomicAdd(totals + kDelOverCapacity, 1ull);
                count[i] = 0;
                start[i] = 0;
            }
            __syncwarp();
            continue;
        }
        unsigned long long base = 0;
        if (lane == 0)
            base = atomicAdd(totals + kDelPoolNeed, (unsigned long long)nf);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (lane == 0) {
            count[i] = (uint32_t)nf;
            start[i] = base + nf > pool_capacity ? kDelNone : (uint32_t)base;
        }
        if (base + nf <= pool_capacity)
            for (int f = (int)lane; f < nf; f += 32)
                pool[base + f] = faces[f];
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------- assembly
__device__ __forceinline__ bool del_lists(const uint32_t *pool, const uint32_t *start, const uint32_t *count,
                                          uint32_t j, uint32_t i) {
    const uint32_t s = start[j];
    if (s == kDelNone)
        return false;
    for (uint32_t k = 0; k < count[j]; ++k)
        if (pool[s + k] == i)
            return true;
    return false;
}

// extra[j] = the cells that found j while j did not find them: row j gets them in addition to its own faces.
__global__ void __launch_bounds__(kDelBlock) delaunay_extra_kernel(uint32_t n, const uint32_t *__restrict__ pool,
                                                                   const uint32_t *__restrict__ start,
                                                                   const uint32_t *__restrict__ count,
                                                                   uint32_t *__restrict__ extra) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || start[i] == kDelNone)
        return;
    for (uint32_t k = 0; k < count[i]; ++k) {
        const uint32_t j = pool[start[i] + k];
        if (!del_lists(pool, start, count, j, i))
            atomicAdd(extra + j, 1u);
    }
}

// Row sizes in the caller's order, as the scan takes them: c = the row's entries, v = those found from one end only.
__global__ void __launch_bounds__(kDelBlock) delaunay_count_kernel(uint32_t n, const uint32_t *__restrict__ order,
                                                                   const uint32_t *__restrict__ start,
                                                                   const uint32_t *__restrict__ count,
                                                                   const uint32_t *__restrict__ extra,
                                                                   unsigned long long *__restrict__ v,
                                                                   uint32_t *__restrict__ c) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || order[i] >= n) // a bad order fails the build (totals[kDelBadOrder]); it must not write out of range
        return;
    const uint32_t own = start[i] == kDelNone ? 0u : count[i];
    v[order[i]] = extra[i];
    c[order[i]] = own + extra[i];
}

// Unsorted rows: cell i's own faces, then (through a per-row cursor) the cells that found i from their end only.
__global__ void __launch_bounds__(kDelBlock) delaunay_fill_kernel(uint32_t n, const uint32_t *__restrict__ order,
                                                                  const uint32_t *__restrict__ pool,
                                                                  const uint32_t *__restrict__ start,
                                                                  const uint32_t *__restrict__ count,
                                                                  const uint32_t *__restrict__ offsets,
                                                                  uint32_t *__restrict__ cursor,
                                                                  uint32_t *__restrict__ rows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || start[i] == kDelNone || order[i] >= n)
        return;
    // every write stays below the edge count, even for an order that is not a permutation (the build then failed)
    const uint32_t r = order[i], base = offsets[r], total = offsets[n];
    for (uint32_t k = 0; k < count[i]; ++k) {
        const uint32_t j = pool[start[i] + k];
        if (base + k < total)
            rows[base + k] = order[j];
        if (!del_lists(pool, start, count, j, i) && order[j] < n) {
            const uint32_t own = start[j] == kDelNone ? 0u : count[j];
            const uint64_t at = (uint64_t)offsets[order[j]] + own + atomicAdd(cursor + j, 1u);
            if (at < total)
                rows[at] = r;
        }
    }
}

// Warp per row: each entry goes to its rank within the row (entries are distinct), so rows come out ascending.
__global__ void __launch_bounds__(kDelBlock) delaunay_sort_kernel(uint32_t n, const uint32_t *__restrict__ offsets,
                                                                  const uint32_t *__restrict__ rows,
                                                                  uint32_t *__restrict__ adjacency) {
    const uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n)
        return;
    const uint32_t lane = threadIdx.x & 31u, b = offsets[r], e = offsets[r + 1];
    for (uint32_t a = b + lane; a < e; a += 32) {
        const uint32_t x = rows[a];
        uint32_t rank = 0;
        for (uint32_t k = b; k < e; ++k)
            rank += rows[k] < x;
        adjacency[b + rank] = x;
    }
}

} // namespace rfb
