// `rs dedupe` (robosat/tools/dedupe.py, robosat/spatial/core.py): which OSM features a predicted feature is not disjoint from,
// and the areas A(P), A(P ∩ U), A(U) of the prediction P and the union U of those features (DESIGN.md §8).
//
// Shapes come packed by robosat_b200/dedupe.py: rings are closed implicitly (next[v] is the vertex the edge from v ends at, and
// no ring repeats a vertex consecutively), exterior rings run counter-clockwise and holes clockwise in projected (x, y), so the
// interior of every feature lies on the left of each of its edges.
//
// Every orientation sign is exact: a floating-point filter (Shewchuk's orient2d bound) and, when it cannot decide, the sign of
// the error-free expansion of the determinant (six TwoProducts via fma summed with TwoSum into a nonoverlapping expansion).
//
// rsb_dedupe_intersects: one warp per candidate pair, on lon/lat vertices. The pair meets iff some edge of one meets some edge
// of the other (closed segments) or the first exterior vertex of some component of one lies strictly inside the other (the
// boundary case is already an edge contact). The edges of the larger shape are spread over the lanes; each lane tests its edge
// against the smaller shape's edges when the edge's box meets that shape's box.
//
// rsb_dedupe_areas: one thread per (prediction, edge) item, on projected vertices relative to the prediction's origin. The
// items of a prediction are the edges of P, then the edges of each OSM feature Q_k of S(P) in ascending feature order. An edge
// is cut at its crossings with the edges of the shapes that can matter to it (a P edge: every Q_k whose box meets the edge's; a
// Q_k edge: P when the edge meets P's box, and the Q_l (l != k) whose boxes it meets when |S(P)| > 1); a feature with a y-band
// index is scanned only over the bands the edge spans. Each piece is classified
// at its midpoint against those shapes: on another shape's boundary (exact collinearity, then the piece's direction against
// that edge's), else by its crossing number, half-open in y. A piece of feature X with X's interior on its left adds
// [R left of it] - [R right of it] times its length fraction to the boundary integral of region R, unless a lower-ranked shape
// of R (P first, then the Q_k in order) has the same piece on its boundary, which then counts it. Because the shoelace term of
// a sub-segment [t0, t1] of an edge is (t1 - t0) times the edge's own term, an edge's contribution is its term times the
// counted length fraction, and an uncut, fully counted edge contributes its term exactly. With |S(P)| = 1, A(U) is Q's
// shoelace sum. The per-item terms go to a workspace and one thread per prediction sums them in item order, so the areas do not
// depend on the batch or the run, and a P equal to its only Q gives I == A(P) == A(U) bit for bit.

#include <stdint.h>

#include <algorithm>

#include "../../include/rsb200.h"
#include "rsb_geom.cuh"
#include "rsb_host.h"

using namespace rsb;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int ISECT_THREADS = 128;
constexpr int AREA_THREADS = 128;
constexpr int SUM_THREADS = 128;
// Shewchuk's ccwerrboundA = (3 + 16 eps) eps, eps = 2^-53
constexpr double CCW_ERRBOUND = (3.0 + 16.0 * 1.1102230246251565e-16) * 1.1102230246251565e-16;

struct Shapes {
    const double2* __restrict__ v;
    const int32_t* __restrict__ next;
    const int64_t* __restrict__ fv;
    const int64_t* __restrict__ eo;
    const int64_t* __restrict__ ext;
    const double* __restrict__ box;
    const int64_t* __restrict__ fb;  // the y-band index (RsbShapes)
    const double* __restrict__ br;
    const int64_t* __restrict__ bo;
    const int32_t* __restrict__ be;
};

Shapes device_shapes(const RsbShapes& s) {
    return Shapes{reinterpret_cast<const double2*>(s.vertices), s.next, s.feature_vertices, s.exterior_offsets, s.exteriors, s.boxes,
                  s.feature_bands, s.band_ranges, s.band_offsets, s.band_edges};
}

__device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = __dadd_rn(a, b);
    const double bv = __dsub_rn(s, a);
    const double av = __dsub_rn(s, bv);
    e = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}

// the exact sign of ax*by - ax*cy - cx*by - ay*bx + ay*cx + cy*bx
__device__ __noinline__ int orient_exact(double2 a, double2 b, double2 c) {
    const double f[6][2] = {{a.x, b.y}, {-a.x, c.y}, {-c.x, b.y}, {-a.y, b.x}, {a.y, c.x}, {c.y, b.x}};
    double t[12];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        t[2 * i] = __dmul_rn(f[i][0], f[i][1]);
        t[2 * i + 1] = __fma_rn(f[i][0], f[i][1], -t[2 * i]);
    }
    double e[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) {  // Shewchuk's GROW-EXPANSION: e[0 .. k) stays nonoverlapping, increasing in magnitude
        double q = t[k];
#pragma unroll
        for (int i = 0; i < k; ++i) {
            double s, h;
            two_sum(q, e[i], s, h);
            e[i] = h;
            q = s;
        }
        e[k] = q;
    }
#pragma unroll
    for (int k = 11; k >= 0; --k)
        if (e[k] != 0.0) return e[k] > 0.0 ? 1 : -1;
    return 0;
}

// +1 when a, b, c turn counter-clockwise, -1 clockwise, 0 collinear; exact
__device__ __forceinline__ int orient(double2 a, double2 b, double2 c) {
    const double l = __dmul_rn(__dsub_rn(a.x, c.x), __dsub_rn(b.y, c.y));
    const double r = __dmul_rn(__dsub_rn(a.y, c.y), __dsub_rn(b.x, c.x));
    const double det = __dsub_rn(l, r);
    const double bound = __dmul_rn(CCW_ERRBOUND, __dadd_rn(fabs(l), fabs(r)));
    if (det > bound) return 1;
    if (-det > bound) return -1;
    return orient_exact(a, b, c);
}

__device__ __forceinline__ bool boxes_meet(double ax0, double ay0, double ax1, double ay1, const double* __restrict__ b) {
    return !(ax1 < b[0] || b[2] < ax0 || ay1 < b[1] || b[3] < ay0);
}

// p, collinear with a and b, lies on the closed segment ab
__device__ __forceinline__ bool within(double2 a, double2 b, double2 p) {
    return fmin(a.x, b.x) <= p.x && p.x <= fmax(a.x, b.x) && fmin(a.y, b.y) <= p.y && p.y <= fmax(a.y, b.y);
}

// the closed segments ab and cd share a point
__device__ bool segments_meet(double2 a, double2 b, double2 c, double2 d) {
    if (fmax(a.x, b.x) < fmin(c.x, d.x) || fmax(c.x, d.x) < fmin(a.x, b.x) || fmax(a.y, b.y) < fmin(c.y, d.y) || fmax(c.y, d.y) < fmin(a.y, b.y))
        return false;
    const int o1 = orient(a, b, c), o2 = orient(a, b, d), o3 = orient(c, d, a), o4 = orient(c, d, b);
    if (o1 * o2 < 0 && o3 * o4 < 0) return true;
    return (o1 == 0 && within(a, b, c)) || (o2 == 0 && within(a, b, d)) || (o3 == 0 && within(c, d, a)) || (o4 == 0 && within(c, d, b));
}

// the upward ray-crossing of p with edge cg, half-open in y: p strictly left of an edge that spans p.y
__device__ __forceinline__ int crosses(double2 c, double2 g, double2 p) {
    if ((c.y > p.y) == (g.y > p.y)) return 0;
    const int o = orient(c, g, p);
    return g.y > c.y ? o > 0 : o < 0;
}

// some edge of feature a of A meets some edge of feature b of B (warp-uniform result)
__device__ bool edges_meet(const Shapes& A, int a, const Shapes& B, int b, int lane) {
    const bool swap = B.fv[b + 1] - B.fv[b] > A.fv[a + 1] - A.fv[a];  // lanes stride over the larger shape's edges
    const double2* sv = swap ? B.v : A.v;
    const int32_t* sn = swap ? B.next : A.next;
    const double2* tv = swap ? A.v : B.v;
    const int32_t* tn = swap ? A.next : B.next;
    const int s = swap ? b : a, t = swap ? a : b;
    const int64_t s0 = (swap ? B.fv : A.fv)[s], s1 = (swap ? B.fv : A.fv)[s + 1];
    const int64_t t0 = (swap ? A.fv : B.fv)[t], t1 = (swap ? A.fv : B.fv)[t + 1];
    const double* tb = (swap ? A.box : B.box) + 4 * static_cast<int64_t>(t);
    for (int64_t base = s0; base < s1; base += 32) {
        bool hit = false;
        const int64_t v = base + lane;
        if (v < s1) {
            const double2 c = sv[v], g = sv[sn[v]];
            if (boxes_meet(fmin(c.x, g.x), fmin(c.y, g.y), fmax(c.x, g.x), fmax(c.y, g.y), tb))
                for (int64_t u = t0; u < t1 && !hit; ++u) hit = segments_meet(c, g, tv[u], tv[tn[u]]);
        }
        if (__any_sync(FULL, hit)) return true;
    }
    return false;
}

// the first exterior vertex of some component of feature a of A lies strictly inside feature b of B (warp-uniform result)
__device__ bool exterior_inside(const Shapes& A, int a, const Shapes& B, int b, int lane) {
    const double* bb = B.box + 4 * static_cast<int64_t>(b);
    const int64_t b0 = B.fv[b], b1 = B.fv[b + 1];
    for (int64_t k = A.eo[a]; k < A.eo[a + 1]; ++k) {
        const double2 p = A.v[A.ext[k]];
        if (!boxes_meet(p.x, p.y, p.x, p.y, bb)) continue;
        int parity = 0;
        for (int64_t base = b0; base < b1; base += 32) {
            const int64_t u = base + lane;
            if (u < b1) parity ^= crosses(B.v[u], B.v[B.next[u]], p);
        }
        if (__popc(__ballot_sync(FULL, parity)) & 1) return true;
    }
    return false;
}

__global__ void __launch_bounds__(ISECT_THREADS) dedupe_intersects_kernel(Shapes P, Shapes Q, const int32_t* __restrict__ pairs, int64_t n, uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = static_cast<int64_t>(gridDim.x) * (ISECT_THREADS / 32);
    for (int64_t w = (static_cast<int64_t>(blockIdx.x) * ISECT_THREADS + threadIdx.x) >> 5; w < n; w += warps) {
        const int p = pairs[2 * w], q = pairs[2 * w + 1];
        const bool hit = edges_meet(P, p, Q, q, lane) || exterior_inside(P, p, Q, q, lane) || exterior_inside(Q, q, P, p, lane);
        if (lane == 0) out[w] = hit ? 1 : 0;
    }
}

// ---- areas ----

struct Edge {
    double2 a, b, d;
    double x0, y0, x1, y1;  // box
};

__device__ __forceinline__ Edge make_edge(double2 a, double2 b) {
    return Edge{a, b, make_double2(__dsub_rn(b.x, a.x), __dsub_rn(b.y, a.y)), fmin(a.x, b.x), fmin(a.y, b.y), fmax(a.x, b.x), fmax(a.y, b.y)};
}

// parameter of p's projection on the line of e
__device__ __forceinline__ double param(const Edge& e, double2 p) {
    const double num = __dadd_rn(__dmul_rn(__dsub_rn(p.x, e.a.x), e.d.x), __dmul_rn(__dsub_rn(p.y, e.a.y), e.d.y));
    const double den = __dadd_rn(__dmul_rn(e.d.x, e.d.x), __dmul_rn(e.d.y, e.d.y));
    return __ddiv_rn(num, den);
}

// the state of one scan of a shape's edges against a piece of e
struct Probe {
    double after, next;  // split parameters in (after, next) lower next
    double tm;           // the piece's midpoint parameter, and the point
    double2 m;
    bool classify, same, opp;
    int parity;
};

__device__ __forceinline__ void lower(Probe& pr, double t) {
    if (t > pr.after && t < pr.next) pr.next = t;
}

// edge cg of another shape against e: the splits it makes and, when classifying, coincidence with the piece and m's crossing
__device__ __forceinline__ void probe_edge(const Edge& e, double2 c, double2 g, Probe& pr) {
    if (pr.classify) pr.parity ^= crosses(c, g, pr.m);
    if (fmax(c.x, g.x) < e.x0 || e.x1 < fmin(c.x, g.x) || fmax(c.y, g.y) < e.y0 || e.y1 < fmin(c.y, g.y)) return;
    const int o1 = orient(e.a, e.b, c), o2 = orient(e.a, e.b, g);
    if (o1 == 0 && o2 == 0) {  // collinear: cut at cg's ends; the piece lies on cg when its midpoint is inside cg's span
        const double tc = param(e, c), tg = param(e, g);
        lower(pr, tc);
        lower(pr, tg);
        if (pr.classify && fmin(tc, tg) < pr.tm && pr.tm < fmax(tc, tg)) {
            const double dot = __dadd_rn(__dmul_rn(e.d.x, __dsub_rn(g.x, c.x)), __dmul_rn(e.d.y, __dsub_rn(g.y, c.y)));
            if (dot > 0.0) pr.same = true;
            else pr.opp = true;
        }
        return;
    }
    if (o1 * o2 > 0) return;
    if (o1 == 0) {  // c on e's line (on e when its parameter is in (0, 1))
        lower(pr, param(e, c));
        return;
    }
    if (o2 == 0) {
        lower(pr, param(e, g));
        return;
    }
    const int o3 = orient(c, g, e.a), o4 = orient(c, g, e.b);
    if (o3 * o4 >= 0) return;  // no crossing, or it is at an end of e
    // the crossing's parameter along e: ((c - a) x f) / (d x f), f = g - c
    const double fx = __dsub_rn(g.x, c.x), fy = __dsub_rn(g.y, c.y);
    const double num = __dsub_rn(__dmul_rn(__dsub_rn(c.x, e.a.x), fy), __dmul_rn(__dsub_rn(c.y, e.a.y), fx));
    const double den = __dsub_rn(__dmul_rn(e.d.x, fy), __dmul_rn(e.d.y, fx));
    lower(pr, __ddiv_rn(num, den));
}

// which sides of the piece lie in one shape's feature
struct Side {
    bool left, right, on;
};

// the band of y in a feature's index (the host computes the same float64 expression)
__device__ __forceinline__ int64_t band_of(double y, double y0, double inv, int64_t nb) {
    return static_cast<int64_t>(fmin(fmax(floor(__dmul_rn(__dsub_rn(y, y0), inv)), 0.0), static_cast<double>(nb - 1)));
}

// Every edge of feature f of S that can cut e or cross m's horizontal ray has a y range meeting [ylo, yhi] = e's y range and
// m.y, so an indexed feature scans only the bands over that range; an edge listed in several of them is probed in the first.
__device__ __forceinline__ Side scan(const Edge& e, const Shapes& S, int f, Probe& pr) {
    pr.same = pr.opp = false;
    pr.parity = 0;
    const int64_t fb = S.fb[f], nb = S.fb[f + 1] - fb;
    if (nb == 0) {
        const int64_t v1 = S.fv[f + 1];
        for (int64_t v = S.fv[f]; v < v1; ++v) probe_edge(e, S.v[v], S.v[S.next[v]], pr);
    } else {
        const double y0 = S.br[2 * f], inv = S.br[2 * f + 1];
        const double ylo = pr.classify ? fmin(e.y0, pr.m.y) : e.y0, yhi = pr.classify ? fmax(e.y1, pr.m.y) : e.y1;
        const int64_t q0 = band_of(ylo, y0, inv, nb), q1 = band_of(yhi, y0, inv, nb);
        for (int64_t b = q0; b <= q1; ++b) {
            const int64_t j1 = S.bo[fb + b + 1];
            for (int64_t j = S.bo[fb + b]; j < j1; ++j) {
                const int v = S.be[j];
                const double2 c = S.v[v], g = S.v[S.next[v]];
                if (max(band_of(fmin(c.y, g.y), y0, inv, nb), q0) != b) continue;
                probe_edge(e, c, g, pr);
            }
        }
    }
    if (pr.same || pr.opp) return Side{pr.same, pr.opp, true};
    return Side{pr.parity != 0, pr.parity != 0, false};
}

__device__ __forceinline__ bool edge_meets_box(const Edge& e, const double* __restrict__ box, int f) {
    return boxes_meet(e.x0, e.y0, e.x1, e.y1, box + 4 * static_cast<int64_t>(f));
}

struct Context {
    Shapes P, Q;
    int p;                               // the prediction's feature
    const int32_t* __restrict__ ids;     // S(P), ascending
    int m;                               // |S(P)|
};

// The counted length fractions (of I, of U) of edge e, which belongs to P (k < 0) or to Q_k.
__device__ void fractions(const Edge& e, const Context& cx, int k, bool near_p, double& frac_i, double& frac_u) {
    frac_i = frac_u = 0.0;
    Probe pr;
    pr.after = 0.0;
    pr.next = 1.0;
    pr.classify = false;
    pr.tm = 0.0;
    pr.m = e.a;
    // pass 0 finds the first cut; pass j > 0 classifies piece j - 1 and finds the cut after it
    double t0 = 0.0, t1 = 0.0;
    for (int pass = 0;; ++pass) {
        bool u_left = false, u_right = false, lower_u = false;
        Side sp{false, false, false};
        if (k < 0) {
            for (int j = 0; j < cx.m; ++j) {
                const int q = cx.ids[j];
                if (!edge_meets_box(e, cx.Q.box, q)) continue;
                const Side s = scan(e, cx.Q, q, pr);
                u_left |= s.left;
            }
        } else {
            if (near_p) sp = scan(e, cx.P, cx.p, pr);
            if (cx.m > 1)
                for (int j = 0; j < cx.m; ++j) {
                    const int q = cx.ids[j];
                    if (j == k || !edge_meets_box(e, cx.Q.box, q)) continue;
                    const Side s = scan(e, cx.Q, q, pr);
                    u_right |= s.right;
                    lower_u |= s.on && j < k;
                }
        }
        if (pass > 0) {
            const double len = __dsub_rn(t1, t0);
            if (k < 0) {
                if (u_left) frac_i = __dadd_rn(frac_i, len);
            } else {
                if (!lower_u && !u_right) frac_u = __dadd_rn(frac_u, len);
                if (!sp.on && !lower_u && sp.left && !u_right) frac_i = __dadd_rn(frac_i, len);
            }
            if (t1 >= 1.0) return;
            t0 = t1;
        }
        t1 = pr.next;
        pr.after = t1;
        pr.next = 1.0;
        pr.classify = true;
        pr.tm = __dmul_rn(0.5, __dadd_rn(t0, t1));
        pr.m = make_double2(__dadd_rn(e.a.x, __dmul_rn(pr.tm, e.d.x)), __dadd_rn(e.a.y, __dmul_rn(pr.tm, e.d.y)));
    }
}

__global__ void __launch_bounds__(AREA_THREADS) dedupe_terms_kernel(Shapes P, Shapes Q, const int32_t* __restrict__ pred, const double* __restrict__ origins,
                                                                    const int64_t* __restrict__ set_offsets, const int32_t* __restrict__ set_ids,
                                                                    int64_t num_segments, const int64_t* __restrict__ item_offsets,
                                                                    const int32_t* __restrict__ segment_pred, int64_t num_items, double* __restrict__ term_i,
                                                                    double* __restrict__ term_a) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * AREA_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * AREA_THREADS + threadIdx.x; i < num_items; i += stride) {
        const int64_t seg = upper_bound(item_offsets, 0, num_segments + 1, i) - 1;
        const int b = segment_pred[seg];
        const int64_t s0 = set_offsets[b];
        const int k = static_cast<int>(seg - (b + s0)) - 1;
        Context cx{P, Q, pred[b], set_ids + s0, static_cast<int>(set_offsets[b + 1] - s0)};
        const double2* xv = k < 0 ? P.v : Q.v;
        const int32_t* xn = k < 0 ? P.next : Q.next;
        const int f = k < 0 ? cx.p : cx.ids[k];
        const int64_t v = (k < 0 ? P.fv : Q.fv)[f] + (i - item_offsets[seg]);
        const Edge e = make_edge(xv[v], xv[xn[v]]);
        const double ox = origins[2 * b], oy = origins[2 * b + 1];
        const double ax = __dsub_rn(e.a.x, ox), ay = __dsub_rn(e.a.y, oy), bx = __dsub_rn(e.b.x, ox), by = __dsub_rn(e.b.y, oy);
        const double term = __dmul_rn(0.5, __dsub_rn(__dmul_rn(ax, by), __dmul_rn(bx, ay)));
        const bool near_p = k >= 0 && edge_meets_box(e, P.box, cx.p);
        double fi = 0.0, fu = 1.0;
        if (k < 0 || near_p || cx.m > 1) fractions(e, cx, k, near_p, fi, fu);
        term_i[i] = __dmul_rn(fi, term);
        term_a[i] = (k < 0 || cx.m == 1) ? term : __dmul_rn(fu, term);
    }
}

// one thread per prediction: the item terms summed in item order
__global__ void __launch_bounds__(SUM_THREADS) dedupe_sum_kernel(int32_t B, const int64_t* __restrict__ set_offsets, const int64_t* __restrict__ item_offsets,
                                                                 const double* __restrict__ term_i, const double* __restrict__ term_a, double* __restrict__ areas) {
    const int b = blockIdx.x * SUM_THREADS + threadIdx.x;
    if (b >= B) return;
    const int64_t s0 = b + set_offsets[b], m = set_offsets[b + 1] - set_offsets[b];
    double ap = 0.0, in = 0.0, un = 0.0;
    for (int64_t i = item_offsets[s0]; i < item_offsets[s0 + 1]; ++i) {
        ap = __dadd_rn(ap, term_a[i]);
        in = __dadd_rn(in, term_i[i]);
    }
    for (int64_t s = s0 + 1; s <= s0 + m; ++s) {
        double u = 0.0;
        for (int64_t i = item_offsets[s]; i < item_offsets[s + 1]; ++i) {
            u = __dadd_rn(u, term_a[i]);
            in = __dadd_rn(in, term_i[i]);
        }
        un = __dadd_rn(un, u);
    }
    areas[3 * static_cast<int64_t>(b)] = ap;
    areas[3 * static_cast<int64_t>(b) + 1] = in;
    areas[3 * static_cast<int64_t>(b) + 2] = un;
}

int check_shapes(const RsbShapes* s, const char* what, const char* name) {
    if (!s) return set_error(RSB_E_INVALID, "%s: null %s shapes", what, name);
    if (s->num_features < 1 || s->num_vertices < 1 || !s->vertices || !s->next || !s->feature_vertices || !s->exterior_offsets || !s->exteriors || !s->boxes ||
        !s->feature_bands || !s->band_ranges || !s->band_offsets || !s->band_edges)
        return set_error(RSB_E_INVALID, "%s: %s shapes need at least one feature, one vertex and every array (num_features=%d num_vertices=%lld)", what, name,
                         s->num_features, (long long)s->num_vertices);
    if (s->num_vertices > 0x7fffffffLL) return set_error(RSB_E_INVALID, "%s: %s shapes have %lld vertices (at most 2^31 - 1)", what, name, (long long)s->num_vertices);
    if ((reinterpret_cast<uintptr_t>(s->vertices) & 15) != 0) return set_error(RSB_E_INVALID, "%s: %s vertices must be 16-byte aligned", what, name);
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_dedupe_intersects(const RsbShapes* predicted, const RsbShapes* osm, const int32_t* pairs, int64_t num_pairs, uint8_t* out, void* stream) {
    int rc = check_shapes(predicted, "dedupe_intersects", "predicted");
    if (rc == RSB_OK) rc = check_shapes(osm, "dedupe_intersects", "osm");
    if (rc != RSB_OK) return rc;
    if (num_pairs < 0 || (num_pairs > 0 && (!pairs || !out)))
        return set_error(RSB_E_INVALID, "dedupe_intersects: num_pairs=%lld with null pairs or out", (long long)num_pairs);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    if (num_pairs == 0) return RSB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t blocks = std::min<int64_t>((num_pairs + ISECT_THREADS / 32 - 1) / (ISECT_THREADS / 32), 64 * num_sms());
    dedupe_intersects_kernel<<<static_cast<unsigned>(blocks), ISECT_THREADS, 0, st>>>(device_shapes(*predicted), device_shapes(*osm), pairs, num_pairs, out);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "dedupe_intersects launch");
}

extern "C" int rsb_dedupe_areas(const RsbShapes* predicted, const RsbShapes* osm, int32_t B, const int32_t* pred, const double* origins, const int64_t* set_offsets,
                                const int32_t* set_ids, int64_t num_segments, const int64_t* item_offsets, const int32_t* segment_pred, int64_t num_items,
                                double* terms, double* areas, void* stream) {
    int rc = check_shapes(predicted, "dedupe_areas", "predicted");
    if (rc == RSB_OK) rc = check_shapes(osm, "dedupe_areas", "osm");
    if (rc != RSB_OK) return rc;
    if (B < 1 || !pred || !origins || !set_offsets || !item_offsets || !segment_pred || !areas)
        return set_error(RSB_E_INVALID, "dedupe_areas: B=%d (need B >= 1) or a null array", B);
    if (num_segments < B || num_items < 0 || (num_items > 0 && !terms) || (num_segments > B && !set_ids))
        return set_error(RSB_E_INVALID, "dedupe_areas: num_segments=%lld num_items=%lld for B=%d", (long long)num_segments, (long long)num_items, B);
    const int dev_rc = rsb_device_ok();
    if (dev_rc != RSB_OK) return dev_rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (num_items > 0) {
        const int64_t blocks = std::min<int64_t>((num_items + AREA_THREADS - 1) / AREA_THREADS, 64 * num_sms());
        dedupe_terms_kernel<<<static_cast<unsigned>(blocks), AREA_THREADS, 0, st>>>(device_shapes(*predicted), device_shapes(*osm), pred, origins, set_offsets, set_ids,
                                                                                    num_segments, item_offsets, segment_pred, num_items, terms, terms + num_items);
    }
    dedupe_sum_kernel<<<static_cast<unsigned>((B + SUM_THREADS - 1) / SUM_THREADS), SUM_THREADS, 0, st>>>(B, set_offsets, item_offsets, terms, terms + num_items, areas);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "dedupe_areas launch");
}
