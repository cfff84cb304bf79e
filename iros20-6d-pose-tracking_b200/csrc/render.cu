// CUDA rasteriser for input A (SURVEY.md 8f row 2): what the reference obtains from OpenGL through vispy
//   window + matrices   predict.py:193-215 (Tracker.render_window), vispy_renderer.py:135-150 (update_cam_mat)
//   light               vispy_renderer.py:171-173
//   shaders             vispy_renderer.py:56-105 (Lambert term 0.4 * max(n.l, 0) + 0.65 ambient, clamp)
//   read-back + depth   vispy_renderer.py:152-169 (glReadPixels RGB8 / DEPTH float, z-buffer -> metric distance -> uint16 mm)
// for all tracks of a frame in one launch, straight into the buffers the preprocess kernel reads -- no GL context, no
// glReadPixels, no host round trip.
//
// Pipeline, two launches chained by programmatic dependent launch:
//   A. render_project_kernel (grid = vertex blocks x n): thread 0 of every CTA builds the track's uniforms in float64 exactly
//      as numpy does (window via bbox.cuh, orthographic matrix rounded to float32, projection product, light = R_gl *
//      (0, .1, -.9) which is what inv(view^T) * (0,.1,-.9,1) evaluates to); every thread projects ONE vertex (float64 on the
//      float32 uniforms), snaps it to 1/256 pixel and stores {X, Y, z_window, 1/w} (24 B) -- each vertex is projected once per
//      track instead of ~6 times per band.
//   B. render_kernel (one CTA per (track, set of every 4th image row); grid = 4 x n -- interleaved rows, so the four CTAs
//      of a track share the object's pixels evenly wherever it sits in the window):
//   1. visibility: triangles are dealt to threads; each gathers its three projected vertices,
//      walks the pixel centres of its bounding box with exact integer edge functions
//      (top-left rule, no culling -- the reference never enables GL_CULL_FACE), interpolates window z and does a 64-bit
//      shared-memory atomicMin on (float32 z bits << 32 | triangle index): depth test LESS, first-drawn wins ties.
//      Triangles with large boxes are rasterised by the whole warp.
//   2. resolve: one thread per pixel re-derives its triangle's barycentrics, interpolates position / normal / colour
//      perspective-correctly, shades, converts the depth the way on_draw does and writes uint8 rgb + uint16 mm.
// Divisions are confined to reciprocals (1/w per vertex, 1/area per triangle, 1/sum(q) and 1/|l| per pixel), as GPUs do.
// All arithmetic is float64 with a fixed association and this file is compiled with -fmad=false, so it is bit-identical
// to the numpy restatement in oracle/se3_oracle.py (render_window).  Near-plane clipping: triangles wholly in front of the
// eye are cut per pixel by the depth test; a triangle with a vertex at or behind the eye plane (w <= 1e-6) takes the
// homogeneous path below (straddler_*), which yields the fragments GL's polygon clipping would.  Scope limit: float32 depth buffer.
#include "render.h"
#include "bbox.cuh"
#include "launch.h"
#include "ptx.cuh"
#include <climits>

namespace se3tn {
namespace {
constexpr int kRS = 176, kBands = 4, kBandRows = kRS / kBands, kSub = 256, kHalf = kSub / 2;
constexpr int kRenderThreads = 512;
constexpr unsigned long long kClearKey = (0x3F800000ull << 32) | 0xFFFFFFFFull;       // depth 1.0, no triangle
constexpr int kBigBox = 96;                                                            // bounding boxes above this many pixels go to the whole warp

struct Uniforms {
    double V[12];            // view (rows 0..2; row 3 = 0 0 0 1), float32 values
    double P00, P02, P11, P12, P22, P23;   // projection (float32 values); P32 = -1
    double A, B;             // projection_matrix[2][2], [3][2] in float64 (depth linearisation)
    double light[3];
    double hx, hy;           // half the viewport in pixels: window x = (ndc + 1) * hx
    int valid, mode;         // mode 0: the 176 x 176 crop window IS the viewport (vispy); 1: the whole camera image is (pyrender)
    int vw, vh;              // viewport in pixels
    int top, left, ch, cw;   // mode 1: crop window in image pixels (rows from the top), what crop_bbox cuts out of the full render
};
static_assert(sizeof(Uniforms) % sizeof(double) == 0, "Uniforms is copied as doubles");

__device__ __forceinline__ long long floor_div(long long a, long long b) {             // b > 0
    long long q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

struct Vtx { long long X, Y; double zw, w; bool ok; };
struct PVtx { int X, Y; double zw, iw; };         // stored form (iw = 1/w); X == INT_MIN marks a vertex that cannot be used (w <= 1e-6, non-finite)

// clip = P . V . p in float64 on the float32 uniforms, fixed association (oracle/se3_oracle.py _project_vertices)
__device__ __forceinline__ void clip_coords(const Uniforms& u, const float* __restrict__ pos, int vi, double c[4]) {
    const double px = pos[3 * vi], py = pos[3 * vi + 1], pz = pos[3 * vi + 2];
    const double v0 = ((u.V[0] * px + u.V[1] * py) + u.V[2] * pz) + u.V[3];
    const double v1 = ((u.V[4] * px + u.V[5] * py) + u.V[6] * pz) + u.V[7];
    const double v2 = ((u.V[8] * px + u.V[9] * py) + u.V[10] * pz) + u.V[11];
    const double v3 = ((0.0 * px + 0.0 * py) + 0.0 * pz) + 1.0;
    // the zero entries of P stay in the sums (x + 0*y is exact for finite y)
    c[0] = ((u.P00 * v0 + 0.0 * v1) + u.P02 * v2) + 0.0 * v3;
    c[1] = ((0.0 * v0 + u.P11 * v1) + u.P12 * v2) + 0.0 * v3;
    c[2] = ((0.0 * v0 + 0.0 * v1) + u.P22 * v2) + u.P23 * v3;
    c[3] = ((0.0 * v0 + 0.0 * v1) + -1.0 * v2) + 0.0 * v3;
}

__device__ __forceinline__ Vtx project(const Uniforms& u, const float* __restrict__ pos, int vi) {
    double c[4];
    clip_coords(u, pos, vi, c);
    const double c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3];
    Vtx r;
    r.w = c3;
    const double xw = (c0 / c3 + 1.0) * u.hx, yw = (c1 / c3 + 1.0) * u.hy;
    r.zw = (c2 / c3 + 1.0) * 0.5;
    const double X = rint(xw * kSub), Y = rint(yw * kSub);
    const double lim = 33554432.0;                   // 2^25 sub-pixels: every edge-function product stays below 2^53, exact in float64
    r.ok = (c3 > 1e-6) && (X == X) && (Y == Y) && fabs(X) < lim && fabs(Y) < lim;
    r.X = r.ok ? static_cast<long long>(X) : 0;
    r.Y = r.ok ? static_cast<long long>(Y) : 0;
    return r;
}

__device__ __forceinline__ Vtx load_projected(const PVtx* __restrict__ pv, int vi) {
    const PVtx q = pv[vi];
    Vtx r; r.ok = q.X != INT_MIN; r.X = q.X; r.Y = q.Y; r.zw = q.zw; r.w = q.iw;
    return r;
}

struct Tri {
    int i0, i1, i2;
    long long x0, y0, x1, y1, x2, y2, area2;
    double z0, z1, z2, w0, w1, w2;
    bool ok;
};

__device__ __forceinline__ Tri setup(const PVtx* __restrict__ pv, const MeshDev& m, int t) {     // T.w* hold 1/w
    Tri T;
    T.i0 = m.faces[3 * t]; T.i1 = m.faces[3 * t + 1]; T.i2 = m.faces[3 * t + 2];
    T.ok = static_cast<unsigned>(T.i0) < static_cast<unsigned>(m.nv) && static_cast<unsigned>(T.i1) < static_cast<unsigned>(m.nv) &&
           static_cast<unsigned>(T.i2) < static_cast<unsigned>(m.nv);
    if (!T.ok) return T;
    const Vtx a = load_projected(pv, T.i0), b = load_projected(pv, T.i1), c = load_projected(pv, T.i2);
    T.ok = a.ok && b.ok && c.ok;
    if (!T.ok) return T;
    T.x0 = a.X; T.y0 = a.Y; T.z0 = a.zw; T.w0 = a.w;
    T.x1 = b.X; T.y1 = b.Y; T.z1 = b.zw; T.w1 = b.w;
    T.x2 = c.X; T.y2 = c.Y; T.z2 = c.zw; T.w2 = c.w;
    T.area2 = (T.x1 - T.x0) * (T.y2 - T.y0) - (T.x2 - T.x0) * (T.y1 - T.y0);
    if (T.area2 == 0) { T.ok = false; return T; }
    if (T.area2 < 0) {                      // no culling: make it counter-clockwise (y up)
        int ti = T.i1; T.i1 = T.i2; T.i2 = ti;
        long long tl = T.x1; T.x1 = T.x2; T.x2 = tl; tl = T.y1; T.y1 = T.y2; T.y2 = tl;
        double td = T.z1; T.z1 = T.z2; T.z2 = td; td = T.w1; T.w1 = T.w2; T.w2 = td;
        T.area2 = -T.area2;
    }
    return T;
}

// Edge functions in float64: coordinates are integers below 2^25 in magnitude, so differences (< 2^26), products (< 2^52)
// and their difference are exact -- the same values the int64 evaluation gives, at one DMUL instead of a multi-word multiply.
struct EdgeSet { double dx0, dy0, dx1, dy1, dx2, dy2, x0, y0, x1, y1, x2, y2; };
__device__ __forceinline__ EdgeSet edge_set(const Tri& T) {
    EdgeSet E;
    E.x0 = static_cast<double>(T.x0); E.y0 = static_cast<double>(T.y0); E.x1 = static_cast<double>(T.x1); E.y1 = static_cast<double>(T.y1);
    E.x2 = static_cast<double>(T.x2); E.y2 = static_cast<double>(T.y2);
    E.dx0 = E.x2 - E.x1; E.dy0 = E.y2 - E.y1; E.dx1 = E.x0 - E.x2; E.dy1 = E.y0 - E.y2; E.dx2 = E.x1 - E.x0; E.dy2 = E.y1 - E.y0;
    return E;
}
__device__ __forceinline__ void edges(const EdgeSet& E, double cx, double cy, double& e0, double& e1, double& e2) {
    e0 = E.dx0 * (cy - E.y1) - E.dy0 * (cx - E.x1);
    e1 = E.dx1 * (cy - E.y2) - E.dy1 * (cx - E.x2);
    e2 = E.dx2 * (cy - E.y0) - E.dy2 * (cx - E.x0);
}
__device__ __forceinline__ bool top_left(long long dx, long long dy) { return dy < 0 || (dy == 0 && dx < 0); }

// one pixel centre against one triangle.  Rows are interleaved over the four CTAs of a track: this CTA owns rows j = 4*jj + band.
// The sample of output pixel (i, j) sits at sub-pixel position (xs[i], ys[j]) of the viewport: the pixel's own centre in mode 0, the
// centre of the camera-image pixel crop_bbox's nearest-neighbour resize picks in mode 1 (outside the viewport: no fragment).
struct Samples { const int* xs; const int* ys; int vw, vh; };
__device__ __forceinline__ void raster_pixel(const Tri& T, const EdgeSet& E, double inv_area, int t, int i, int j, bool tl0, bool tl1, bool tl2, const Samples& sm, unsigned long long* keys) {
    const int sx = sm.xs[i], sy = sm.ys[j];
    if (static_cast<unsigned>(sx >> 8) >= static_cast<unsigned>(sm.vw) || static_cast<unsigned>(sy >> 8) >= static_cast<unsigned>(sm.vh)) return;
    const double cx = static_cast<double>(sx), cy = static_cast<double>(sy);
    double e0, e1, e2;
    edges(E, cx, cy, e0, e1, e2);
    if (!((e0 > 0 || (e0 == 0 && tl0)) && (e1 > 0 || (e1 == 0 && tl1)) && (e2 > 0 || (e2 == 0 && tl2)))) return;
    const double l0 = e0 * inv_area, l1 = e1 * inv_area, l2 = e2 * inv_area;
    const double z = (l0 * T.z0 + l1 * T.z1) + l2 * T.z2;
    const float z32 = static_cast<float>(z);
    if (!(z32 >= 0.f && z32 < 1.f)) return;           // depth clip; LESS against the cleared 1.0
    const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z32)) << 32) | static_cast<unsigned>(t);
    atomicMin(&keys[(j >> 2) * kRS + i], key);
}

// ---- triangles the screen-space set-up cannot take (a vertex at or behind the eye plane, or projected beyond 2^25 sub-pixels) ----
// GL clips such a triangle against the near plane.  Here it is rasterised in homogeneous coordinates: with M the clip-space
// (x, y, w) of the three vertices as columns, beta = M^-1 (px, py, 1) are the perspective-correct weights of the point seen through
// the pixel centre (px, py in NDC), scaled so that its w is 1 -- the point lies inside the triangle and in front of the eye iff all
// beta >= 0 -- and the ordinary depth test 0 <= z_window removes what lies before the near plane: the same fragments polygon
// clipping produces, with no new vertices.  Same arithmetic, same association as oracle/se3_oracle.py (_straddler_setup).
struct Strad {
    double A[3], B[3], C[3], idet, z[3], w[3];
    int i[3];
    int ia, ib, ja, jb;
    bool ok;
};

__device__ __noinline__ void straddler_setup(const Uniforms& u, const MeshDev& m, int t, Strad& S) {
    S.ok = false;
    double cl[3][4];
    bool finite = true, eye_side = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        S.i[k] = m.faces[3 * t + k];
        clip_coords(u, m.pos, S.i[k], cl[k]);
#pragma unroll
        for (int c = 0; c < 4; ++c) finite = finite && isfinite(cl[k][c]);
        eye_side = eye_side && (cl[k][2] + cl[k][3] < 0.0);
    }
    if (!finite || eye_side) return;                // nothing of it lies beyond the near plane
    // pixel box of the part beyond the near plane (only has to be conservative: one pixel of margin, the whole window when in doubt)
    double mnx = 1e300, mxx = -1e300, mny = 1e300, mxy = -1e300;
    bool any = false, wild = false;
    auto take = [&](double x, double y, double w) {
        const double xs = (x / w + 1.0) * u.hx, ys = (y / w + 1.0) * u.hy;
        if (!(isfinite(xs) && isfinite(ys) && fabs(xs) < 1e9 && fabs(ys) < 1e9)) wild = true;
        mnx = fmin(mnx, xs); mxx = fmax(mxx, xs); mny = fmin(mny, ys); mxy = fmax(mxy, ys);
        any = true;
    };
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const int b = (a + 1) % 3;
        const double da = cl[a][2] + cl[a][3], db = cl[b][2] + cl[b][3];
        if (da >= 0.0) take(cl[a][0], cl[a][1], cl[a][3]);
        if ((da >= 0.0) != (db >= 0.0)) {
            const double s = da / (da - db);
            take(cl[a][0] + s * (cl[b][0] - cl[a][0]), cl[a][1] + s * (cl[b][1] - cl[a][1]), cl[a][3] + s * (cl[b][3] - cl[a][3]));
        }
    }
    if (!any) return;
    if (wild) { S.ia = 0; S.ib = u.vw - 1; S.ja = 0; S.jb = u.vh - 1; }          // viewport pixels
    else {
        S.ia = max(0, static_cast<int>(floor(mnx)) - 1); S.ib = min(u.vw - 1, static_cast<int>(ceil(mxx)) + 1);
        S.ja = max(0, static_cast<int>(floor(mny)) - 1); S.jb = min(u.vh - 1, static_cast<int>(ceil(mxy)) + 1);
    }
    if (S.ia > S.ib || S.ja > S.jb) return;
    const double x0 = cl[0][0], y0 = cl[0][1], w0 = cl[0][3], x1 = cl[1][0], y1 = cl[1][1], w1 = cl[1][3], x2 = cl[2][0], y2 = cl[2][1], w2 = cl[2][3];
    S.A[0] = y1 * w2 - y2 * w1; S.A[1] = y2 * w0 - y0 * w2; S.A[2] = y0 * w1 - y1 * w0;
    S.B[0] = x2 * w1 - x1 * w2; S.B[1] = x0 * w2 - x2 * w0; S.B[2] = x1 * w0 - x0 * w1;
    S.C[0] = x1 * y2 - x2 * y1; S.C[1] = x2 * y0 - x0 * y2; S.C[2] = x0 * y1 - x1 * y0;
    const double det = (x0 * S.A[0] + x1 * S.A[1]) + x2 * S.A[2];
    if (det == 0.0 || !isfinite(det)) return;
    S.idet = 1.0 / det;
    S.z[0] = cl[0][2]; S.z[1] = cl[1][2]; S.z[2] = cl[2][2];
    S.w[0] = w0; S.w[1] = w1; S.w[2] = w2;
    S.ok = true;
}

// (i, j): VIEWPORT pixel (its centre in NDC is ((2i + 1 - vw) / vw, (2j + 1 - vh) / vh))
__device__ __forceinline__ void straddler_weights(const Strad& S, int i, int j, int vw, int vh, double& b0, double& b1, double& b2) {
    const double px = static_cast<double>(2 * i + 1 - vw) / static_cast<double>(vw), py = static_cast<double>(2 * j + 1 - vh) / static_cast<double>(vh);
    b0 = ((S.A[0] * px + S.B[0] * py) + S.C[0]) * S.idet;
    b1 = ((S.A[1] * px + S.B[1] * py) + S.C[1]) * S.idet;
    b2 = ((S.A[2] * px + S.B[2] * py) + S.C[2]) * S.idet;
}

__device__ __forceinline__ void straddler_pixel(const Strad& S, int t, int i, int j, const Samples& sm, unsigned long long* keys) {
    const int ipx = sm.xs[i] >> 8, jpx = sm.ys[j] >> 8;
    if (static_cast<unsigned>(ipx) >= static_cast<unsigned>(sm.vw) || static_cast<unsigned>(jpx) >= static_cast<unsigned>(sm.vh)) return;
    double b0, b1, b2;
    straddler_weights(S, ipx, jpx, sm.vw, sm.vh, b0, b1, b2);
    if (!(b0 >= 0.0 && b1 >= 0.0 && b2 >= 0.0)) return;
    const double zc = (b0 * S.z[0] + b1 * S.z[1]) + b2 * S.z[2], wc = (b0 * S.w[0] + b1 * S.w[1]) + b2 * S.w[2];
    const float z32 = static_cast<float>((zc / wc + 1.0) * 0.5);
    if (!(z32 >= 0.f && z32 < 1.f)) return;           // the near-plane cut (and the far one)
    const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z32)) << 32) | static_cast<unsigned>(t);
    atomicMin(&keys[(j >> 2) * kRS + i], key);
}

// out of line (own stack frame): the ordinary triangles' register allocation must not pay for the rare path
// output pixels whose sample lies in [lo, hi] (sub-pixel units): tab is non-decreasing
__device__ __forceinline__ int first_at_least(const int* tab, long long v) {       // first index with tab[i] >= v (kRS if none)
    int lo = 0, hi = kRS;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (tab[mid] < v) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ int last_at_most(const int* tab, long long v) {         // last index with tab[i] <= v (-1 if none)
    int lo = 0, hi = kRS;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (tab[mid] <= v) lo = mid + 1; else hi = mid; }
    return lo - 1;
}

__device__ __noinline__ void raster_straddler(const Uniforms& u, const MeshDev& m, int t, int band, int lane, const Samples& sm, unsigned long long* keys) {
    Strad S;
    straddler_setup(u, m, t, S);
    if (!S.ok) return;
    // viewport-pixel box -> output pixels whose sample falls inside it
    const int ia = first_at_least(sm.xs, static_cast<long long>(S.ia) * kSub), ib = last_at_most(sm.xs, static_cast<long long>(S.ib) * kSub + (kSub - 1));
    const int ja = first_at_least(sm.ys, static_cast<long long>(S.ja) * kSub), jb = last_at_most(sm.ys, static_cast<long long>(S.jb) * kSub + (kSub - 1));
    if (ia > ib || ja > jb) return;
    const int j0 = ja + ((band - (ja & 3)) & 3);             // first row >= ja that this CTA owns
    if (j0 > jb) return;
    const int bw = ib - ia + 1, cnt = bw * ((jb - j0) / 4 + 1);
    for (int k = lane; k < cnt; k += 32) straddler_pixel(S, t, ia + k % bw, j0 + 4 * (k / bw), sm, keys);
}

__device__ __noinline__ void resolve_straddler(const Uniforms& u, const MeshDev& m, int t, int ipx, int jpx, double* q, int* idx) {
    Strad S;
    straddler_setup(u, m, t, S);
    straddler_weights(S, ipx, jpx, u.vw, u.vh, q[0], q[1], q[2]);
    idx[0] = S.i[0]; idx[1] = S.i[1]; idx[2] = S.i[2];
}

__device__ void make_uniforms(const RenderArgs& a, int n, int nf, Uniforms& u) {
        const double* pose = a.poses + n * 16;
        int top, left, ch, cw;
        // view = inv(glcam_in_cvcam) . ob2cam (rows 1, 2 negated), uploaded as float32
        for (int c = 0; c < 4; ++c) {
            u.V[c] = static_cast<double>(static_cast<float>(pose[c]));
            u.V[4 + c] = static_cast<double>(static_cast<float>(-pose[4 + c]));
            u.V[8 + c] = static_cast<double>(static_cast<float>(-pose[8 + c]));
        }
        const double nr = 0.1, fr = 2.0;
        u.mode = a.mode;
        if (a.mode != 0) {
            // the whole camera image is the viewport (pyrender IntrinsicsCamera, offscreen_renderer.py:52-53).  Mode 1: crop_bbox's
            // window (predict.py:211: scale (1000, 1000, 1000), no y flip) selects the samples; mode 2 (the coverage pass) has none
            if (a.mode == 1) bbox_window(pose, a.fx, a.fy, a.cx, a.cy, a.object_width[n], 1000.0, 1000.0, 1000.0, top, left, ch, cw);
            else top = left = 0, ch = a.vh, cw = a.vw;
            u.valid = (cw > 0 && ch > 0 && nf > 0 && a.vw > 0 && a.vh > 0) ? 1 : 0;
            u.vw = a.vw; u.vh = a.vh; u.hx = a.vw * 0.5; u.hy = a.vh * 0.5;
            u.top = top; u.left = left; u.ch = ch; u.cw = cw;
            u.P00 = static_cast<float>(2.0 * a.fx / a.vw); u.P02 = static_cast<float>(1.0 - 2.0 * a.cx / a.vw);
            u.P11 = static_cast<float>(2.0 * a.fy / a.vh); u.P12 = static_cast<float>(2.0 * a.cy / a.vh - 1.0);
            u.P22 = static_cast<float>((fr + nr) / (nr - fr)); u.P23 = static_cast<float>((2 * fr * nr) / (nr - fr));
            u.A = u.B = 0.0; u.light[0] = u.light[1] = u.light[2] = 0.0;
            if (!(isfinite(u.P00) && isfinite(u.P02) && isfinite(u.P11) && isfinite(u.P12))) u.valid = 0;
            return;
        }
        bbox_window(pose, a.fx, a.fy, a.cx, a.cy, a.object_width[n], 1000.0, -1000.0, 1000.0, top, left, ch, cw);   // predict.py:202
        const int right = left + cw, bottom = top + ch;
        u.valid = (cw != 0 && ch != 0 && nf > 0) ? 1 : 0;
        u.vw = u.vh = kRS; u.hx = u.hy = kRS * 0.5;
        u.top = top; u.left = left; u.ch = ch; u.cw = cw;
        const double o00 = static_cast<float>(2.0 / (right - left)), o03 = static_cast<float>(static_cast<double>(-(right + left)) / (right - left));
        const double o11 = static_cast<float>(2.0 / (top - bottom)), o13 = static_cast<float>(static_cast<double>(-(top + bottom)) / (top - bottom));
        const double o22 = static_cast<float>(-2.0 / (fr - nr)), o23 = static_cast<float>(-(fr + nr) / (fr - nr));
        const double P00 = o00 * a.fx, P02 = o00 * (-a.cx) + o03 * (-1.0);
        const double P11 = o11 * a.fy, P12 = o11 * (-a.cy) + o13 * (-1.0);
        const double P22 = o22 * (nr + fr) + o23 * (-1.0), P23 = o22 * (nr * fr);
        u.A = P22; u.B = P23;
        u.P00 = static_cast<float>(P00); u.P02 = static_cast<float>(P02); u.P11 = static_cast<float>(P11);
        u.P12 = static_cast<float>(P12); u.P22 = static_cast<float>(P22); u.P23 = static_cast<float>(P23);
        if (!(isfinite(u.P00) && isfinite(u.P02) && isfinite(u.P11) && isfinite(u.P12))) u.valid = 0;
        // light_direction = (inv(view^T) . (0, .1, -.9, 1))[:3] = R_gl . (0, .1, -.9)     (vispy_renderer.py:172)
        for (int r = 0; r < 3; ++r) {
            const double sgn = r == 0 ? 1.0 : -1.0;
            const double r0 = sgn * pose[4 * r], r1 = sgn * pose[4 * r + 1], r2 = sgn * pose[4 * r + 2];
            u.light[r] = static_cast<double>(static_cast<float>((r0 * 0.0 + r1 * 0.1) + r2 * (-0.9)));
        }
    }

constexpr int kProjThreads = 256;
__global__ void __launch_bounds__(kProjThreads)
render_project_kernel(RenderArgs a)
{
    __shared__ Uniforms u;
    ptx::grid_dep_launch();
    const int n = blockIdx.y;
    // poses come from the previous step's pose update, or in a refinement round from the previous round's head, which this
    // launch may start under: every read of them, and every write of `projected` / `uniforms` (which the previous round's
    // render_kernel read), stays behind this wait
    ptx::grid_dep_wait();
    int mid = a.mesh_ids ? a.mesh_ids[n] : 0;
    if (mid < 0 || mid >= a.n_meshes) mid = 0;
    const MeshDev m = a.meshes[mid];
    if (static_cast<int>(blockIdx.x * blockDim.x) >= m.nv && blockIdx.x != 0) return;
    if (threadIdx.x == 0) make_uniforms(a, n, m.nf, u);
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < sizeof(Uniforms) / sizeof(double))          // one copy per track for render_kernel
        reinterpret_cast<double*>(a.uniforms + static_cast<size_t>(n) * sizeof(Uniforms))[threadIdx.x] = reinterpret_cast<const double*>(&u)[threadIdx.x];
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= m.nv) return;
    PVtx q; q.X = INT_MIN; q.Y = 0; q.zw = 0; q.iw = 0;
    if (u.valid) {
        const Vtx v = project(u, m.pos, vi);
        if (v.ok) { q.X = static_cast<int>(v.X); q.Y = static_cast<int>(v.Y); q.zw = v.zw; q.iw = 1.0 / v.w; }
    }
    reinterpret_cast<PVtx*>(a.projected)[static_cast<size_t>(n) * a.max_nv + vi] = q;
}

__global__ void __launch_bounds__(kRenderThreads, 2)
render_kernel(RenderArgs a)
{
    extern __shared__ unsigned long long keys[];            // [kBandRows][kRS]: rows band, band + 4, band + 8, ...
    __shared__ Uniforms u;
    ptx::grid_dep_launch();
    const int n = blockIdx.y, band = blockIdx.x;
    for (int k = threadIdx.x; k < kBandRows * kRS; k += blockDim.x) keys[k] = kClearKey;
    ptx::grid_dep_wait();                                    // projected vertices + uniforms come from render_project_kernel
    int mid = a.mesh_ids ? a.mesh_ids[n] : 0;
    if (mid < 0 || mid >= a.n_meshes) mid = 0;
    const MeshDev m = a.meshes[mid];
    const PVtx* __restrict__ pv = reinterpret_cast<const PVtx*>(a.projected) + static_cast<size_t>(n) * a.max_nv;
    if (threadIdx.x < sizeof(Uniforms) / sizeof(double))
        reinterpret_cast<double*>(&u)[threadIdx.x] = reinterpret_cast<const double*>(a.uniforms + static_cast<size_t>(n) * sizeof(Uniforms))[threadIdx.x];
    __syncthreads();
    // sample positions of the 176 output columns / rows (rows bottom-up: window y grows with the index)
    __shared__ int s_xs[kRS], s_ys[kRS];
    if (threadIdx.x < 2 * kRS) {
        const int k = threadIdx.x < kRS ? threadIdx.x : threadIdx.x - kRS;
        const bool isx = threadIdx.x < kRS;
        int v = k * kSub + kHalf;                               // mode 0: the pixel's own centre
        if (u.mode == 1 && u.valid) {
            // crop_bbox (Utils.py:343-344): cv2 INTER_NEAREST source index floor(dst * (1 / (176 / size))), clamped -- as in crop_kernel
            const int size = isx ? u.cw : u.ch;
            const int dst = isx ? k : (kRS - 1 - k);            // output row r = 175 - k (the image's rows run top-down)
            const double inv = 1.0 / (static_cast<double>(kRS) / size);
            int src = static_cast<int>(floor(dst * inv)); if (src > size - 1) src = size - 1;
            long long pix = static_cast<long long>(isx ? u.left : u.top) + src;           // camera-image column / row
            if (!isx) pix = static_cast<long long>(u.vh) - 1 - pix;                        // GL window rows run bottom-up
            pix = max(-1ll, min(static_cast<long long>(isx ? u.vw : u.vh), pix));         // outside the viewport: no fragment (kept monotone)
            v = static_cast<int>(pix) * kSub + kHalf;
        }
        (isx ? s_xs : s_ys)[k] = v;
    }
    __syncthreads();
    const Samples sm = {s_xs, s_ys, u.vw, u.vh};
    const bool tables = u.mode != 0;
    const int lane = threadIdx.x & 31;
    // first row >= ja that this CTA owns
    auto first_row = [band](int ja) { return ja + ((band - (ja & 3)) & 3); };
    // output columns / rows whose sample lies inside [mn, mx] (sub-pixel units)
    auto span = [&](const int* tab, long long mn, long long mx, int& a0, int& a1) {
        if (tables) { a0 = first_at_least(tab, mn); a1 = last_at_most(tab, mx); }
        else { a0 = static_cast<int>(max(0ll, floor_div(mn - kHalf + kSub - 1, kSub))); a1 = static_cast<int>(min(static_cast<long long>(kRS - 1), floor_div(mx - kHalf, kSub))); }
    };
    if (u.valid) {
        // ---------------- pass 1: visibility ----------------
        const int nf_pad = (m.nf + 31) & ~31;                // whole warps walk the loop (ballots below)
        // the rows of triangle t decide whether this CTA has to look at it at all (three 4-byte loads instead of the full set-up);
        // they are fetched one iteration ahead so the two dependent L2 round trips overlap the previous triangle's work
        // returns 0: nothing to do, 1: ordinary triangle (rows in y0..y2), 2: a vertex has no screen position (near-plane straddler)
        auto fetch_rows = [&](int t, int& y0, int& y1, int& y2) -> int {
            if (t >= m.nf) return 0;
            const unsigned i0 = m.faces[3 * t], i1 = m.faces[3 * t + 1], i2 = m.faces[3 * t + 2];
            if (!(i0 < static_cast<unsigned>(m.nv) && i1 < static_cast<unsigned>(m.nv) && i2 < static_cast<unsigned>(m.nv))) return 0;
            const int2 a = *reinterpret_cast<const int2*>(&pv[i0]), b = *reinterpret_cast<const int2*>(&pv[i1]), c = *reinterpret_cast<const int2*>(&pv[i2]);
            y0 = a.y; y1 = b.y; y2 = c.y;
            return (a.x == INT_MIN || b.x == INT_MIN || c.x == INT_MIN) ? 2 : 1;
        };
        int ny0 = 0, ny1 = 0, ny2 = 0;
        int nvalid = fetch_rows(threadIdx.x, ny0, ny1, ny2);
        for (int t = threadIdx.x; t < nf_pad; t += blockDim.x) {
            bool big = false;
            bool mine = false;
            const bool valid = nvalid == 1, strad = nvalid == 2; const int y0 = ny0, y1 = ny1, y2 = ny2;
            nvalid = fetch_rows(t + blockDim.x, ny0, ny1, ny2);
            if (valid) {
                const long long mny = min(y0, min(y1, y2)), mxy = max(y0, max(y1, y2));
                int ja, jb;
                span(s_ys, mny, mxy, ja, jb);
                mine = ja <= jb && first_row(ja) <= jb;
            }
            if (mine) {
                const Tri T = setup(pv, m, t);
                if (T.ok) {
                    const long long mnx = min(T.x0, min(T.x1, T.x2)), mxx = max(T.x0, max(T.x1, T.x2));
                    const long long mny = min(T.y0, min(T.y1, T.y2)), mxy = max(T.y0, max(T.y1, T.y2));
                    int ia, ib, ja, jb;
                    span(s_xs, mnx, mxx, ia, ib); span(s_ys, mny, mxy, ja, jb);
                    const int j0 = first_row(ja);
                    if (ia <= ib && j0 <= jb) {
                        if ((ib - ia + 1) * ((jb - j0) / 4 + 1) > kBigBox) big = true;
                        else {
                            const bool tl0 = top_left(T.x2 - T.x1, T.y2 - T.y1), tl1 = top_left(T.x0 - T.x2, T.y0 - T.y2), tl2 = top_left(T.x1 - T.x0, T.y1 - T.y0);
                            const double inv_area = 1.0 / static_cast<double>(T.area2);
                            const EdgeSet E = edge_set(T);
                            for (int j = j0; j <= jb; j += 4)
                                for (int i = ia; i <= ib; ++i) raster_pixel(T, E, inv_area, t, i, j, tl0, tl1, tl2, sm, keys);
                        }
                    }
                }
            }
            unsigned bigmask = __ballot_sync(0xffffffffu, big);
            while (bigmask) {                                // large triangles: the whole warp walks the bounding box
                const int src = __ffs(bigmask) - 1; bigmask &= bigmask - 1;
                const int tb = __shfl_sync(0xffffffffu, t, src);
                const Tri T = setup(pv, m, tb);
                const long long mnx = min(T.x0, min(T.x1, T.x2)), mxx = max(T.x0, max(T.x1, T.x2));
                const long long mny = min(T.y0, min(T.y1, T.y2)), mxy = max(T.y0, max(T.y1, T.y2));
                int ia, ib, ja, jb;
                span(s_xs, mnx, mxx, ia, ib); span(s_ys, mny, mxy, ja, jb);
                const int j0 = first_row(ja);
                const bool tl0 = top_left(T.x2 - T.x1, T.y2 - T.y1), tl1 = top_left(T.x0 - T.x2, T.y0 - T.y2), tl2 = top_left(T.x1 - T.x0, T.y1 - T.y0);
                const double inv_area = 1.0 / static_cast<double>(T.area2);
                const EdgeSet E = edge_set(T);
                const int bw = ib - ia + 1, cnt = bw * ((jb - j0) / 4 + 1);
                for (int k = lane; k < cnt; k += 32) raster_pixel(T, E, inv_area, tb, ia + k % bw, j0 + 4 * (k / bw), tl0, tl1, tl2, sm, keys);
            }
            unsigned smask = __ballot_sync(0xffffffffu, strad);
            while (smask) {                                  // near-plane straddlers (rare): the whole warp, homogeneous weights
                const int src = __ffs(smask) - 1; smask &= smask - 1;
                const int tb = __shfl_sync(0xffffffffu, t, src);
                raster_straddler(u, m, tb, band, lane, sm, keys);
            }
        }
    }
    __syncthreads();
    // ---------------- pass 2: resolve + shade ----------------
    const double far_dist = u.B / (u.A + 1.0);
    for (int k = threadIdx.x; k < kBandRows * kRS; k += blockDim.x) {
        const int j = 4 * (k / kRS) + band, i = k % kRS;
        const unsigned long long key = keys[k];
        const unsigned t = static_cast<unsigned>(key & 0xFFFFFFFFull);
        unsigned r8 = 0, g8 = 0, b8 = 0, mm = 0;
        if (u.valid && t != 0xFFFFFFFFu) {
            const Tri T = setup(pv, m, static_cast<int>(t));
            double q0, q1, q2;                               // perspective-correct weights (not normalised)
            int i0, i1, i2;
            if (T.ok) {
                double e0, e1, e2;
                edges(edge_set(T), static_cast<double>(s_xs[i]), static_cast<double>(s_ys[j]), e0, e1, e2);
                const double inv_area = 1.0 / static_cast<double>(T.area2);
                const double l0 = e0 * inv_area, l1 = e1 * inv_area, l2 = e2 * inv_area;
                q0 = l0 * T.w0; q1 = l1 * T.w1; q2 = l2 * T.w2;                  // T.w* = 1/w
                i0 = T.i0; i1 = T.i1; i2 = T.i2;
            } else {                                         // near-plane straddler: the homogeneous weights are the perspective-correct ones
                double q[3]; int idx[3];
                resolve_straddler(u, m, static_cast<int>(t), s_xs[i] >> 8, s_ys[j] >> 8, q, idx);
                q0 = q[0]; q1 = q[1]; q2 = q[2]; i0 = idx[0]; i1 = idx[1]; i2 = idx[2];
            }
            const double rq = 1.0 / ((q0 + q1) + q2);
            double pos[3], nrm[3], col[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double c0 = static_cast<float>(m.col[3 * i0 + c] / 255.0), c1 = static_cast<float>(m.col[3 * i1 + c] / 255.0), c2 = static_cast<float>(m.col[3 * i2 + c] / 255.0);
                col[c] = ((q0 * c0 + q1 * c1) + q2 * c2) * rq;
            }
            const float d32 = __uint_as_float(static_cast<unsigned>(key >> 32));
            if (u.mode == 1) {
                // pyrender with ambient light 1 and no other light (offscreen_renderer.py:50): the fragment is its base colour;
                // depth read-back linearised in float32: 2 n f / (f + n - (2 d - 1)(f - n)), then (depth * 1000).astype(uint16) (predict.py:213)
                r8 = static_cast<unsigned>(rint(fmin(fmax(col[0], 0.0), 1.0) * 255.0));
                g8 = static_cast<unsigned>(rint(fmin(fmax(col[1], 0.0), 1.0) * 255.0));
                b8 = static_cast<unsigned>(rint(fmin(fmax(col[2], 0.0), 1.0) * 255.0));
                const float zn = 0.1f, zf = 2.0f;
                const float zndc = __fsub_rn(__fmul_rn(2.0f, d32), 1.0f);
                const float den = __fsub_rn(__fadd_rn(zf, zn), __fmul_rn(zndc, __fsub_rn(zf, zn)));
                const float metres = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, zn), zf), den);
                mm = static_cast<unsigned>(static_cast<unsigned short>(static_cast<int>(__fmul_rn(metres, 1000.0f))));
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    pos[c] = ((q0 * static_cast<double>(m.pos[3 * i0 + c]) + q1 * static_cast<double>(m.pos[3 * i1 + c])) + q2 * static_cast<double>(m.pos[3 * i2 + c])) * rq;
                    nrm[c] = ((q0 * static_cast<double>(m.nrm[3 * i0 + c]) + q1 * static_cast<double>(m.nrm[3 * i1 + c])) + q2 * static_cast<double>(m.nrm[3 * i2 + c])) * rq;
                }
                const double x0 = (-u.light[0]) - pos[0], x1 = (-u.light[1]) - pos[1], x2 = (-u.light[2]) - pos[2];
                const double il = 1.0 / sqrt((x0 * x0 + x1 * x1) + x2 * x2);
                const double d = (nrm[0] * (x0 * il) + nrm[1] * (x1 * il)) + nrm[2] * (x2 * il);
                // fmax drops a NaN operand: a NaN Lambert term (a zero-length normal normalised to NaN) counts as 0, the fragment
                // gets the ambient 0.65 alone.  GLSL leaves max() of a NaN undefined; NVIDIA's max instruction returns the other
                // operand as fmax does.  oracle/se3_oracle.py (render_window) states the same rule
                const double lightv = 0.4 * fmax(d, 0.0) + 0.65;
                r8 = static_cast<unsigned>(rint(fmin(fmax(lightv * col[0], 0.0), 1.0) * 255.0));
                g8 = static_cast<unsigned>(rint(fmin(fmax(lightv * col[1], 0.0), 1.0) * 255.0));
                b8 = static_cast<unsigned>(rint(fmin(fmax(lightv * col[2], 0.0), 1.0) * 255.0));
                // on_draw: distance = B / (depth * -2.0 + 1.0 - A) * -1 (float32 until `- A`), background -> 0, mm = uint16(distance * 1000)
                const float tt = __fadd_rn(__fmul_rn(d32, -2.0f), 1.0f);
                const double dist = (u.B / (static_cast<double>(tt) - u.A)) * -1.0;
                if (!(dist >= far_dist)) mm = static_cast<unsigned>(static_cast<unsigned short>(static_cast<int>(dist * 1000.0)));
            }
        }
        const int orow = u.mode == 1 ? (kRS - 1 - j) : j;         // mode 1: rows were walked bottom-up, the image is stored top-down
        const size_t o = (static_cast<size_t>(n) * kRS + orow) * kRS + i;
        if (a.rgb) { a.rgb[o * 3] = static_cast<uint8_t>(r8); a.rgb[o * 3 + 1] = static_cast<uint8_t>(g8); a.rgb[o * 3 + 2] = static_cast<uint8_t>(b8); }
        a.depth[o] = static_cast<uint16_t>(mm);
        if (a.tri) a.tri[o] = (u.valid && t != 0xFFFFFFFFu) ? static_cast<int32_t>(t) : -1;
    }
}

// ---------------- coverage: the nearest depth of every pixel of the WHOLE camera image (pyrender mode, uniforms of mode 2) ----------------
// What np.sum(depth > 0.1) needs of Renderer.render's depth (produce_train_pair_data.py:101-102): only the nearest fragment of each
// pixel, so no triangle index is kept -- zmin[j][i] = min over fragments of the float32 window-z bits (positive floats order as their
// bits; -0.0 never wins, as it never wins the 64-bit keys of render_kernel or of the oracle).  Same set-up, edge functions, top-left
// rule, depth clip and near-plane path as render_kernel; one thread per triangle, boxes above kBigBox pixels walked by the warp.
constexpr int kCoverThreads = 256;
constexpr unsigned kCoverClear = 0x7F7F7F7Fu;         // cudaMemset byte 0x7F: above every z in [0, 1)

__device__ __forceinline__ void cover_pixel(const Tri& T, const EdgeSet& E, double inv_area, int i, int j, bool tl0, bool tl1, bool tl2,
                                            unsigned* zmin, int vw) {
    const double cx = static_cast<double>(i * kSub + kHalf), cy = static_cast<double>(j * kSub + kHalf);
    double e0, e1, e2;
    edges(E, cx, cy, e0, e1, e2);
    if (!((e0 > 0 || (e0 == 0 && tl0)) && (e1 > 0 || (e1 == 0 && tl1)) && (e2 > 0 || (e2 == 0 && tl2)))) return;
    const double l0 = e0 * inv_area, l1 = e1 * inv_area, l2 = e2 * inv_area;
    const double z = (l0 * T.z0 + l1 * T.z1) + l2 * T.z2;
    const float z32 = static_cast<float>(z);
    if (!(z32 >= 0.f && z32 < 1.f)) return;
    atomicMin(&zmin[static_cast<size_t>(j) * vw + i], __float_as_uint(z32));
}

__device__ __noinline__ void cover_straddler(const Uniforms& u, const MeshDev& m, int t, int lane, unsigned* zmin) {
    Strad S;
    straddler_setup(u, m, t, S);
    if (!S.ok) return;
    const int bw = S.ib - S.ia + 1, cnt = bw * (S.jb - S.ja + 1);
    for (int k = lane; k < cnt; k += 32) {
        const int i = S.ia + k % bw, j = S.ja + k / bw;
        double b0, b1, b2;
        straddler_weights(S, i, j, u.vw, u.vh, b0, b1, b2);
        if (!(b0 >= 0.0 && b1 >= 0.0 && b2 >= 0.0)) continue;
        const double zc = (b0 * S.z[0] + b1 * S.z[1]) + b2 * S.z[2], wc = (b0 * S.w[0] + b1 * S.w[1]) + b2 * S.w[2];
        const float z32 = static_cast<float>((zc / wc + 1.0) * 0.5);
        if (!(z32 >= 0.f && z32 < 1.f)) continue;
        atomicMin(&zmin[static_cast<size_t>(j) * u.vw + i], __float_as_uint(z32));
    }
}

// grid (triangle blocks, n): zmin (n, vh, vw), window rows bottom-up
__global__ void __launch_bounds__(kCoverThreads)
coverage_kernel(RenderArgs a, unsigned* __restrict__ zmin_all)
{
    __shared__ Uniforms u;
    const int n = blockIdx.y;
    ptx::grid_dep_wait();                                    // projected vertices + uniforms come from render_project_kernel
    int mid = a.mesh_ids ? a.mesh_ids[n] : 0;
    if (mid < 0 || mid >= a.n_meshes) mid = 0;
    const MeshDev m = a.meshes[mid];
    if (static_cast<int>(blockIdx.x * blockDim.x) >= m.nf) return;      // whole CTA past this model's triangles
    if (threadIdx.x < sizeof(Uniforms) / sizeof(double))
        reinterpret_cast<double*>(&u)[threadIdx.x] = reinterpret_cast<const double*>(a.uniforms + static_cast<size_t>(n) * sizeof(Uniforms))[threadIdx.x];
    __syncthreads();
    if (!u.valid) return;
    const PVtx* __restrict__ pv = reinterpret_cast<const PVtx*>(a.projected) + static_cast<size_t>(n) * a.max_nv;
    unsigned* zmin = zmin_all + static_cast<size_t>(n) * u.vw * u.vh;
    const int lane = threadIdx.x & 31;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    bool big = false, strad = false;
    if (t < m.nf) {
        const unsigned i0 = m.faces[3 * t], i1 = m.faces[3 * t + 1], i2 = m.faces[3 * t + 2];
        const bool idx_ok = i0 < static_cast<unsigned>(m.nv) && i1 < static_cast<unsigned>(m.nv) && i2 < static_cast<unsigned>(m.nv);
        strad = idx_ok && (pv[i0].X == INT_MIN || pv[i1].X == INT_MIN || pv[i2].X == INT_MIN);
        const Tri T = (idx_ok && !strad) ? setup(pv, m, t) : Tri{};
        if (idx_ok && !strad && T.ok) {
            const long long mnx = min(T.x0, min(T.x1, T.x2)), mxx = max(T.x0, max(T.x1, T.x2));
            const long long mny = min(T.y0, min(T.y1, T.y2)), mxy = max(T.y0, max(T.y1, T.y2));
            const int ia = static_cast<int>(max(0ll, floor_div(mnx - kHalf + kSub - 1, kSub))), ib = static_cast<int>(min(static_cast<long long>(u.vw - 1), floor_div(mxx - kHalf, kSub)));
            const int ja = static_cast<int>(max(0ll, floor_div(mny - kHalf + kSub - 1, kSub))), jb = static_cast<int>(min(static_cast<long long>(u.vh - 1), floor_div(mxy - kHalf, kSub)));
            if (ia <= ib && ja <= jb) {
                if (static_cast<long long>(ib - ia + 1) * (jb - ja + 1) > kBigBox) big = true;
                else {
                    const bool tl0 = top_left(T.x2 - T.x1, T.y2 - T.y1), tl1 = top_left(T.x0 - T.x2, T.y0 - T.y2), tl2 = top_left(T.x1 - T.x0, T.y1 - T.y0);
                    const double inv_area = 1.0 / static_cast<double>(T.area2);
                    const EdgeSet E = edge_set(T);
                    for (int j = ja; j <= jb; ++j)
                        for (int i = ia; i <= ib; ++i) cover_pixel(T, E, inv_area, i, j, tl0, tl1, tl2, zmin, u.vw);
                }
            }
        }
    }
    unsigned bigmask = __ballot_sync(0xffffffffu, big);
    while (bigmask) {                                        // large triangles: the whole warp walks the bounding box
        const int src = __ffs(bigmask) - 1; bigmask &= bigmask - 1;
        const int tb = __shfl_sync(0xffffffffu, t, src);
        const Tri T = setup(pv, m, tb);
        const long long mnx = min(T.x0, min(T.x1, T.x2)), mxx = max(T.x0, max(T.x1, T.x2));
        const long long mny = min(T.y0, min(T.y1, T.y2)), mxy = max(T.y0, max(T.y1, T.y2));
        const int ia = static_cast<int>(max(0ll, floor_div(mnx - kHalf + kSub - 1, kSub))), ib = static_cast<int>(min(static_cast<long long>(u.vw - 1), floor_div(mxx - kHalf, kSub)));
        const int ja = static_cast<int>(max(0ll, floor_div(mny - kHalf + kSub - 1, kSub))), jb = static_cast<int>(min(static_cast<long long>(u.vh - 1), floor_div(mxy - kHalf, kSub)));
        const bool tl0 = top_left(T.x2 - T.x1, T.y2 - T.y1), tl1 = top_left(T.x0 - T.x2, T.y0 - T.y2), tl2 = top_left(T.x1 - T.x0, T.y1 - T.y0);
        const double inv_area = 1.0 / static_cast<double>(T.area2);
        const EdgeSet E = edge_set(T);
        const int bw = ib - ia + 1, cnt = bw * (jb - ja + 1);
        for (int k = lane; k < cnt; k += 32) cover_pixel(T, E, inv_area, ia + k % bw, ja + k / bw, tl0, tl1, tl2, zmin, u.vw);
    }
    unsigned smask = __ballot_sync(0xffffffffu, strad);
    while (smask) {                                          // near-plane straddlers (rare): the whole warp, homogeneous weights
        const int src = __ffs(smask) - 1; smask &= smask - 1;
        cover_straddler(u, m, __shfl_sync(0xffffffffu, t, src), lane, zmin);
    }
}

// Per row: visible = #(seg == class id) over the H x W frame, covered = #(linearised float32 depth of zmin > 0.1f).  One CTA
// strip of pixels per row, a block reduction, one atomicAdd per CTA into the zeroed counts (integer: any order is exact).
constexpr int kCountThreads = 256, kCountBlocks = 64;
__global__ void __launch_bounds__(kCountThreads)
coverage_count_kernel(const uint8_t* __restrict__ seg, const int* __restrict__ class_ids, const unsigned* __restrict__ zmin_all,
                      int HW, int* __restrict__ visible, int* __restrict__ covered)
{
    const int n = blockIdx.y;
    const int cid = class_ids[n];
    const unsigned* zmin = zmin_all + static_cast<size_t>(n) * HW;
    const float zn = 0.1f, zf = 2.0f;
    int cv = 0, cc = 0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        cv += static_cast<int>(seg[p]) == cid;
        const unsigned zb = zmin[p];
        if (zb != kCoverClear) {
            // offscreen_renderer.py -> pyrender's float32 linearisation, as render_kernel's mode 1 and render_full_frame_unlit
            const float zndc = __fsub_rn(__fmul_rn(2.0f, __uint_as_float(zb)), 1.0f);
            const float den = __fsub_rn(__fadd_rn(zf, zn), __fmul_rn(zndc, __fsub_rn(zf, zn)));
            const float metres = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, zn), zf), den);
            cc += metres > 0.1f;
        }
    }
    __shared__ int s_v[kCountThreads / 32], s_c[kCountThreads / 32];
    for (int o = 16; o > 0; o >>= 1) { cv += __shfl_xor_sync(0xffffffffu, cv, o); cc += __shfl_xor_sync(0xffffffffu, cc, o); }
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = cv; s_c[threadIdx.x >> 5] = cc; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int v = 0, c = 0;
        for (int w = 0; w < kCountThreads / 32; ++w) { v += s_v[w]; c += s_c[w]; }
        atomicAdd(&visible[n], v); atomicAdd(&covered[n], c);
    }
}
}  // namespace

size_t render_uniform_bytes() { return sizeof(Uniforms); }
size_t render_projected_bytes_per_vertex() { return sizeof(PVtx); }

cudaError_t launch_render(const RenderArgs& a, int n, cudaStream_t s, bool pdl) {
    if (n <= 0) return cudaSuccess;
    const size_t smem = static_cast<size_t>(kBandRows) * kRS * sizeof(unsigned long long);
    cudaError_t e = set_max_dynamic_smem<render_kernel>(smem);
    if (e != cudaSuccess) return e;
    if (!a.projected || !a.uniforms || a.max_nv <= 0) return cudaErrorInvalidValue;
    e = launch_kernel(render_project_kernel, dim3((a.max_nv + kProjThreads - 1) / kProjThreads, n), dim3(kProjThreads), 0, s, pdl, a);
    if (e != cudaSuccess) return e;
    return launch_kernel(render_kernel, dim3(kBands, n), dim3(kRenderThreads), smem, s, true, a);
}

cudaError_t launch_coverage(RenderArgs a, int n, int max_nf, const uint8_t* seg, const int* class_ids, unsigned* zmin,
                            int* visible, int* covered, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (!a.projected || !a.uniforms || a.max_nv <= 0 || max_nf <= 0 || a.vw <= 0 || a.vh <= 0) return cudaErrorInvalidValue;
    a.mode = 2; a.object_width = nullptr;
    const size_t hw = static_cast<size_t>(a.vw) * a.vh;
    cudaError_t e = cudaMemsetAsync(zmin, 0x7F, static_cast<size_t>(n) * hw * sizeof(unsigned), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(visible, 0, n * sizeof(int), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(covered, 0, n * sizeof(int), s);
    if (e != cudaSuccess) return e;
    e = launch_kernel(render_project_kernel, dim3((a.max_nv + kProjThreads - 1) / kProjThreads, n), dim3(kProjThreads), 0, s, false, a);
    if (e != cudaSuccess) return e;
    e = launch_kernel(coverage_kernel, dim3((max_nf + kCoverThreads - 1) / kCoverThreads, n), dim3(kCoverThreads), 0, s, false, a, zmin);
    if (e != cudaSuccess) return e;
    return launch_kernel(coverage_count_kernel, dim3(kCountBlocks, n), dim3(kCountThreads), 0, s, false, seg, class_ids,
                         static_cast<const unsigned*>(zmin), static_cast<int>(hw), visible, covered);
}

}  // namespace se3tn
