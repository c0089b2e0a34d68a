// Device functions of the geometry ops, shared by the standalone op kernels (geometry_ops.cu) and
// by the fused glue kernels between the network blocks (net.cu).
//
// Arithmetic follows the reference CPU kernels operation for operation (see oracle/geometry_ops_impl.h
// for the restatement these are checked against); reference file:line on each function.
#pragma once
#include "common.cuh"
#include <climits>
#include <cmath>

namespace demon {

// `(int)x` as x86 cvttss2si/cvttsd2si does it (warp2d.cc:196 `p2.template cast<int>()`): NaN and
// out-of-range give INT_MIN.  CUDA's own conversion saturates and maps NaN to 0, which would turn a
// NaN displacement into a valid sample at pixel 0.
template <class T>
__device__ __forceinline__ int cvtt_x86(T x) {
  if (!(x > (T)-2147483649.0 && x < (T)2147483648.0)) return INT_MIN;
  return (int)x;
}

// Bilinear sample position of warp2d (warp2d.cc:186-200): integer corner + the four weights.
template <class T>
struct WarpTap {
  int x0, y0;   // p2i
  T w0, w1, w2, w3;
};

template <class T>
__device__ __forceinline__ WarpTap<T> warp2d_tap(int x, int y, T vx, T vy, int x_size, int y_size, bool normalized) {
  WarpTap<T> r;
  if (normalized) { vx = fmul(vx, (T)x_size); vy = fmul(vy, (T)y_size); }
  T p2x = fadd((T)x, vx), p2y = fadd((T)y, vy);
  r.x0 = cvtt_x86(p2x);
  r.y0 = cvtt_x86(p2y);
  T a = fsub(p2x, (T)r.x0), b = fsub(p2y, (T)r.y0);
  T na = fsub((T)1, a), nb = fsub((T)1, b);
  r.w0 = fmul(na, nb); r.w1 = fmul(a, nb); r.w2 = fmul(na, b); r.w3 = fmul(a, b);
  return r;
}

// VALUE-mode validity test, warp2d.cc:236.  (x3 = x0+1 computed with wrap like the x86 add.)
__device__ __forceinline__ bool warp2d_valid(int x0, int y0, int x_size, int y_size) {
  int x3 = (int)((unsigned)x0 + 1u), y3 = (int)((unsigned)y0 + 1u);
  return x0 >= 0 && x3 > 0 && x3 < x_size && y0 >= 0 && y3 > 0 && y3 < y_size;
}

// dot(values, weights) as Eigen's 4-wide reduction does it: (p0+p2)+(p1+p3)
template <class T>
__device__ __forceinline__ T warp2d_blend(T v0, T v1, T v2, T v3, const WarpTap<T>& t) {
  return fadd(fadd(fmul(v0, t.w0), fmul(v2, t.w2)), fadd(fmul(v1, t.w1), fmul(v3, t.w3)));
}

__device__ __forceinline__ int clampi(int v, int n) { return v < 0 ? 0 : (v > n - 1 ? n - 1 : v); }

// ---- rotation formats, rotation_format.h:38-82 (Eigen AngleAxis / Quaternion::toRotationMatrix) ----
__device__ __forceinline__ float tsqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ double tsqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float tsin(float x) { return sinf(x); }
__device__ __forceinline__ double tsin(double x) { return sin(x); }
__device__ __forceinline__ float tcos(float x) { return cosf(x); }
__device__ __forceinline__ double tcos(double x) { return cos(x); }
__device__ __forceinline__ float tabs(float x) { return fabsf(x); }
__device__ __forceinline__ double tabs(double x) { return fabs(x); }

__host__ __device__ __forceinline__ int rotation_step(int format) { return format == 0 ? 9 : (format == 1 ? 4 : 3); }

template <class T>
__device__ void to_rotation_matrix(T* R, const T* data, int format) {
  if (format == DEMON_ROT_MATRIX) {
    for (int i = 0; i < 9; ++i) R[i] = data[i];
  } else if (format == DEMON_ROT_QUATERNION) {
    T w = data[0], x = data[1], y = data[2], z = data[3];
    T n = tsqrt(fadd(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z)), fmul(w, w)));
    w = fdiv(w, n); x = fdiv(x, n); y = fdiv(y, n); z = fdiv(z, n);
    T tx = fmul((T)2, x), ty = fmul((T)2, y), tz = fmul((T)2, z);
    T twx = fmul(tx, w), twy = fmul(ty, w), twz = fmul(tz, w);
    T txx = fmul(tx, x), txy = fmul(ty, x), txz = fmul(tz, x);
    T tyy = fmul(ty, y), tyz = fmul(tz, y), tzz = fmul(tz, z);
    R[0] = fsub((T)1, fadd(tyy, tzz)); R[1] = fsub(txy, twz);             R[2] = fadd(txz, twy);
    R[3] = fadd(txy, twz);             R[4] = fsub((T)1, fadd(txx, tzz)); R[5] = fsub(tyz, twx);
    R[6] = fsub(txz, twy);             R[7] = fadd(tyz, twx);             R[8] = fsub((T)1, fadd(txx, tyy));
  } else {
    T ax = data[0], ay = data[1], az = data[2];
    T angle = tsqrt(fadd(fadd(fmul(ax, ax), fmul(ay, ay)), fmul(az, az)));
    if (angle > (T)1.0e-6) {
      ax = fdiv(ax, angle); ay = fdiv(ay, angle); az = fdiv(az, angle);
      T s = tsin(angle), c = tcos(angle);
      T sx = fmul(s, ax), sy = fmul(s, ay), sz = fmul(s, az);
      T omc = fsub((T)1, c);
      T c1x = fmul(omc, ax), c1y = fmul(omc, ay), c1z = fmul(omc, az);
      T tmp;
      tmp = fmul(c1x, ay); R[1] = fsub(tmp, sz); R[3] = fadd(tmp, sz);
      tmp = fmul(c1x, az); R[2] = fadd(tmp, sy); R[6] = fsub(tmp, sy);
      tmp = fmul(c1y, az); R[5] = fsub(tmp, sx); R[7] = fadd(tmp, sx);
      R[0] = fadd(fmul(c1x, ax), c); R[4] = fadd(fmul(c1y, ay), c); R[8] = fadd(fmul(c1z, az), c);
    } else {
      R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    }
  }
}

// ---- depth_to_flow: per-sample camera, depthtoflow.cc:264-274 --------------------------------
template <class T>
struct D2FCamera {
  T fx, fy, cx, cy, inv_fx, inv_fy;
  T R[9];
  T t[3];
  T inv_w, inv_h;
};

template <class T>
__device__ void d2f_camera(D2FCamera<T>& cam, const T* intrinsics, const T* rotation, const T* translation,
                           int rotation_format, int w, int h) {
  cam.fx = fmul(intrinsics[0], (T)w); cam.fy = fmul(intrinsics[1], (T)h);
  cam.cx = fmul(intrinsics[2], (T)w); cam.cy = fmul(intrinsics[3], (T)h);
  cam.inv_fx = fdiv((T)1, cam.fx); cam.inv_fy = fdiv((T)1, cam.fy);
  to_rotation_matrix(cam.R, rotation, rotation_format);
  cam.t[0] = translation[0]; cam.t[1] = translation[1]; cam.t[2] = translation[2];
  cam.inv_w = (T)(1.0 / w); cam.inv_h = (T)(1.0 / h);   // depthtoflow.cc:261-262: double, then cast
}

// depthtoflow.cc:283-303 + compute_flow depthtoflow.cc:158-185
template <class T>
__device__ __forceinline__ void d2f_pixel(T& fvx, T& fvy, T d, int x, int y, const D2FCamera<T>& cam,
                                          bool inverse_depth, bool normalize_flow) {
  if (inverse_depth) d = fdiv((T)1, d);
  if (d > 0 && isfinite(d)) {
    T p1x = fadd((T)x, (T)0.5), p1y = fadd((T)y, (T)0.5);
    T t2x = fmul(fsub(p1x, cam.cx), cam.inv_fx), t2y = fmul(fsub(p1y, cam.cy), cam.inv_fy);
    T X0 = fmul(d, t2x), X1 = fmul(d, t2y), X2 = d;
    const T* R = cam.R;
    T p2x = fadd(fadd(fadd(fmul(R[0], X0), fmul(R[1], X1)), fmul(R[2], X2)), cam.t[0]);
    T p2y = fadd(fadd(fadd(fmul(R[3], X0), fmul(R[4], X1)), fmul(R[5], X2)), cam.t[1]);
    T p2z = fadd(fadd(fadd(fmul(R[6], X0), fmul(R[7], X1)), fmul(R[8], X2)), cam.t[2]);
    p2x = fadd(fmul(cam.fx, fdiv(p2x, p2z)), cam.cx);
    p2y = fadd(fmul(cam.fy, fdiv(p2y, p2z)), cam.cy);
    fvx = fsub(p2x, p1x); fvy = fsub(p2y, p1y);
    if (normalize_flow) { fvx = fmul(fvx, cam.inv_w); fvy = fmul(fvy, cam.inv_h); }
  } else {
    fvx = (T)NAN; fvy = (T)NAN;
  }
}

// ---- flow_to_depth: per-sample projection matrices, flowtodepth.cc:402-419 --------------------
// Everything from here to the solved point is carried in DOUBLE, for both T = float and T = double.  The
// triangulation is ill conditioned wherever the flow is close to the infinite-depth flow (cond(A) reaches 1e5 on
// the flows the network produces), so each float rounding -- of R, of K*[R|t], of the rows of A -- moves the
// result by cond * 6e-8, i.e. up to 1e-3 relative on those pixels.  The reference's float path has exactly that
// noise (its own realisation of it: Eigen's JacobiSVD); carrying double here puts this kernel at the exact
// solution for the given float inputs, which is the closest any implementation can be to every float realisation.
struct F2DCamera {
  double P1[3][4];
  double P2[3][4];
  double inv_w, inv_h;
};

template <class T>
__device__ void f2d_camera(F2DCamera& cam, const T* intrinsics, const T* rotation, const T* translation,
                           int rotation_format, int w, int h) {
  const double K[9] = {(double)intrinsics[0], 0, (double)intrinsics[2], 0, (double)intrinsics[1], (double)intrinsics[3], 0, 0, 1};
  double rd[9], R[9];
  const int step = rotation_step(rotation_format);
  for (int i = 0; i < step; ++i) rd[i] = (double)rotation[i];
  to_rotation_matrix<double>(R, rd, rotation_format);
  double Rt[3][4];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) { cam.P1[i][j] = K[3 * i + j]; Rt[i][j] = R[3 * i + j]; }
    cam.P1[i][3] = 0; Rt[i][3] = (double)translation[i];
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j)
      cam.P2[i][j] = fadd(fadd(fmul(K[3 * i + 0], Rt[0][j]), fmul(K[3 * i + 1], Rt[1][j])), fmul(K[3 * i + 2], Rt[2][j]));
  cam.inv_w = 1.0 / w; cam.inv_h = 1.0 / h;
}

// Least squares argmin |A X - b| for the 4x3 system of triangulateLinear (flowtodepth.cc:251-281).
// The reference calls Eigen's JacobiSVD in precision T on a heap-allocated dynamic matrix.  Here: Householder
// QR in double -- backward stable, error cond(A) * 1e-16, so the result is the exact least-squares solution
// to float output precision.
// EXACT rank deficiency shows up as a zero pivot -> non-finite X -> output 0, the same value the reference
// produces through its minimum-norm solution (X.z = 0 fails `X.z() > 0`, flowtodepth.cc:464).
// Deviation, stated plainly: for NUMERICALLY rank-deficient pixels (the flow within ~1e-7 relative of the
// infinite-depth flow, cond(A) above ~1e7) the reference's float JacobiSVD drops the small singular value by Eigen's
// rank rule and returns the minimum-norm X, i.e. a tiny inverse depth or 0; the QR below has no rank threshold and
// returns the exact least-squares solution of the float inputs, a large |X.z| of either sign (depth 0 or a finite
// noisy value).  Both are "depth unknown" answers; the reference's own tests (test_FlowToDepth2.py, 1e-4) do not
// exercise such pixels and pass.
__device__ __forceinline__ void lsq_4x3_qr(double X[3], double A[4][3], double b[4]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double norm2 = 0;
#pragma unroll
    for (int i = k; i < 4; ++i) norm2 += A[i][k] * A[i][k];
    double norm = sqrt(norm2);
    double alpha = A[k][k] > 0 ? -norm : norm;
    double v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = (i < k) ? 0.0 : A[i][k];
    v[k] -= alpha;
    double vnorm2 = 0;
#pragma unroll
    for (int i = k; i < 4; ++i) vnorm2 += v[i] * v[i];
    double beta = vnorm2 > 0 ? 2.0 / vnorm2 : 0.0;
#pragma unroll
    for (int j = k; j < 3; ++j) {
      double s = 0;
#pragma unroll
      for (int i = k; i < 4; ++i) s += v[i] * A[i][j];
      s *= beta;
#pragma unroll
      for (int i = k; i < 4; ++i) A[i][j] -= s * v[i];
    }
    double s = 0;
#pragma unroll
    for (int i = k; i < 4; ++i) s += v[i] * b[i];
    s *= beta;
#pragma unroll
    for (int i = k; i < 4; ++i) b[i] -= s * v[i];
  }
  X[2] = b[2] / A[2][2];
  X[1] = (b[1] - A[1][2] * X[2]) / A[1][1];
  X[0] = (b[0] - A[0][1] * X[1] - A[0][2] * X[2]) / A[0][0];
}

// flowtodepth.cc:430-474 for one pixel: rows of A and b as in triangulateLinear (flowtodepth.cc:261-273)
template <class T>
__device__ __forceinline__ T f2d_pixel(T fx_, T fy_, int x, int y, const F2DCamera& cam,
                                       bool inverse_depth, bool normalized_flow) {
  const double x1x = (x + 0.5) * cam.inv_w, x1y = (y + 0.5) * cam.inv_h;
  double fx = (double)fx_, fy = (double)fy_;
  if (!normalized_flow) { fx *= cam.inv_w; fy *= cam.inv_h; }
  const double x2x = x1x + fx, x2y = x1y + fy;
  double A[4][3], b[4];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    A[0][j] = x1y * cam.P1[2][j] - cam.P1[1][j];
    A[1][j] = cam.P1[0][j] - x1x * cam.P1[2][j];
    A[2][j] = x2y * cam.P2[2][j] - cam.P2[1][j];
    A[3][j] = cam.P2[0][j] - x2x * cam.P2[2][j];
  }
  b[0] = cam.P1[1][3] - x1y * cam.P1[2][3];
  b[1] = x1x * cam.P1[2][3] - cam.P1[0][3];
  b[2] = cam.P2[1][3] - x2y * cam.P2[2][3];
  b[3] = x2x * cam.P2[2][3] - cam.P2[0][3];
  double X[3];
  lsq_4x3_qr(X, A, b);
  T Xx = (T)X[0], Xy = (T)X[1], Xz = (T)X[2];
  if (isfinite(Xx) && isfinite(Xy) && isfinite(Xz) && Xz > 0)
    return inverse_depth ? (T)(1.0 / X[2]) : Xz;
  return (T)0;
}

// median of the clamped 3x3 window, median3x3downsample.cc:121-177: five passes that bubble the
// minimum of v[k..8] into v[k] with a strict '>' compare; the result is v[4].  Kept compare for
// compare so that ties and NaNs select the same element as the reference.
template <class T>
__device__ __forceinline__ T median9_reference_order(T v[9]) {
#pragma unroll
  for (int k = 0; k < 5; ++k)
#pragma unroll
    for (int j = k + 1; j < 9; ++j)
      if (v[k] > v[j]) { T tmp = v[k]; v[k] = v[j]; v[j] = tmp; }
  return v[4];
}

// ---- scale_invariant_gradient: one delta's term of one axis, scaleinvariantgradient.cc:174-189 --------------------
// wgt * (vn - v0) / (|v0| + |vn| + eps); vn is the neighbour at +delta, or v0 itself where that lies outside the image.
template <class T>
__device__ __forceinline__ T sig_term(T v0, T vn, T wgt, T eps) {
  return fdiv(fmul(wgt, fsub(vn, v0)), fadd(fadd(tabs(v0), tabs(vn)), eps));
}

// its partial derivatives by the centre and by the neighbour, scaleinvariantgradient.cc:247-268
template <class T>
__device__ __forceinline__ T sig_dcenter(T c, T n, T eps) {
  const T sum_abs = fadd(fadd(tabs(c), tabs(n)), eps);
  const T sign = (c < 0) ? (T)1 : (T)-1;
  return fadd(fdiv((T)-1, sum_abs), fdiv(fmul(sign, fsub(n, c)), fmul(sum_abs, sum_abs)));
}
template <class T>
__device__ __forceinline__ T sig_dneighbour(T c, T n, T eps) {
  const T sum_abs = fadd(fadd(tabs(c), tabs(n)), eps);
  const T sign = (n < 0) ? (T)1 : (T)-1;
  return fadd(fdiv((T)1, sum_abs), fdiv(fmul(sign, fsub(n, c)), fmul(sum_abs, sum_abs)));
}

// ---- depth_to_normals (depthtonormals.cc:147-238) --------------------------------------------------------------------------
// inv_K of K = [[a, s, cx], [0, b, cy], [0, 0, 1]] the way Eigen 3.3 inverts a fixed 3x3 matrix
// (Eigen/src/LU/InverseImpl.h, compute_inverse<.,.,3>: cofactors times 1/det), restricted to the four entries the callers
// read.  depth_to_normals passes s = 0; the multi-view reader's cameras (multivih5datareader.cpp:385,446,1497) keep a skew.
template <class T>
struct D2NCamera { T i00, i02, i11, i12; };

template <class T>
__device__ __forceinline__ D2NCamera<T> eigen_inverse_k(T a, T s, T b, T cx, T cy) {
  // cofactors of column 0: (b*1 - cy*0, 0*cx - 1*s, s*cy - cx*b); det = (c0*a + c1*0) + c2*0; invdet = 1 / det
  const T c0 = fsub(fmul(b, (T)1), fmul(cy, (T)0));
  const T c1 = fsub(fmul((T)0, cx), fmul((T)1, s));
  const T c2 = fsub(fmul(s, cy), fmul(cx, b));
  const T det = fadd(fadd(fmul(c0, a), fmul(c1, (T)0)), fmul(c2, (T)0));
  const T invdet = fdiv((T)1, det);
  D2NCamera<T> c;
  c.i00 = fmul(c0, invdet);                                                     // result.row(0) = cofactors_col0 * invdet
  c.i02 = fmul(c2, invdet);
  c.i11 = fmul(fsub(fmul((T)1, a), fmul((T)0, cx)), invdet);                    // cofactor<1,1> = m22*m00 - m20*m02
  c.i12 = fmul(fsub(fmul(cx, (T)0), fmul(a, cy)), invdet);                      // cofactor<2,1> = m02*m10 - m00*m12
  return c;
}

template <class T>
__device__ __forceinline__ void d2n_point(T p[3], int x, int y, T depth, const D2NCamera<T>& c) {   // compute3dPoint, depthtonormals.cc:95-101
  p[0] = fmul(fadd(fmul(fadd((T)x, (T)0.5), c.i00), c.i02), depth);
  p[1] = fmul(fadd(fmul(fadd((T)y, (T)0.5), c.i11), c.i12), depth);
  p[2] = depth;
}
template <class T>
__device__ __forceinline__ void d2n_cross(T r[3], const T a[3], const T b[3]) {
  r[0] = fsub(fmul(a[1], b[2]), fmul(a[2], b[1]));
  r[1] = fsub(fmul(a[2], b[0]), fmul(a[0], b[2]));
  r[2] = fsub(fmul(a[0], b[1]), fmul(a[1], b[0]));
}
template <class T>
__device__ __forceinline__ void d2n_normalize(T v[3]) {   // MatrixBase::normalize(): z = squaredNorm(); if (z > 0) v /= sqrt(z)
  const T z = fadd(fadd(fmul(v[0], v[0]), fmul(v[1], v[1])), fmul(v[2], v[2]));
  if (z > (T)0) {
    const T n = sqrt(z);   // IEEE sqrt (sqrt.rn for float: no -use_fast_math in this build)
    v[0] = fdiv(v[0], n); v[1] = fdiv(v[1], n); v[2] = fdiv(v[2], n);
  }
}

// The normal of pixel (x, y) of the depth plane dm [H][W] with the sample's normalised intrinsics k[4]; NaN on the border
// and next to a non-positive / non-finite depth.
template <class T>
__device__ __forceinline__ void d2n_pixel(T nrm[3], const T* __restrict__ dm, const T* __restrict__ k, int x, int y, int H, int W,
                                          bool inverse_depth) {
  const T nan = (T)NAN;
  nrm[0] = nan; nrm[1] = nan; nrm[2] = nan;
  if (x == 0 || y == 0 || x == W - 1 || y == H - 1) return;
  const size_t i = (size_t)y * W + x;
  T d = __ldg(dm + i), d_y0 = __ldg(dm + i - W), d_x0 = __ldg(dm + i - 1), d_y1 = __ldg(dm + i + W), d_x1 = __ldg(dm + i + 1);
  if (inverse_depth) { d = fdiv((T)1, d); d_y0 = fdiv((T)1, d_y0); d_x0 = fdiv((T)1, d_x0); d_y1 = fdiv((T)1, d_y1); d_x1 = fdiv((T)1, d_x1); }
  const bool bad = d <= 0 || !isfinite(d) || d_y0 <= 0 || !isfinite(d_y0) || d_x0 <= 0 || !isfinite(d_x0) || d_y1 <= 0 || !isfinite(d_y1) ||
                   d_x1 <= 0 || !isfinite(d_x1);
  if (bad) return;
  const D2NCamera<T> c = eigen_inverse_k(fmul(__ldg(k + 0), (T)W), (T)0, fmul(__ldg(k + 1), (T)H), fmul(__ldg(k + 2), (T)W),
                                         fmul(__ldg(k + 3), (T)H));
  T p[3], p_y0[3], p_x0[3], p_y1[3], p_x1[3];
  d2n_point(p, x, y, d, c);
  d2n_point(p_y0, x, y - 1, d_y0, c);
  d2n_point(p_x0, x - 1, y, d_x0, c);
  d2n_point(p_y1, x, y + 1, d_y1, c);
  d2n_point(p_x1, x + 1, y, d_x1, c);
  T a1[3], b1[3], a0[3], b0[3], v1[3], v0[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) { a1[j] = fsub(p[j], p_x1[j]); b1[j] = fsub(p_y1[j], p[j]); a0[j] = fsub(p[j], p_x0[j]); b0[j] = fsub(p_y0[j], p[j]); }
  d2n_cross(v1, a1, b1);
  d2n_cross(v0, a0, b0);
  d2n_normalize(v1);
  d2n_normalize(v0);
  T v[3] = {fadd(v1[0], v0[0]), fadd(v1[1], v0[1]), fadd(v1[2], v0[2])};
  d2n_normalize(v);
  nrm[0] = v[0]; nrm[1] = v[1]; nrm[2] = v[2];
}

}  // namespace demon
