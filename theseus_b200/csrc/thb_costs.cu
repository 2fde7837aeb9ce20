// Fused cost-function kernels: residual + analytic Jacobians + weighting (linearize), residual-only
// error pass, retract, commit, LM control, and the stand-alone Lie kernels.
//
// One thread = one (cost function k, batch item b); b is the fast index so that the 96-byte SE3 chunks
// of consecutive batch items are read from consecutive addresses.  All Lie math lives in registers
// (thb_lie.cuh).  Kernels are HBM/latency bound (AI ~ 4 flop/B, SURVEY.md 8d): no tensor cores here
// by construction.
//
// Reference semantics: theseus/embodied/measurements/between.py:34-45, theseus/embodied/misc/local_cost_fn.py:40-61,
// theseus/core/cost_weight.py:81-90,125-136, theseus/optimizer/sparse_linearization.py:102-140.
#include "thb_common.cuh"
#include "thb_lie.cuh"

namespace thb {

constexpr int kErrCostsPerThread = 8;

template <typename T> struct GroupDev {
  int kind, weight_kind, K, dim;
  const T* const* x0;
  const T* const* x1;
  const T* const* aux;
  const T* const* w;
  const int32_t* bstride;
  const int64_t* a_off;
  const int32_t* a_stride;
  const int32_t* bp;
  const int32_t* row0;
  const T* const* aux2;
  const T* const* aux3;
  const T* const* aux4;
  const int32_t* bstride2;
  int robust_kind;
  const T* const* log_radius;
  const int32_t* bstride_lr;
  const T* const* x2;
  const T* const* x3;
  const int32_t* bstride3;
  int grid_rows, grid_cols;
};

template <typename T> static GroupDev<T> to_dev(const thb_cost_group* g) {
  GroupDev<T> d;
  d.kind = g->kind;
  d.weight_kind = g->weight_kind;
  d.K = g->K;
  d.dim = g->dim;
  d.x0 = reinterpret_cast<const T* const*>(g->x0);
  d.x1 = reinterpret_cast<const T* const*>(g->x1);
  d.aux = reinterpret_cast<const T* const*>(g->aux);
  d.w = reinterpret_cast<const T* const*>(g->w);
  d.bstride = g->bstride;
  d.a_off = g->a_off;
  d.a_stride = g->a_stride;
  d.bp = g->bp;
  d.row0 = g->row0;
  d.aux2 = reinterpret_cast<const T* const*>(g->aux2);
  d.aux3 = reinterpret_cast<const T* const*>(g->aux3);
  d.aux4 = reinterpret_cast<const T* const*>(g->aux4);
  d.bstride2 = g->bstride2;
  d.robust_kind = g->robust_kind;
  d.log_radius = reinterpret_cast<const T* const*>(g->log_radius);
  d.bstride_lr = g->bstride_lr;
  d.x2 = reinterpret_cast<const T* const*>(g->x2);
  d.x3 = reinterpret_cast<const T* const*>(g->x3);
  d.bstride3 = g->bstride3;
  d.grid_rows = g->grid_rows;
  d.grid_cols = g->grid_cols;
  return d;
}

// Robust wrapper (theseus/core/robust_cost_function.py:87-135; losses robust_loss.py:33-52; _EPS = _LOSS_EPS = 1e-20).
// x = squared norm of the weighted error.  linearize: rescale = sqrt(rho'(x) + eps) applied to J and e;
// evaluate: the error metric sees rho(x) (+ dim*eps) instead of x.
template <typename T> __device__ __forceinline__ T t_exp(T x);
template <> __device__ __forceinline__ float t_exp<float>(float x) { return expf(x); }
template <> __device__ __forceinline__ double t_exp<double>(double x) { return exp(x); }
template <typename T> __device__ __forceinline__ T robust_radius(const GroupDev<T>& g, int k, int64_t b) {
  return t_exp((g.log_radius[k] + (int64_t)g.bstride_lr[k] * b)[0]);
}
template <typename T> __device__ __forceinline__ T robust_rescale(const GroupDev<T>& g, int k, int64_t b, T x) {
  const T radius = robust_radius(g, k, b);
  T lin;
  if (g.robust_kind == THB_ROBUST_WELSCH) lin = t_exp(-x / (radius + T(1e-20)));
  else lin = t_sqrt(radius / (x > radius ? x : radius) + T(1e-20));
  return t_sqrt(lin + T(1e-20));
}
template <typename T> __device__ __forceinline__ T robust_value(const GroupDev<T>& g, int k, int64_t b, T x, int dim) {
  const T radius = robust_radius(g, k, b);
  T val;
  if (g.robust_kind == THB_ROBUST_WELSCH) val = radius - radius * t_exp(-x / (radius + T(1e-20)));
  else val = (x > radius) ? (T(2) * t_sqrt(radius * (x > radius ? x : radius) + T(1e-20)) - radius) : x;
  // the reference spreads rho over `dim` entries sqrt(rho/dim + eps); their squares sum to rho + dim*eps
  return val + T(dim) * T(1e-20);
}

template <typename T, int N> __device__ __forceinline__ void load_n(const T* p, T* r) {
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = p[i];
}
// 12 scalars of an SE3 element; 16-byte vector loads when aligned (always true for [B,3,4] tensors)
__device__ __forceinline__ void load_se3(const double* p, double* r) {
  const double2* q = reinterpret_cast<const double2*>(p);
#pragma unroll
  for (int i = 0; i < 6; i++) {
    double2 v = q[i];
    r[2 * i] = v.x;
    r[2 * i + 1] = v.y;
  }
}
__device__ __forceinline__ void load_se3(const float* p, float* r) {
  const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int i = 0; i < 3; i++) {
    float4 v = q[i];
    r[4 * i] = v.x;
    r[4 * i + 1] = v.y;
    r[4 * i + 2] = v.z;
    r[4 * i + 3] = v.w;
  }
}

// weights: returns true if all weights of this (k,b) are exactly zero (masked cost function,
// theseus/core/cost_function.py:37-55,107-122)
template <typename T, int DIM> __device__ __forceinline__ bool load_weight(const GroupDev<T>& g, int k, int64_t b, T* w) {
  const T* wp = g.w[k] + (int64_t)g.bstride[k * 4 + 3] * b;
  bool all_zero = true;
  if (g.weight_kind == THB_WEIGHT_SCALE) {
    const T s = wp[0];
#pragma unroll
    for (int r = 0; r < DIM; r++) w[r] = s;
    all_zero = (s == T(0));
  } else {
#pragma unroll
    for (int r = 0; r < DIM; r++) {
      w[r] = wp[r];
      all_zero = all_zero && (w[r] == T(0));
    }
  }
  return all_zero;
}

// ------------------------------------------------------------------------------------------------
// residual (+ Jacobians) of one SE3 cost function.  J0/J1 row-major 6x6, already weighted; e weighted.
template <typename T, bool WITH_J, bool BETWEEN>
__device__ __forceinline__ void se3_cost(const GroupDev<T>& g, int k, int64_t b, const T* w, T* e, T* J0, T* J1) {
  T X0[12], Z[12], D[12], E[12];
  load_se3(g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b, X0);
  load_se3(g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b, Z);
  if (BETWEEN) {
    T X1[12];
    load_se3(g.x1[k] + (int64_t)g.bstride[k * 4 + 1] * b, X1);
    se3_between(X0, X1, D);  // D = X0^-1 X1
    se3_between(Z, D, E);    // E = Z^-1 D
  } else {
    se3_between(Z, X0, E);   // E = T^-1 X
  }
  T Jl[36];
  se3_log_jlog<T, WITH_J>(E, e, Jl);
#pragma unroll
  for (int r = 0; r < 6; r++) e[r] *= w[r];
  if (WITH_J) {
    if (BETWEEN) {
      // J0 = -dlog @ Ad(D^-1)  (between.py:43); J1 = dlog
      T Di[12], Ad[36];
      se3_inverse(D, Di);
      se3_adjoint(Di, Ad);
#pragma unroll
      for (int r = 0; r < 6; r++) {
#pragma unroll
        for (int c = 0; c < 6; c++) {
          T s = T(0);
#pragma unroll
          for (int q = 0; q < 6; q++) s += Jl[r * 6 + q] * Ad[q * 6 + c];
          J0[r * 6 + c] = (-s) * w[r];
        }
      }
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) J1[r * 6 + c] = Jl[r * 6 + c] * w[r];
    } else {
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) J0[r * 6 + c] = Jl[r * 6 + c] * w[r];
    }
  }
}

template <typename T, bool WITH_J, bool BETWEEN>
__device__ __forceinline__ void so3_cost(const GroupDev<T>& g, int k, int64_t b, const T* w, T* e, T* J0, T* J1) {
  T X0[9], Z[9], D[9], E[9];
  load_n<T, 9>(g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b, X0);
  load_n<T, 9>(g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b, Z);
  if (BETWEEN) {
    T X1[9];
    load_n<T, 9>(g.x1[k] + (int64_t)g.bstride[k * 4 + 1] * b, X1);
    so3_between(X0, X1, D);
    so3_between(Z, D, E);
  } else {
    so3_between(Z, X0, E);
  }
  So3LogAux<T> a = so3_log<T, 3>(E, e);
  T Jl[9], bw[3];
  if (WITH_J) so3_jlog<T, 3>(e, a, Jl, bw);
  if (WITH_J) {
    if (BETWEEN) {
      // Ad(D^-1) = D^T
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
          T s = Jl[r * 3 + 0] * D[c * 3 + 0] + Jl[r * 3 + 1] * D[c * 3 + 1] + Jl[r * 3 + 2] * D[c * 3 + 2];
          J0[r * 3 + c] = (-s) * w[r];
          J1[r * 3 + c] = Jl[r * 3 + c] * w[r];
        }
    } else {
#pragma unroll
      for (int i = 0; i < 9; i++) J0[i] = Jl[i] * w[i / 3];
    }
  }
#pragma unroll
  for (int r = 0; r < 3; r++) e[r] *= w[r];
}

template <typename T, bool WITH_J, bool BETWEEN>
__device__ __forceinline__ void se2_cost(const GroupDev<T>& g, int k, int64_t b, const T* w, T* e, T* J0, T* J1) {
  T X0[4], Z[4], D[4], E[4];
  load_n<T, 4>(g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b, X0);
  load_n<T, 4>(g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b, Z);
  if (BETWEEN) {
    T X1[4];
    load_n<T, 4>(g.x1[k] + (int64_t)g.bstride[k * 4 + 1] * b, X1);
    se2_between(X0, X1, D);
    se2_between(Z, D, E);
  } else {
    se2_between(Z, X0, E);
  }
  T Jl[9];
  se2_log_jlog<T, WITH_J>(E, e, Jl);
#pragma unroll
  for (int r = 0; r < 3; r++) e[r] *= w[r];
  if (WITH_J) {
    if (BETWEEN) {
      T Di[4], Ad[9];
      se2_inverse(D, Di);
      se2_adjoint(Di, Ad);
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const T s = Jl[r * 3 + 0] * Ad[0 * 3 + c] + Jl[r * 3 + 1] * Ad[1 * 3 + c] + Jl[r * 3 + 2] * Ad[2 * 3 + c];
          J0[r * 3 + c] = (-s) * w[r];
          J1[r * 3 + c] = Jl[r * 3 + c] * w[r];
        }
    } else {
#pragma unroll
      for (int i = 0; i < 9; i++) J0[i] = Jl[i] * w[i / 3];
    }
  }
}

// Reprojection (theseus/embodied/measurements/reprojection.py:54-94): q = R p + t, proj = -q_xy/q_z,
// e = proj * f (1 + n (k1 + n k2)) - z with n = |proj|^2.  Jacobians by the quotient rule on
// [R, -R hat(p) | R] (torchlie se3_impl.py:764-777), exactly as the reference composes them.
template <typename T, bool WITH_J>
__device__ __forceinline__ void reprojection_cost(const GroupDev<T>& g, int k, int64_t b, const T* w, T* e, T* Jc, T* Jp) {
  T X[12], p[3];
  load_se3(g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b, X);
  load_n<T, 3>(g.x1[k] + (int64_t)g.bstride[k * 4 + 1] * b, p);
  const T f = (g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b)[0];
  const T* z = g.aux2[k] + (int64_t)g.bstride2[k * 3 + 0] * b;
  const T k1 = (g.aux3[k] + (int64_t)g.bstride2[k * 3 + 1] * b)[0];
  const T k2 = (g.aux4[k] + (int64_t)g.bstride2[k * 3 + 2] * b)[0];
  T q[3];
#pragma unroll
  for (int i = 0; i < 3; i++) q[i] = X[i * 4 + 3] + (X[i * 4 + 0] * p[0] + X[i * 4 + 1] * p[1] + X[i * 4 + 2] * p[2]);
  const T pr0 = -q[0] / q[2], pr1 = -q[1] / q[2];
  const T n = pr0 * pr0 + pr1 * pr1;
  const T pf = f * (T(1) + n * (k1 + n * k2));
  e[0] = (pr0 * pf - z[0]) * w[0];
  e[1] = (pr1 * pf - z[1]) * w[1];
  if (WITH_J) {
    const T dpf = f * (k1 + T(2) * n * k2);
    // J (3 x 9) = [R | -R hat(p) | R]
    T J[3][9];
#pragma unroll
    for (int i = 0; i < 3; i++) {
      const T r0 = X[i * 4 + 0], r1 = X[i * 4 + 1], r2 = X[i * 4 + 2];
      J[i][0] = r0; J[i][1] = r1; J[i][2] = r2;
      // -(R hat(p)): hat(p) = [[0,-p2,p1],[p2,0,-p0],[-p1,p0,0]]
      J[i][3] = -(r1 * p[2] - r2 * p[1]);
      J[i][4] = -(-r0 * p[2] + r2 * p[0]);
      J[i][5] = -(r0 * p[1] - r1 * p[0]);
      J[i][6] = r0; J[i][7] = r1; J[i][8] = r2;
    }
#pragma unroll
    for (int c = 0; c < 9; c++) {
      const T jz = J[2][c] / q[2];
      const T pj0 = (q[0] * jz - J[0][c]) / q[2];   // (N D'/D - N') / D
      const T pj1 = (q[1] * jz - J[1][c]) / q[2];
      const T nj = T(2) * (pr0 * pj0 + pr1 * pj1);
      const T o0 = (pj0 * pf + (T(2) * pr0 * (pr0 * pj0 + pr1 * pj1)) * dpf) * w[0];
      const T o1 = (pj1 * pf + (T(2) * pr1 * (pr0 * pj0 + pr1 * pj1)) * dpf) * w[1];
      (void)nj;
      if (c < 6) { Jc[0 * 6 + c] = o0; Jc[1 * 6 + c] = o1; }
      else { Jp[0 * 3 + (c - 6)] = o0; Jp[1 * 3 + (c - 6)] = o1; }
    }
  }
}

// Difference on Vector/Point: e = (x - target) * w ; J = I * w   (geometry/vector.py local/jacobians)
// true if every weight of this (k, b) is zero: the cost function is masked like the other kinds (load_weight), its x / target not read
template <typename T> __device__ __forceinline__ bool vector_masked(const GroupDev<T>& g, const T* wp) {
  if (g.weight_kind == THB_WEIGHT_SCALE) return wp[0] == T(0);
  for (int r = 0; r < g.dim; r++)
    if (wp[r] != T(0)) return false;
  return true;
}

// ------------------------------------------------------------------------------------------------
// Motion-planning cost functions: Collision2D (embodied/collision/collision.py:44-73 + signed_distance_field.py:163-241),
// DoubleIntegrator / GPMotionModel (motionmodel/double_integrator.py:45-80) with GPCostWeight (:131-170), HingeCost and
// Nonholonomic (motionmodel/misc.py:62-84, 126-178).  Every optimisation variable of one of these cost functions has the same dof D;
// a cost function's row block is DIM x (NVARS * D).  The unweighted Jacobian is written straight into the warp's staging area (the
// layout of A_val) and the weight is applied there.
template <typename T> __device__ __forceinline__ T t_floor(T x);
template <> __device__ __forceinline__ float t_floor<float>(float x) { return floorf(x); }
template <> __device__ __forceinline__ double t_floor<double>(double x) { return floor(x); }

// Planar pushing (tactile pose estimation): QuasiStaticPushingPlanar (motionmodel/quasi_static_pushing_planar.py:19-297) over four SE2
// poses and EffectorObjectContactPlanar (collision/eff_obj_contact.py:21-126) over two, both with D = 3.
template <int KIND, int D> struct Mp {
  static constexpr bool COLL = KIND == THB_COST_COLLISION2D_POINT2 || KIND == THB_COST_COLLISION2D_SE2;
  static constexpr bool DI = KIND == THB_COST_DOUBLE_INTEGRATOR_VECTOR || KIND == THB_COST_DOUBLE_INTEGRATOR_SE2;
  static constexpr bool NH = KIND == THB_COST_NONHOLONOMIC_SE2 || KIND == THB_COST_NONHOLONOMIC_VECTOR;
  static constexpr bool QSP = KIND == THB_COST_QUASI_STATIC_PUSHING_PLANAR;
  static constexpr bool EOC = KIND == THB_COST_EFF_OBJ_CONTACT_PLANAR;
  static constexpr int DIM = (COLL || NH || EOC) ? 1 : (DI ? 2 * D : D);
  static constexpr int NVARS = (DI || QSP) ? 4 : ((NH || EOC) ? 2 : 1);
  static constexpr int BPW = NVARS > 2 ? NVARS : 2;   // row length of the group's bp table
  static constexpr int COLS = NVARS * D;
  static constexpr int NV = DIM * COLS;
};

template <typename T> __device__ __forceinline__ const T* mp_var(const GroupDev<T>& g, int v, int k, int64_t b) {
  if (v == 0) return g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b;
  if (v == 1) return g.x1[k] + (int64_t)g.bstride[k * 4 + 1] * b;
  if (v == 2) return g.x2[k] + (int64_t)g.bstride3[k * 2 + 0] * b;
  return g.x3[k] + (int64_t)g.bstride3[k * 2 + 1] * b;
}
template <typename T> __device__ __forceinline__ const T* mp_aux(const GroupDev<T>& g, int q, int k, int64_t b) {
  if (q == 0) return g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b;
  const T* const* p = (q == 1) ? g.aux2 : ((q == 2) ? g.aux3 : g.aux4);
  return p[k] + (int64_t)g.bstride2[k * 3 + (q - 1)] * b;
}

// Signed distance of the point (px, py) in the SDF grid data [R, C] whose cell (r, c) lies at (ox, oy) + (c, r) * cell, by bilinear
// interpolation (signed_distance_field.py:163-241), and its gradient (jx, jy); 0 and a zero gradient outside the grid.
template <typename T>
__device__ __forceinline__ void sdf_lookup(const T* data, int R, int C, T ox, T oy, T cell, T px, T py, T& dist, T& jx, T& jy) {
  const bool oob = (px < ox) || (px > ox + (T(C) - T(1)) * cell) || (py < oy) || (py > oy + (T(R) - T(1)) * cell);
  dist = T(0), jx = T(0), jy = T(0);
  if (!oob) {
    const T col = (px - ox) / cell, row = (py - oy) / cell;
    const T lr = t_floor(row), lc = t_floor(col);
    const T hr = lr + T(1), hc = lc + T(1);
    auto clampi = [](T v, int hi) { return !(v >= T(0)) ? 0 : (v > T(hi) ? hi : (int)v); };
    const int lri = clampi(lr, R - 1), lci = clampi(lc, C - 1), hri = clampi(hr, R - 1), hci = clampi(hc, C - 1);
    const T g00 = data[(int64_t)lri * C + lci], g10 = data[(int64_t)hri * C + lci];
    const T g01 = data[(int64_t)lri * C + hci], g11 = data[(int64_t)hri * C + hci];
    const T hrd = hr - row, hcd = hc - col, lrd = row - lr, lcd = col - lc;
    dist = hrd * hcd * g00 + lrd * hcd * g10 + hrd * lcd * g01 + lrd * lcd * g11;
    jx = (hrd * (g01 - g00) + lrd * (g11 - g10)) / cell;
    jy = (hcd * (g10 - g00) + lcd * (g11 - g01)) / cell;
  }
}

// Unweighted error e[DIM] and (WITH_J) Jacobian rows S[r * stride + bp[v] + c] of one cost function.
template <typename T, int KIND, int D, bool WITH_J>
__device__ __forceinline__ void mp_cost(const GroupDev<T>& g, int k, int64_t b, T* e, T* S, int stride, const int* bp) {
  using M = Mp<KIND, D>;
  if constexpr (M::COLL) {
    // e = max(eps - sdf, 0), J = -d sdf where sdf <= eps
    const T* x = mp_var(g, 0, k, b);
    const T* org = mp_aux(g, 0, k, b);
    const T cell = mp_aux(g, 2, k, b)[0];
    const T eps = mp_aux(g, 3, k, b)[0];
    T dist, jx, jy;
    sdf_lookup(mp_aux(g, 1, k, b), g.grid_rows, g.grid_cols, org[0], org[1], cell, x[0], x[1], dist, jx, jy);
    const T err = eps - dist;
    e[0] = err < T(0) ? T(0) : err;
    if (WITH_J) {
      if (dist > eps) jx = jy = T(0);
      if (KIND == THB_COST_COLLISION2D_POINT2) {
        S[bp[0] + 0] = -jx;
        S[bp[0] + 1] = -jy;
      } else {   // d xy / d tangent of SE2 = [R | 0] (se2.py:143-150)
        const T c = x[2], s = x[3];
        S[bp[0] + 0] = -(jx * c + jy * s);
        S[bp[0] + 1] = -(jx * -s + jy * c);
        S[bp[0] + 2] = T(0);
      }
    }
  } else if constexpr (M::DI) {
    // e = [local(pose1, pose2) - dt vel1, vel2 - vel1]
    const T* v1 = mp_var(g, 1, k, b);
    const T* v2 = mp_var(g, 3, k, b);
    const T dt = mp_aux(g, 0, k, b)[0];
    T pd[D], J1[D * D], J2[D * D];
    if constexpr (KIND == THB_COST_DOUBLE_INTEGRATOR_SE2) {
      T X1[4], X2[4], Dm[4], Jl[9];
      load_n<T, 4>(mp_var(g, 0, k, b), X1);
      load_n<T, 4>(mp_var(g, 2, k, b), X2);
      se2_between(X1, X2, Dm);
      se2_log_jlog<T, WITH_J>(Dm, pd, Jl);
      if (WITH_J) {   // local's Jacobians: -dlog Ad(D^-1), dlog (as Between with an identity measurement)
        T Di[4], Ad[9];
        se2_inverse(Dm, Di);
        se2_adjoint(Di, Ad);
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
          for (int c = 0; c < 3; c++) {
            J1[r * 3 + c] = -(Jl[r * 3 + 0] * Ad[0 * 3 + c] + Jl[r * 3 + 1] * Ad[1 * 3 + c] + Jl[r * 3 + 2] * Ad[2 * 3 + c]);
            J2[r * 3 + c] = Jl[r * 3 + c];
          }
      }
    } else {
      const T* p1 = mp_var(g, 0, k, b);
      const T* p2 = mp_var(g, 2, k, b);
#pragma unroll
      for (int i = 0; i < D; i++) pd[i] = p2[i] - p1[i];
#pragma unroll
      for (int i = 0; i < D * D; i++) {
        J1[i] = (i / D == i % D) ? T(-1) : T(0);
        J2[i] = (i / D == i % D) ? T(1) : T(0);
      }
    }
#pragma unroll
    for (int i = 0; i < D; i++) {
      e[i] = pd[i] - dt * v1[i];
      e[D + i] = v2[i] - v1[i];
    }
    if (WITH_J) {
#pragma unroll
      for (int r = 0; r < D; r++)
#pragma unroll
        for (int c = 0; c < D; c++) {
          const bool diag = r == c;
          T* top = S + r * stride;
          T* bot = S + (D + r) * stride;
          top[bp[0] + c] = J1[r * D + c];
          top[bp[1] + c] = diag ? -dt : T(0);
          top[bp[2] + c] = J2[r * D + c];
          top[bp[3] + c] = T(0);
          bot[bp[0] + c] = T(0);
          bot[bp[1] + c] = diag ? T(-1) : T(0);
          bot[bp[2] + c] = T(0);
          bot[bp[3] + c] = diag ? T(1) : T(0);
        }
    }
  } else if constexpr (M::QSP) {
    // p = R2^T (s2 - t2) (contact point in the frame of obj2), v = R2^T (t2 - t1), vp = R2^T (s2 - s1), w = theta(obj1^-1 obj2);
    // e = D [v, w] - [vp, 0] with D = [[1, 0, -py], [0, 1, px], [-py, px, -c^2]]
    const T* o1 = mp_var(g, 0, k, b);
    const T* o2 = mp_var(g, 1, k, b);
    const T* e1 = mp_var(g, 2, k, b);
    const T* e2 = mp_var(g, 3, k, b);
    const T c2 = mp_aux(g, 0, k, b)[0];
    const T c = o2[2], s = o2[3];
    auto unrot_x = [&](T x, T y) { return c * x + s * y; };
    auto unrot_y = [&](T x, T y) { return -s * x + c * y; };
    const T px = unrot_x(e2[0] - o2[0], e2[1] - o2[1]), py = unrot_y(e2[0] - o2[0], e2[1] - o2[1]);
    const T vx = unrot_x(o2[0] - o1[0], o2[1] - o1[1]), vy = unrot_y(o2[0] - o1[0], o2[1] - o1[1]);
    const T vpx = unrot_x(e2[0] - e1[0], e2[1] - e1[1]), vpy = unrot_y(e2[0] - e1[0], e2[1] - e1[1]);
    const T w = t_atan2(o1[2] * s - o1[3] * c, o1[2] * c + o1[3] * s);
    e[0] = vx - py * w - vpx;
    e[1] = vy + px * w - vpy;
    e[2] = -py * vx + px * vy - c2 * w;
    if (WITH_J) {
      // column j of variable v from the derivatives of (p, v, vp, w) along that tangent direction
      auto col = [&](int v, int j, T dpx, T dpy, T dvx, T dvy, T dvpx, T dvpy, T dw) {
        S[0 * stride + bp[v] + j] = dvx - w * dpy - py * dw - dvpx;
        S[1 * stride + bp[v] + j] = dvy + w * dpx + px * dw - dvpy;
        S[2 * stride + bp[v] + j] = -vx * dpy - py * dvx + vy * dpx + px * dvy - c2 * dw;
      };
      // R2^T R_x of a pose x: the rotation by x's angle minus obj2's, with columns (rc, rs) and (-rs, rc)
      auto rel = [&](const T* x, T& rc, T& rs) { rc = c * x[2] + s * x[3]; rs = c * x[3] - s * x[2]; };
      const T z = T(0);
      T rc, rs;
      rel(o1, rc, rs);   // obj1: dv/du = -R2^T R1, dw/dtheta = -1
      col(0, 0, z, z, -rc, -rs, z, z, z);
      col(0, 1, z, z, rs, -rc, z, z, z);
      col(0, 2, z, z, z, z, z, z, T(-1));
      // obj2: dp = [-I | (py, -px)], dv = [I | (vy, -vx)], dvp = [0 | (vpy, -vpx)], dw/dtheta = 1
      col(1, 0, T(-1), z, T(1), z, z, z, z);
      col(1, 1, z, T(-1), z, T(1), z, z, z);
      col(1, 2, py, -px, vy, -vx, vpy, -vpx, T(1));
      rel(e1, rc, rs);   // eff1: dvp/du = -R2^T Re1
      col(2, 0, z, z, z, z, -rc, -rs, z);
      col(2, 1, z, z, z, z, rs, -rc, z);
      col(2, 2, z, z, z, z, z, z, z);
      rel(e2, rc, rs);   // eff2: dp/du = dvp/du = R2^T Re2
      col(3, 0, rc, rs, z, z, rc, rs, z);
      col(3, 1, -rs, rc, z, z, -rs, rc, z);
      col(3, 2, z, z, z, z, z, z, z);
    }
  } else if constexpr (M::EOC) {
    // p = R_obj^T (t_eff - t_obj), e = |sdf(p) - r|; J = s d sdf/dp dp/d(obj, eff) with s = -1 where sdf < r (eff_obj_contact.py:101-103)
    const T* o = mp_var(g, 0, k, b);
    const T* ef = mp_var(g, 1, k, b);
    const T* org = mp_aux(g, 0, k, b);
    const T cell = mp_aux(g, 2, k, b)[0];
    const T r = mp_aux(g, 3, k, b)[0];
    const T c = o[2], s = o[3];
    const T dx = ef[0] - o[0], dy = ef[1] - o[1];
    const T px = c * dx + s * dy, py = -s * dx + c * dy;
    T dist, jx, jy;
    sdf_lookup(mp_aux(g, 1, k, b), g.grid_rows, g.grid_cols, org[0], org[1], cell, px, py, dist, jx, jy);
    const T diff = dist - r;
    e[0] = diff < T(0) ? -diff : diff;
    if (WITH_J) {
      const T sg = dist < r ? T(-1) : T(1);
      const T gx = sg * jx, gy = sg * jy;
      // dp/d obj = [[-1, 0, py], [0, -1, -px]];  dp/d eff = [R_obj^T R_eff | 0]
      S[bp[0] + 0] = -gx;
      S[bp[0] + 1] = -gy;
      S[bp[0] + 2] = gx * py - gy * px;
      const T rc = c * ef[2] + s * ef[3], rs = c * ef[3] - s * ef[2];
      S[bp[1] + 0] = gx * rc + gy * rs;
      S[bp[1] + 1] = -gx * rs + gy * rc;
      S[bp[1] + 2] = T(0);
    }
  } else if constexpr (KIND == THB_COST_HINGE) {
    // limits tightened by the threshold; above the upper limit wins (misc.py:62-84)
    const T* x = mp_var(g, 0, k, b);
    const T* dl = mp_aux(g, 0, k, b);
    const T* ul = mp_aux(g, 1, k, b);
    const T* th = mp_aux(g, 2, k, b);
#pragma unroll
    for (int i = 0; i < D; i++) {
      const T down = dl[i] + th[i], up = ul[i] - th[i], v = x[i];
      const bool below = v < down, above = v > up;
      e[i] = above ? (v - up) : (below ? (down - v) : T(0));
      if (WITH_J) {
#pragma unroll
        for (int c = 0; c < D; c++) S[i * stride + bp[0] + c] = (c == i) ? (above ? T(1) : (below ? T(-1) : T(0))) : T(0);
      }
    }
  } else {   // Nonholonomic (misc.py:126-178)
    const T* v = mp_var(g, 1, k, b);
    if constexpr (KIND == THB_COST_NONHOLONOMIC_SE2) {
      e[0] = v[1];
      if (WITH_J) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
          S[bp[0] + c] = T(0);
          S[bp[1] + c] = (c == 1) ? T(1) : T(0);
        }
      }
    } else {
      const T* p = mp_var(g, 0, k, b);
      T s, c;
      t_sincos(p[2], &s, &c);
      e[0] = v[1] * c - v[0] * s;
      if (WITH_J) {
        S[bp[0] + 0] = T(0);
        S[bp[0] + 1] = T(0);
        S[bp[0] + 2] = -(v[1] * s + v[0] * c);
        S[bp[1] + 0] = -s;
        S[bp[1] + 1] = c;
        S[bp[1] + 2] = T(0);
      }
    }
  }
}

// The cost weight of one (k, b): per-row factors (Scale / Diagonal) or the GP weight's upper factor U = cholesky(W^T)^T of
// W = [[12/dt^3 Q, -6/dt^2 Q], [-6/dt^2 Q, 4/dt Q]], Q = Qc_inv (double_integrator.py:131-152).  The Cholesky reads only the lower
// triangle of W^T, i.e. M(i, j) = W(j, i) for i >= j: for a non-symmetric Q that matrix is not S (x) Q of either triangle, so the
// 2D x 2D factor is formed here in full (at most 6 x 6) rather than as chol(S)^T (x) chol(Q)^T.
template <typename T, int DIM, int D> struct MpWeight {
  bool gp;
  T w[DIM];
  T U[DIM * DIM];   // GP: U(p, q) for q >= p

  __device__ __forceinline__ bool load(const GroupDev<T>& g, int k, int64_t b) {
    gp = g.weight_kind == THB_WEIGHT_GP;
    if constexpr (DIM == 2 * D) {
      if (gp) {
        const T* Q = g.w[k] + (int64_t)g.bstride[k * 4 + 3] * b;
        const T dt = mp_aux(g, 1, k, b)[0];
        const T s00 = T(12) / (dt * dt * dt), s01 = T(-6) / (dt * dt), s11 = T(4) / dt;   // S = [[s00, s01], [s01, s11]]
        auto M = [&](int i, int j) {   // i >= j: W(j, i)
          const int blk = j / D + i / D;
          return (blk == 0 ? s00 : (blk == 1 ? s01 : s11)) * Q[(j % D) * D + (i % D)];
        };
        // U^T U = M column by column: U(j, j) = sqrt(M(j, j) - sum_q U(q, j)^2), U(j, i) = (M(i, j) - sum_q U(q, i) U(q, j)) / U(j, j)
#pragma unroll
        for (int j = 0; j < DIM; j++) {
          T d = M(j, j);
#pragma unroll
          for (int q = 0; q < j; q++) d -= U[q * DIM + j] * U[q * DIM + j];
          const T ujj = t_sqrt(d);
          const T rjj = T(1) / ujj;   // one division per column, the row scaled by it (as LAPACK's potf2 does)
          U[j * DIM + j] = ujj;
#pragma unroll
          for (int i = j + 1; i < DIM; i++) {
            T t = M(i, j);
#pragma unroll
            for (int q = 0; q < j; q++) t -= U[q * DIM + i] * U[q * DIM + j];
            U[j * DIM + i] = t * rjj;
          }
        }
        return false;
      }
    }
    return load_weight<T, DIM>(g, k, b, w);   // (mp_dof admits a GP weight only for the DoubleIntegrator kinds, DIM = 2 D)
  }
  // columns 0..ncols-1 of the DIM x ld row block v (ncols = 1, ld = 1: a vector) <- W v
  __device__ __forceinline__ void apply(T* v, int ld, int ncols) const {
    if (!gp) {
      for (int j = 0; j < ncols; j++)
#pragma unroll
        for (int r = 0; r < DIM; r++) v[r * ld + j] *= w[r];
      return;
    }
    if constexpr (DIM == 2 * D) {
      for (int j = 0; j < ncols; j++) {
        // row p reads rows q >= p only: overwriting in increasing p is safe
#pragma unroll
        for (int p = 0; p < DIM; p++) {
          T acc = T(0);
#pragma unroll
          for (int q = p; q < DIM; q++) acc += U[p * DIM + q] * v[q * ld + j];
          v[p * ld + j] = acc;
        }
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
// One policy per cost family for linearize_kernel / error_kernel.  A policy gives
//   DIM      rows of a cost function (VectorCost: 0, its g.dim rows are known at run time only)
//   NV       values of its row block staged per thread for the warp-cooperative store (0: each thread stores its own rows)
//   ROBUST   whether the group's robust loss applies (RobustCostFunction routes the Lie and Reprojection kinds only)
//   load(g, k, b)                the weights of (k, b); true if they are all zero (masked cost function: nothing else is read)
//   linearize(g, k, b, e, row)   the weighted error e and weighted Jacobian rows, written to row (row-major, A_val layout).  ROBUST
//                                policies keep their Jacobians in J instead, so that the robust rescale happens in registers, and
//                                write them with store(g, k, row)
//   error(g, k, b, acc)          adds the cost function's share of the error metric to acc (after load)
template <int N, typename T> __device__ __forceinline__ T sum_sq(const T* e) {
  T x = T(0);
#pragma unroll
  for (int r = 0; r < N; r++) x += e[r] * e[r];
  return x;
}

template <typename T, int KIND> struct LieCost {
  static constexpr int DIM = (KIND == THB_COST_BETWEEN_SE3 || KIND == THB_COST_LOCAL_SE3) ? 6 : 3;
  static constexpr bool BETWEEN = (KIND == THB_COST_BETWEEN_SE3 || KIND == THB_COST_BETWEEN_SO3 || KIND == THB_COST_BETWEEN_SE2);
  static constexpr bool IS_SE2 = (KIND == THB_COST_BETWEEN_SE2 || KIND == THB_COST_LOCAL_SE2);
  static constexpr int NV = DIM * DIM * (BETWEEN ? 2 : 1), NJ = NV;
  static constexpr bool ROBUST = true;
  T w[DIM], J[NJ];   // J0, then (Between) J1

  __device__ __forceinline__ bool load(const GroupDev<T>& g, int k, int64_t b) { return load_weight<T, DIM>(g, k, b, w); }
  template <bool WITH_J> __device__ __forceinline__ void cost(const GroupDev<T>& g, int k, int64_t b, T* e) {
    if (DIM == 6) se3_cost<T, WITH_J, BETWEEN>(g, k, b, w, e, J, J + DIM * DIM);
    else if (IS_SE2) se2_cost<T, WITH_J, BETWEEN>(g, k, b, w, e, J, J + DIM * DIM);
    else so3_cost<T, WITH_J, BETWEEN>(g, k, b, w, e, J, J + DIM * DIM);
  }
  __device__ __forceinline__ void linearize(const GroupDev<T>& g, int k, int64_t b, T* e, T*) { cost<true>(g, k, b, e); }
  static __device__ __forceinline__ T sqnorm(const T* e) { return sum_sq<DIM>(e); }
  __device__ __forceinline__ void store(const GroupDev<T>& g, int k, T* row) const {
    const int stride = g.a_stride[k];
    const int bp0 = g.bp[k * 2 + 0];
#pragma unroll
    for (int r = 0; r < DIM; r++)
#pragma unroll
      for (int c = 0; c < DIM; c++) row[r * stride + bp0 + c] = J[r * DIM + c];
    if (BETWEEN) {   // after J0: J1 wins where bp0 == bp1
      const int bp1 = g.bp[k * 2 + 1];
#pragma unroll
      for (int r = 0; r < DIM; r++)
#pragma unroll
        for (int c = 0; c < DIM; c++) row[r * stride + bp1 + c] = J[DIM * DIM + r * DIM + c];
    }
  }
  __device__ __forceinline__ void error(const GroupDev<T>& g, int k, int64_t b, T& acc) {
    T e[DIM];
    cost<false>(g, k, b, e);
    const T x = sum_sq<DIM>(e);
    acc += (g.robust_kind != THB_ROBUST_NONE) ? robust_value(g, k, b, x, DIM) : x;
  }
};

template <typename T> struct ReprojectionCost {
  static constexpr int DIM = 2, NV = 0, NJ = 18;
  static constexpr bool ROBUST = true;
  T w[2], J[NJ];   // camera block 2 x 6, then point block 2 x 3

  __device__ __forceinline__ bool load(const GroupDev<T>& g, int k, int64_t b) { return load_weight<T, 2>(g, k, b, w); }
  __device__ __forceinline__ void linearize(const GroupDev<T>& g, int k, int64_t b, T* e, T*) {
    reprojection_cost<T, true>(g, k, b, w, e, J, J + 12);
  }
  static __device__ __forceinline__ T sqnorm(const T* e) { return e[0] * e[0] + e[1] * e[1]; }
  __device__ __forceinline__ void store(const GroupDev<T>& g, int k, T* row) const {
    const int stride = g.a_stride[k];
    const int bp0 = g.bp[k * 2 + 0], bp1 = g.bp[k * 2 + 1];
#pragma unroll
    for (int r = 0; r < 2; r++) {
#pragma unroll
      for (int c = 0; c < 6; c++) row[r * stride + bp0 + c] = J[r * 6 + c];
#pragma unroll
      for (int c = 0; c < 3; c++) row[r * stride + bp1 + c] = J[12 + r * 3 + c];
    }
  }
  __device__ __forceinline__ void error(const GroupDev<T>& g, int k, int64_t b, T& acc) {
    T e[2];
    reprojection_cost<T, false>(g, k, b, w, e, nullptr, nullptr);
    const T x = sqnorm(e);
    acc += (g.robust_kind != THB_ROBUST_NONE) ? robust_value(g, k, b, x, 2) : x;
  }
};

// A Vector cost function has one variable: its row block is the g.dim x g.dim diagonal of the weights (stride = g.dim).
template <typename T> struct VectorCost {
  static constexpr int DIM = 0, NV = 0;
  static constexpr bool ROBUST = false;
  const T* wp;

  __device__ __forceinline__ bool load(const GroupDev<T>& g, int k, int64_t b) {
    wp = g.w[k] + (int64_t)g.bstride[k * 4 + 3] * b;
    return vector_masked(g, wp);
  }
  __device__ __forceinline__ T weight(const GroupDev<T>& g, int r) const { return (g.weight_kind == THB_WEIGHT_SCALE) ? wp[0] : wp[r]; }
  __device__ __forceinline__ void linearize(const GroupDev<T>& g, int k, int64_t, T*, T* row) const {
    const int stride = g.a_stride[k];
    const int bp0 = g.bp[k * 2 + 0];
    for (int r = 0; r < g.dim; r++) {
      const T w = weight(g, r);
      for (int c = 0; c < g.dim; c++) row[r * stride + bp0 + c] = (r == c) ? w : T(0);
    }
  }
  // b = -e, row by row (+0 where masked)
  __device__ __forceinline__ void residual(const GroupDev<T>& g, int k, int64_t b, bool masked, T* brow) const {
    const T* x = g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b;
    const T* tg = g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b;
    for (int r = 0; r < g.dim; r++) brow[r] = masked ? T(0) : -((x[r] - tg[r]) * weight(g, r));
  }
  // each row's e * e straight into acc (not summed per cost function first)
  __device__ __forceinline__ void error(const GroupDev<T>& g, int k, int64_t b, T& acc) const {
    const T* x = g.x0[k] + (int64_t)g.bstride[k * 4 + 0] * b;
    const T* tg = g.aux[k] + (int64_t)g.bstride[k * 4 + 2] * b;
    for (int r = 0; r < g.dim; r++) {
      const T e = (x[r] - tg[r]) * weight(g, r);
      acc += e * e;
    }
  }
};

// The weight is applied after the cost, to e and to the staged rows; no robust loss.
template <typename T, int KIND, int D> struct MpCost {
  using M = Mp<KIND, D>;
  static constexpr int DIM = M::DIM, NV = M::NV;
  static constexpr bool ROBUST = false;
  MpWeight<T, M::DIM, D> W;

  __device__ __forceinline__ bool load(const GroupDev<T>& g, int k, int64_t b) { return W.load(g, k, b); }
  __device__ __forceinline__ void linearize(const GroupDev<T>& g, int k, int64_t b, T* e, T* row) const {
    const int stride = g.a_stride[k];
    int bp[M::NVARS];
#pragma unroll
    for (int v = 0; v < M::NVARS; v++) bp[v] = g.bp[k * M::BPW + v];
    mp_cost<T, KIND, D, true>(g, k, b, e, row, stride, bp);
    W.apply(e, 1, 1);
    W.apply(row, stride, stride);
  }
  __device__ __forceinline__ void error(const GroupDev<T>& g, int k, int64_t b, T& acc) const {
    T e[DIM];
    mp_cost<T, KIND, D, false>(g, k, b, e, nullptr, 0, nullptr);
    W.apply(e, 1, 1);
    acc += sum_sq<DIM>(e);
  }
};

template <typename T, class Cost>
__global__ void __launch_bounds__(128) linearize_kernel(GroupDev<T> g, int64_t B, T* __restrict__ A_val, int64_t nnz,
                                                        T* __restrict__ bvec, int64_t m) {
  constexpr bool STAGED = Cost::NV > 0;
  extern __shared__ double lin_stage_raw[];
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = t < (int64_t)g.K * B;
  if (!STAGED && !valid) return;               // (staged: no early exit, every lane takes part in the warp-cooperative store below)
  const int k = valid ? (int)(t / B) : 0;
  const int64_t b = valid ? t - (int64_t)k * B : 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T* stage = reinterpret_cast<T*>(lin_stage_raw) + (size_t)warp * 32 * (Cost::NV + 1);
  auto row = [&]() { return STAGED ? stage + lane * (Cost::NV + 1) : A_val + b * nnz + g.a_off[k]; };
  Cost c;
  T e[Cost::DIM > 0 ? Cost::DIM : 1];
  const bool masked = c.load(g, k, b);
  if (masked) {
#pragma unroll
    for (int r = 0; r < Cost::DIM; r++) e[r] = T(0);
    const int nv = (Cost::DIM > 0 ? Cost::DIM : g.dim) * g.a_stride[k];
    T* z = row();
    for (int i = 0; i < nv; i++) z[i] = T(0);
  } else {
    c.linearize(g, k, b, e, row());
    if constexpr (Cost::ROBUST) {
      if (g.robust_kind != THB_ROBUST_NONE) {
        const T sc = robust_rescale(g, k, b, Cost::sqnorm(e));
#pragma unroll
        for (int r = 0; r < Cost::DIM; r++) e[r] *= sc;
#pragma unroll
        for (int i = 0; i < Cost::NJ; i++) c.J[i] *= sc;
      }
      c.store(g, k, row());
    }
  }
  if constexpr (STAGED) {
    // A cost function's rows of A_val are ONE contiguous run of DIM * stride values per batch item (stride = its row length), but
    // the items of a warp lie nnz values apart: storing from the computing thread writes 8 bytes to 32 different sectors per
    // instruction.  The warp's 32 runs are staged in shared memory and the whole warp stores each run with consecutive lanes
    // (256-byte segments).
    const int nv = Cost::DIM * g.a_stride[k];   // <= NV: the row block spans the cost function's own variables
    __syncwarp();
    const unsigned long long my_dst = valid ? reinterpret_cast<unsigned long long>(A_val + b * nnz + g.a_off[k]) : 0ull;
    for (int i = 0; i < 32; i++) {
      const unsigned long long d = __shfl_sync(0xffffffffu, my_dst, i);
      const int nvi = __shfl_sync(0xffffffffu, nv, i);
      if (d != 0ull) {
        T* dst = reinterpret_cast<T*>(d);
        const T* src = stage + i * (Cost::NV + 1);
        for (int v = lane; v < nvi; v += 32) dst[v] = src[v];
      }
    }
  }
  if (valid) {
    T* brow = bvec + b * m + g.row0[k];
    if constexpr (Cost::DIM > 0) {
#pragma unroll
      for (int r = 0; r < Cost::DIM; r++) brow[r] = -e[r];
    } else {
      c.residual(g, k, b, masked, brow);
    }
  }
}

// One thread = kErrCostsPerThread cost functions of one batch item; partial[chunk, b] = half their summed squared error.
template <typename T, class Cost>
__global__ void __launch_bounds__(128) error_kernel(GroupDev<T> g, int64_t B, T* __restrict__ partial) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int nchunks = (g.K + kErrCostsPerThread - 1) / kErrCostsPerThread;
  if (t >= (int64_t)nchunks * B) return;
  const int c = (int)(t / B);
  const int64_t b = t - (int64_t)c * B;
  T acc = T(0);
  const int k1 = min(g.K, (c + 1) * kErrCostsPerThread);
  for (int k = c * kErrCostsPerThread; k < k1; k++) {
    Cost cost;
    if (cost.load(g, k, b)) continue;
    cost.error(g, k, b, acc);
  }
  partial[(int64_t)c * B + b] = acc * T(0.5);
}

// Checks the fields the motion-planning kinds read; the pose dof D of the kernel instance (0 = no fused kernel for this group).
static int mp_dof(const thb_cost_group* g) {
  const bool gp = g->weight_kind == THB_WEIGHT_GP;
  if (g->weight_kind != THB_WEIGHT_SCALE && g->weight_kind != THB_WEIGHT_DIAGONAL && !gp) return 0;
  switch (g->kind) {
    case THB_COST_COLLISION2D_POINT2:
    case THB_COST_COLLISION2D_SE2:
      if (gp || g->aux2 == nullptr || g->aux3 == nullptr || g->aux4 == nullptr || g->bstride2 == nullptr || g->grid_rows < 1 || g->grid_cols < 1)
        return 0;
      return g->kind == THB_COST_COLLISION2D_POINT2 ? 2 : 3;
    case THB_COST_DOUBLE_INTEGRATOR_VECTOR:
    case THB_COST_DOUBLE_INTEGRATOR_SE2: {
      if (g->x2 == nullptr || g->x3 == nullptr || g->bstride3 == nullptr || (gp && (g->aux2 == nullptr || g->bstride2 == nullptr))) return 0;
      const int d = g->dim / 2;
      if (g->kind == THB_COST_DOUBLE_INTEGRATOR_SE2) return g->dim == 6 ? 3 : 0;
      return (g->dim % 2 == 0 && d >= 1 && d <= 3) ? d : 0;
    }
    case THB_COST_HINGE:
      if (gp || g->aux2 == nullptr || g->aux3 == nullptr || g->bstride2 == nullptr) return 0;
      return (g->dim >= 1 && g->dim <= 3) ? g->dim : 0;
    case THB_COST_NONHOLONOMIC_SE2:
    case THB_COST_NONHOLONOMIC_VECTOR: return gp ? 0 : 3;
    case THB_COST_QUASI_STATIC_PUSHING_PLANAR:
      if (gp || g->x2 == nullptr || g->x3 == nullptr || g->bstride3 == nullptr || g->dim != 3) return 0;
      return 3;
    case THB_COST_EFF_OBJ_CONTACT_PLANAR:
      if (gp || g->aux2 == nullptr || g->aux3 == nullptr || g->aux4 == nullptr || g->bstride2 == nullptr || g->grid_rows < 1 || g->grid_cols < 1 ||
          g->dim != 1)
        return 0;
      return 3;
    default: return 0;
  }
}

template <typename T> __global__ void error_reduce_kernel(const T* __restrict__ partial, int nchunks, int64_t B, T* __restrict__ err) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  T s = T(0);
  for (int c = 0; c < nchunks; c++) s += partial[(int64_t)c * B + b];
  err[b] = s;
}

// ------------------------------------------------------------------------------------------------
template <typename T> struct VarDev {
  int N;
  const T* const* x;
  T* const* out;
  const int32_t* kind;
  const int32_t* col;
  const int32_t* dof;
};
template <typename T> static VarDev<T> to_dev(const thb_var_table* v) {
  VarDev<T> d;
  d.N = v->N;
  d.x = reinterpret_cast<const T* const*>(v->x);
  d.out = reinterpret_cast<T* const*>(v->out);
  d.kind = v->kind;
  d.col = v->col;
  d.dof = v->dof;
  return d;
}

template <typename T>
__global__ void __launch_bounds__(128) retract_kernel(VarDev<T> v, int64_t B, const T* __restrict__ delta, int64_t n, T step,
                                                      const uint8_t* __restrict__ ignore) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)v.N * B) return;
  const int i = (int)(t / B);
  const int64_t b = t - (int64_t)i * B;
  const int kind = v.kind[i];
  const bool keep = ignore != nullptr && ignore[b] != 0;
  const T* d = delta + b * n + v.col[i];
  if (kind == THB_VAR_SE3) {
    const T* xp = v.x[i] + b * 12;
    T* op = v.out[i] + b * 12;
    T X[12], O[12];
    load_se3(xp, X);
    if (keep) {
#pragma unroll
      for (int q = 0; q < 12; q++) O[q] = X[q];
    } else {
      T xi[6], G[12];
#pragma unroll
      for (int q = 0; q < 6; q++) xi[q] = d[q] * step;
      se3_exp(xi, G);
      se3_compose(X, G, O);
    }
#pragma unroll
    for (int q = 0; q < 12; q++) op[q] = O[q];
  } else if (kind == THB_VAR_SO3) {
    const T* xp = v.x[i] + b * 9;
    T* op = v.out[i] + b * 9;
    T X[9], O[9];
    load_n<T, 9>(xp, X);
    if (keep) {
#pragma unroll
      for (int q = 0; q < 9; q++) O[q] = X[q];
    } else {
      T w[3], R[9];
#pragma unroll
      for (int q = 0; q < 3; q++) w[q] = d[q] * step;
      so3_exp<T, 3>(w, R);
      mat3_mul(X, R, O);
    }
#pragma unroll
    for (int q = 0; q < 9; q++) op[q] = O[q];
  } else if (kind == THB_VAR_SE2) {
    const T* xp = v.x[i] + b * 4;
    T* op = v.out[i] + b * 4;
    T X[4], O[4];
    load_n<T, 4>(xp, X);
    if (keep) {
#pragma unroll
      for (int q = 0; q < 4; q++) O[q] = X[q];
    } else {
      T xi[3], G[4];
#pragma unroll
      for (int q = 0; q < 3; q++) xi[q] = d[q] * step;
      se2_exp(xi, G);
      se2_compose(X, G, O);
    }
#pragma unroll
    for (int q = 0; q < 4; q++) op[q] = O[q];
  } else if (kind == THB_VAR_SO2) {  // storage [cos, sin], tangent theta: X * exp(theta) (geometry/so2.py:167-186 exp_map, :224-230 compose)
    const T* xp = v.x[i] + b * 2;
    T* op = v.out[i] + b * 2;
    const T c0 = xp[0], s0 = xp[1];
    if (keep) {
      op[0] = c0;
      op[1] = s0;
    } else {
      T s1, c1;
      t_sincos(d[0] * step, &s1, &c1);
      op[0] = c0 * c1 - s0 * s1;
      op[1] = s0 * c1 + c0 * s1;
    }
  } else {  // Vector / Point: x + delta
    const int dof = v.dof[i];
    const T* xp = v.x[i] + b * dof;
    T* op = v.out[i] + b * dof;
    for (int q = 0; q < dof; q++) op[q] = keep ? xp[q] : (xp[q] + d[q] * step);
  }
}

template <typename T>
__global__ void commit_kernel(VarDev<T> v, int64_t B, const uint8_t* __restrict__ keep_old) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)v.N * B) return;
  const int i = (int)(t / B);
  const int64_t b = t - (int64_t)i * B;
  if (keep_old != nullptr && keep_old[b]) return;
  const int kind = v.kind[i];
  const int sz = (kind == THB_VAR_SE3) ? 12 : ((kind == THB_VAR_SO3) ? 9 : ((kind == THB_VAR_SE2) ? 4 : ((kind == THB_VAR_SO2) ? 2 : v.dof[i])));
  const T* src = v.out[i] + b * sz;
  T* dst = const_cast<T*>(v.x[i]) + b * sz;
  for (int q = 0; q < sz; q++) dst[q] = src[q];
}

// ------------------------------------------------------------------------------------------------
// LM control: one CTA per batch item reduces den over n columns (levenberg_marquardt.py:172-201); partial sums per thread, per warp
// (shuffles) and per CTA (warp order) -- a fixed order, so the accept decision is reproducible.  (One WARP per item leaves too few
// warps to stream the three n-vectors of a large batch.)
constexpr int kLmCtrlThreads = 256;
template <typename T>
__global__ void __launch_bounds__(kLmCtrlThreads) lm_control_kernel(const T* __restrict__ delta, const T* __restrict__ Atb, const T* __restrict__ diag, int64_t B,
                                  int64_t n, T step, const T* __restrict__ err_prev, const T* __restrict__ err_new,
                                  T* __restrict__ lam, int ellipsoidal, T accept, T down, T up, uint8_t* __restrict__ reject,
                                  T* __restrict__ err_out, int32_t* __restrict__ stats) {
  __shared__ T part[kLmCtrlThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t b = blockIdx.x;
  if (b >= B) return;
  const T l = lam[b];
  T acc = T(0);
#pragma unroll 4
  for (int64_t j = tid; j < n; j += kLmCtrlThreads) {
    const T d = delta[b * n + j] * step;
    const T le = ellipsoidal ? (l * diag[b * n + j]) : l;
    acc += d * (le * d + Atb[b * n + j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) part[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    T sum = T(0);
#pragma unroll
    for (int q = 0; q < kLmCtrlThreads / 32; q++) sum += part[q];
    const T den = sum / T(2);
    const T rho = (err_prev[b] - err_new[b]) / den;
    const bool rej = rho <= accept;  // NaN compares false -> accepted, like torch's `rho <= damping_accept`
    T nl = rej ? (l * up) : (l / down);
    nl = (nl < T(1e-7)) ? T(1e-7) : ((nl > T(1e7)) ? T(1e7) : nl);
    lam[b] = nl;
    reject[b] = rej ? 1 : 0;
    err_out[b] = rej ? err_prev[b] : err_new[b];
    if (rej) atomicAdd(&stats[0], 1);
  }
}

// ------------------------------------------------------------------------------------------------
// stand-alone Lie kernels
template <typename T> __global__ void k_se3_exp(const T* __restrict__ xi, T* __restrict__ G, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  T x[6], g[12];
  load_n<T, 6>(xi + i * 6, x);
  se3_exp(x, g);
#pragma unroll
  for (int q = 0; q < 12; q++) G[i * 12 + q] = g[q];
}
template <typename T> __global__ void k_se3_log(const T* __restrict__ G, T* __restrict__ xi, T* __restrict__ J, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  T g[12], x[6], jl[36];
  load_se3(G + i * 12, g);
  if (J != nullptr) {
    se3_log_jlog<T, true>(g, x, jl);
#pragma unroll
    for (int q = 0; q < 36; q++) J[i * 36 + q] = jl[q];
  } else {
    se3_log_jlog<T, false>(g, x, jl);
  }
#pragma unroll
  for (int q = 0; q < 6; q++) xi[i * 6 + q] = x[q];
}
template <typename T> __global__ void k_se3_adjoint(const T* __restrict__ G, T* __restrict__ A, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  T g[12], a[36];
  load_se3(G + i * 12, g);
  se3_adjoint(g, a);
#pragma unroll
  for (int q = 0; q < 36; q++) A[i * 36 + q] = a[q];
}
template <typename T> __global__ void k_se3_inverse(const T* __restrict__ G, T* __restrict__ O, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  T g[12], o[12];
  load_se3(G + i * 12, g);
  se3_inverse(g, o);
#pragma unroll
  for (int q = 0; q < 12; q++) O[i * 12 + q] = o[q];
}
template <typename T> __global__ void k_se3_compose(const T* __restrict__ G0, const T* __restrict__ G1, T* __restrict__ O, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  T a[12], b[12], o[12];
  load_se3(G0 + i * 12, a);
  load_se3(G1 + i * 12, b);
  se3_compose(a, b, o);
#pragma unroll
  for (int q = 0; q < 12; q++) O[i * 12 + q] = o[q];
}

// ------------------------------------------------------------------------------------------------
static inline unsigned grid_for(int64_t total, int threads) { return (unsigned)((total + threads - 1) / threads); }

// The motion-planning kinds whose pose dof D varies: the MpCost instance of the dof mp_dof() checked.
template <typename T, int KIND, class F> static int with_mp_dof(int dof, F& f) {
  if (dof == 1) return f(MpCost<T, KIND, 1>());
  if (dof == 2) return f(MpCost<T, KIND, 2>());
  if (dof == 3) return f(MpCost<T, KIND, 3>());
  return THB_ERR_BAD_ARG;
}

// Calls f(Cost()) with the policy of g->kind (and, for the motion-planning kinds, its pose dof) and returns what f returns;
// THB_ERR_BAD_ARG if the group lacks a field its kind reads, THB_ERR_UNSUPPORTED for an unknown kind.
template <typename T, class F> static int with_cost_kind(const thb_cost_group* g, F f) {
  const int dof = mp_dof(g);   // 0 for the other kinds
  switch (g->kind) {
    case THB_COST_BETWEEN_SE3: return f(LieCost<T, THB_COST_BETWEEN_SE3>());
    case THB_COST_LOCAL_SE3: return f(LieCost<T, THB_COST_LOCAL_SE3>());
    case THB_COST_BETWEEN_SO3: return f(LieCost<T, THB_COST_BETWEEN_SO3>());
    case THB_COST_LOCAL_SO3: return f(LieCost<T, THB_COST_LOCAL_SO3>());
    case THB_COST_BETWEEN_SE2: return f(LieCost<T, THB_COST_BETWEEN_SE2>());
    case THB_COST_LOCAL_SE2: return f(LieCost<T, THB_COST_LOCAL_SE2>());
    case THB_COST_LOCAL_VECTOR: return f(VectorCost<T>());
    case THB_COST_REPROJECTION:
      if (g->aux2 == nullptr || g->aux3 == nullptr || g->aux4 == nullptr || g->bstride2 == nullptr) return THB_ERR_BAD_ARG;
      return f(ReprojectionCost<T>());
    case THB_COST_COLLISION2D_POINT2: return dof ? f(MpCost<T, THB_COST_COLLISION2D_POINT2, 2>()) : THB_ERR_BAD_ARG;
    case THB_COST_COLLISION2D_SE2: return dof ? f(MpCost<T, THB_COST_COLLISION2D_SE2, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_DOUBLE_INTEGRATOR_SE2: return dof ? f(MpCost<T, THB_COST_DOUBLE_INTEGRATOR_SE2, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_NONHOLONOMIC_SE2: return dof ? f(MpCost<T, THB_COST_NONHOLONOMIC_SE2, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_NONHOLONOMIC_VECTOR: return dof ? f(MpCost<T, THB_COST_NONHOLONOMIC_VECTOR, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_QUASI_STATIC_PUSHING_PLANAR: return dof ? f(MpCost<T, THB_COST_QUASI_STATIC_PUSHING_PLANAR, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_EFF_OBJ_CONTACT_PLANAR: return dof ? f(MpCost<T, THB_COST_EFF_OBJ_CONTACT_PLANAR, 3>()) : THB_ERR_BAD_ARG;
    case THB_COST_DOUBLE_INTEGRATOR_VECTOR: return with_mp_dof<T, THB_COST_DOUBLE_INTEGRATOR_VECTOR>(dof, f);
    case THB_COST_HINGE: return with_mp_dof<T, THB_COST_HINGE>(dof, f);
    default: return THB_ERR_UNSUPPORTED;
  }
}

// A kernel instance that needs more than the default 48 KB of dynamic shared memory opts in, once.
template <typename T, class Cost> static int allow_linearize_smem(size_t smem) {
  static bool done = false;
  if (!done && smem > 48 * 1024) {
    THB_CUDA(cudaFuncSetAttribute(linearize_kernel<T, Cost>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    done = true;
  }
  return THB_OK;
}

template <typename T>
static int linearize_group(const thb_cost_group* g, int64_t B, T* A_val, int64_t nnz, T* b, int64_t m, thb_stream_t s) {
  if (g == nullptr || g->K < 0 || B < 0) return THB_ERR_BAD_ARG;
  if (g->K == 0 || B == 0) return THB_OK;
  const GroupDev<T> d = to_dev<T>(g);
  const unsigned grid = grid_for((int64_t)g->K * B, 128);
  return with_cost_kind<T>(g, [&](auto cost) {
    using Cost = decltype(cost);
    const size_t smem = Cost::NV > 0 ? (size_t)4 * 32 * (Cost::NV + 1) * sizeof(T) : 0;   // 4 warps x 32 staged rows
    const int rc = allow_linearize_smem<T, Cost>(smem);
    if (rc != THB_OK) return rc;
    linearize_kernel<T, Cost><<<grid, 128, smem, thb_cs(s)>>>(d, B, A_val, nnz, b, m);
    THB_CHECK_LAUNCH();
    return THB_OK;
  });
}

template <typename T> static int error_group(const thb_cost_group* g, int64_t B, T* partial, thb_stream_t s) {
  if (g == nullptr || g->K < 0 || B < 0) return THB_ERR_BAD_ARG;
  if (g->K == 0 || B == 0) return THB_OK;
  const GroupDev<T> d = to_dev<T>(g);
  const int nchunks = (g->K + kErrCostsPerThread - 1) / kErrCostsPerThread;
  const unsigned grid = grid_for((int64_t)nchunks * B, 128);
  return with_cost_kind<T>(g, [&](auto cost) {
    error_kernel<T, decltype(cost)><<<grid, 128, 0, thb_cs(s)>>>(d, B, partial);
    THB_CHECK_LAUNCH();
    return THB_OK;
  });
}

template <typename T>
static int retract_impl(const thb_var_table* vt, int64_t B, const T* delta, int64_t n, T step, const uint8_t* ignore, thb_stream_t s) {
  if (vt == nullptr || vt->N < 0 || B < 0) return THB_ERR_BAD_ARG;
  if (vt->N == 0 || B == 0) return THB_OK;
  retract_kernel<T><<<grid_for((int64_t)vt->N * B, 128), 128, 0, thb_cs(s)>>>(to_dev<T>(vt), B, delta, n, step, ignore);
  THB_CHECK_LAUNCH();
  return THB_OK;
}
template <typename T> static int commit_impl(const thb_var_table* vt, int64_t B, const uint8_t* keep_old, thb_stream_t s) {
  if (vt == nullptr || vt->N < 0 || B < 0) return THB_ERR_BAD_ARG;
  if (vt->N == 0 || B == 0) return THB_OK;
  commit_kernel<T><<<grid_for((int64_t)vt->N * B, 128), 128, 0, thb_cs(s)>>>(to_dev<T>(vt), B, keep_old);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

}  // namespace thb

// ================================================================================================
template <typename T>
static int lm_control_impl(const T* delta, const T* Atb, const T* diag, int64_t B, int64_t n, T step, const T* err_prev, const T* err_new,
                           T* lam, int32_t ellipsoidal, T damping_accept, T down_ratio, T up_ratio, uint8_t* reject, T* err_out,
                           int32_t* stats, thb_stream_t s) {
  if (B <= 0) return THB_OK;
  if (ellipsoidal && diag == nullptr) return THB_ERR_BAD_ARG;
  THB_CUDA(cudaMemsetAsync(stats, 0, sizeof(int32_t) * 4, thb_cs(s)));
  const int threads = thb::kLmCtrlThreads;
  const unsigned grid = (unsigned)B;
  thb::lm_control_kernel<T><<<grid, threads, 0, thb_cs(s)>>>(delta, Atb, diag, B, n, step, err_prev, err_new, lam, ellipsoidal,
                                                              damping_accept, down_ratio, up_ratio, reject, err_out, stats);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

extern "C" {

int64_t thb_launch_counter_ = 0;
int64_t thb_launch_count(void) { return thb_launch_counter_; }
int thb_version(void) { return 100; }
int thb_compiled_arch(void) {
#ifdef THB_ARCH
  return THB_ARCH;
#else
  return 100;
#endif
}

int thb_linearize_group_f64(const thb_cost_group* g, int64_t B, double* A_val, int64_t nnz, double* b, int64_t m, thb_stream_t s) {
  return thb::linearize_group<double>(g, B, A_val, nnz, b, m, s);
}
int thb_linearize_group_f32(const thb_cost_group* g, int64_t B, float* A_val, int64_t nnz, float* b, int64_t m, thb_stream_t s) {
  return thb::linearize_group<float>(g, B, A_val, nnz, b, m, s);
}
int thb_error_num_chunks(int32_t K) { return (K + thb::kErrCostsPerThread - 1) / thb::kErrCostsPerThread; }
int thb_error_group_f64(const thb_cost_group* g, int64_t B, double* partial, thb_stream_t s) { return thb::error_group<double>(g, B, partial, s); }
int thb_error_group_f32(const thb_cost_group* g, int64_t B, float* partial, thb_stream_t s) { return thb::error_group<float>(g, B, partial, s); }
int thb_error_reduce_f64(const double* partial, int32_t nchunks, int64_t B, double* err, thb_stream_t s) {
  if (B <= 0) return THB_OK;
  thb::error_reduce_kernel<double><<<thb::grid_for(B, 128), 128, 0, thb_cs(s)>>>(partial, nchunks, B, err);
  THB_CHECK_LAUNCH();
  return THB_OK;
}
int thb_error_reduce_f32(const float* partial, int32_t nchunks, int64_t B, float* err, thb_stream_t s) {
  if (B <= 0) return THB_OK;
  thb::error_reduce_kernel<float><<<thb::grid_for(B, 128), 128, 0, thb_cs(s)>>>(partial, nchunks, B, err);
  THB_CHECK_LAUNCH();
  return THB_OK;
}
int thb_retract_f64(const thb_var_table* vt, int64_t B, const double* delta, int64_t n, double step, const uint8_t* ignore, thb_stream_t s) {
  return thb::retract_impl<double>(vt, B, delta, n, step, ignore, s);
}
int thb_retract_f32(const thb_var_table* vt, int64_t B, const float* delta, int64_t n, float step, const uint8_t* ignore, thb_stream_t s) {
  return thb::retract_impl<float>(vt, B, delta, n, step, ignore, s);
}
int thb_commit_f64(const thb_var_table* vt, int64_t B, const uint8_t* keep_old, thb_stream_t s) { return thb::commit_impl<double>(vt, B, keep_old, s); }
int thb_commit_f32(const thb_var_table* vt, int64_t B, const uint8_t* keep_old, thb_stream_t s) { return thb::commit_impl<float>(vt, B, keep_old, s); }

int thb_lm_control_f64(const double* delta, const double* Atb, const double* diag, int64_t B, int64_t n, double step,
                       const double* err_prev, const double* err_new, double* lam, int32_t ellipsoidal, double damping_accept,
                       double down_ratio, double up_ratio, uint8_t* reject, double* err_out, int32_t* stats, thb_stream_t s) {
  return lm_control_impl<double>(delta, Atb, diag, B, n, step, err_prev, err_new, lam, ellipsoidal, damping_accept, down_ratio, up_ratio,
                                 reject, err_out, stats, s);
}
int thb_lm_control_f32(const float* delta, const float* Atb, const float* diag, int64_t B, int64_t n, float step, const float* err_prev,
                       const float* err_new, float* lam, int32_t ellipsoidal, float damping_accept, float down_ratio, float up_ratio,
                       uint8_t* reject, float* err_out, int32_t* stats, thb_stream_t s) {
  return lm_control_impl<float>(delta, Atb, diag, B, n, step, err_prev, err_new, lam, ellipsoidal, damping_accept, down_ratio, up_ratio,
                                reject, err_out, stats, s);
}

int thb_fill_zero(void* ptr, int64_t bytes, thb_stream_t s) {
  THB_CUDA(cudaMemsetAsync(ptr, 0, (size_t)bytes, thb_cs(s)));
  return THB_OK;
}

#define THB_LIE_ENTRY(NAME, T, KERNEL, ...)                                                        \
  {                                                                                                \
    if (N <= 0) return THB_OK;                                                                     \
    KERNEL<T><<<thb::grid_for(N, 128), 128, 0, thb_cs(s)>>>(__VA_ARGS__);                          \
    THB_CHECK_LAUNCH();                                                                            \
    return THB_OK;                                                                                 \
  }
int thb_se3_exp_f64(const double* t, double* g, int64_t N, thb_stream_t s) THB_LIE_ENTRY(exp, double, thb::k_se3_exp, t, g, N)
int thb_se3_log_f64(const double* g, double* t, double* j, int64_t N, thb_stream_t s) THB_LIE_ENTRY(log, double, thb::k_se3_log, g, t, j, N)
int thb_se3_adjoint_f64(const double* g, double* a, int64_t N, thb_stream_t s) THB_LIE_ENTRY(adj, double, thb::k_se3_adjoint, g, a, N)
int thb_se3_inverse_f64(const double* g, double* o, int64_t N, thb_stream_t s) THB_LIE_ENTRY(inv, double, thb::k_se3_inverse, g, o, N)
int thb_se3_compose_f64(const double* a, const double* b, double* o, int64_t N, thb_stream_t s) THB_LIE_ENTRY(cmp, double, thb::k_se3_compose, a, b, o, N)
int thb_se3_exp_f32(const float* t, float* g, int64_t N, thb_stream_t s) THB_LIE_ENTRY(exp, float, thb::k_se3_exp, t, g, N)
int thb_se3_log_f32(const float* g, float* t, float* j, int64_t N, thb_stream_t s) THB_LIE_ENTRY(log, float, thb::k_se3_log, g, t, j, N)
int thb_se3_adjoint_f32(const float* g, float* a, int64_t N, thb_stream_t s) THB_LIE_ENTRY(adj, float, thb::k_se3_adjoint, g, a, N)
int thb_se3_inverse_f32(const float* g, float* o, int64_t N, thb_stream_t s) THB_LIE_ENTRY(inv, float, thb::k_se3_inverse, g, o, N)
int thb_se3_compose_f32(const float* a, const float* b, float* o, int64_t N, thb_stream_t s) THB_LIE_ENTRY(cmp, float, thb::k_se3_compose, a, b, o, N)

}  // extern "C"
