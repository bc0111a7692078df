// Exponential and 3-D power cones: per-cone arithmetic, one thread per cone (internal header).
//
// Device counterpart of the reference's nonsymmetric 3-D cones
//   /root/reference/src/solver/core/cones/expcone.rs, powcone.rs, nonsymmetric_common.rs
// and of the fixed 3x3 symmetric kernels they use (src/algebra/dense/fixed/dense3x3/{core,cholesky}.rs).
// A cone is three rows: everything lives in registers, there is nothing to share between threads, so the
// functions below are plain scalar code marked __host__ __device__.  cones_nonsym.cu wraps them in kernels
// (thread k = cone k, state in structure-of-arrays layout so that neighbouring threads read neighbouring
// doubles); tests/host_harness/ns3_host.cpp compiles the very same functions with g++ so that the CPU test
// suite can check them against the oracle without a GPU (test infrastructure only -- the product library
// never runs them on the host).
#pragma once
#include <cmath>

#if defined(__CUDACC__)
#define CB_HD __host__ __device__ __forceinline__
#else
#define CB_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define CB_UNROLL _Pragma("unroll")
#else
#define CB_UNROLL
#endif

namespace cb {
namespace ns3 {

constexpr double EPS = 2.220446049250313e-16;        // f64::EPSILON
constexpr double SQRT_EPS = 1.4901161193847656e-08;  // sqrt(f64::EPSILON)
constexpr int J_ZERO = 1 << 20;                      // "the step collapsed to zero" marker of the backtracking search
enum { KIND_EXP = 4, KIND_POW = 5 };                 // == CT_EXP / CT_POW
enum { STRAT_PRIMAL_DUAL = 0, STRAT_DUAL = 1 };      // ScalingStrategy (cones/mod.rs)

CB_HD double lsafe(double x) { return x <= 0.0 ? -INFINITY : log(x); }   // scalarmath.rs:14-20
CB_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// packed upper triangle of a symmetric 3x3, column by column: [h00 h01 h11 h02 h12 h22]
struct Sym3 {
  double d[6];
  CB_HD void mul(double* y, const double* x) const {                       // dense3x3/core.rs:20-27
    y[0] = d[0] * x[0] + d[1] * x[1] + d[3] * x[2];
    y[1] = d[1] * x[0] + d[2] * x[1] + d[4] * x[2];
    y[2] = d[3] * x[0] + d[4] * x[1] + d[5] * x[2];
  }
  CB_HD double quad(const double* y, const double* x) const {              // dense3x3/core.rs:39-46
    double t[3];
    mul(t, x);
    return y[0] * t[0] + y[1] * t[1] + y[2] * t[2];
  }
  CB_HD double fro() const {                                               // dense3x3/core.rs:29-37
    return sqrt(d[0] * d[0] + d[2] * d[2] + d[5] * d[5] + 2.0 * (d[1] * d[1] + d[3] * d[3] + d[4] * d[4]));
  }
};

// x = H^-1 b through an explicit 3x3 Cholesky factor; false when H is not positive definite
// (dense3x3/cholesky.rs:13-60)
CB_HD bool chol3_solve(const Sym3& H, double* x, const double* b) {
  if (!(H.d[0] > 0.0)) return false;
  const double l00 = sqrt(H.d[0]);
  const double l10 = H.d[1] / l00;
  const double t1 = H.d[2] - l10 * l10;
  if (!(t1 > 0.0)) return false;
  const double l11 = sqrt(t1);
  const double l20 = H.d[3] / l00;
  const double l21 = (H.d[4] - l10 * l20) / l11;
  const double t2 = H.d[5] - l20 * l20 - l21 * l21;
  if (!(t2 > 0.0)) return false;
  const double l22 = sqrt(t2);
  const double c0 = b[0] / l00;
  const double c1 = (b[1] - l10 * c0) / l11;
  const double c2 = (b[2] - l20 * c0 - l21 * c1) / l22;
  x[2] = c2 / l22;
  x[1] = (c1 - l21 * x[2]) / l11;
  x[0] = (c0 - l10 * x[1] - l20 * x[2]) / l00;
  return true;
}

// ------------------------------------------------------------------------------------------ exponential cone
// Wright omega function, w + log w = z for z >= 0: series start + two refinement steps (expcone.rs:397-456)
CB_HD double wright_omega(double z) {
  if (z < 0.0) return NAN;
  double w;
  if (z < 1.0 + 3.14159265358979323846) {
    const double t = z - 1.0;
    w = 1.0 + t * (0.5 + t * (1.0 / 16.0 + t * (-1.0 / 192.0 + t * (-1.0 / 3072.0 + t * (13.0 / 61440.0)))));
  } else {
    const double lz = log(z), zi = 1.0 / z;
    w = z - lz + lz * zi * (1.0 + zi * ((0.5 * lz - 1.0) + zi * (lz * lz / 3.0 - 1.5 * lz + 1.0)));
  }
  double r = z - w - lsafe(w);
CB_UNROLL
  for (int it = 0; it < 2; it++) {
    const double wp1 = w + 1.0;
    const double t = wp1 * (wp1 + (2.0 * r) / 3.0);
    w *= 1.0 + (r / wp1) * (t - 0.5 * r) / (t - r);
    const double r2 = r * r, p2 = wp1 * wp1;
    r = (2.0 * w * w - 8.0 * w - 1.0) / (72.0 * p2 * p2 * p2) * (r2 * r2);
  }
  return w;
}

// s3 >= s2 exp(s1/s2), s2, s3 > 0 (expcone.rs:205-217)
CB_HD bool exp_primal_feasible(const double* s) {
  return s[2] > 0.0 && s[1] > 0.0 && (s[1] * lsafe(s[2] / s[1]) - s[0]) > 0.0;
}
// z3 >= -z1 exp(z2/z1 - 1), z3 > 0, z1 < 0 (expcone.rs:220-231)
CB_HD bool exp_dual_feasible(const double* z) {
  return z[2] > 0.0 && z[0] < 0.0 && (z[1] - z[0] - z[0] * lsafe(-z[2] / z[0])) > 0.0;
}
CB_HD double exp_barrier_primal(const double* s) {                         // expcone.rs:233-250
  double w = wright_omega(1.0 - s[0] / s[1] - lsafe(s[1] / s[2]));
  w = (w - 1.0) * (w - 1.0) / w;
  return -lsafe(w) - 2.0 * lsafe(s[1]) - lsafe(s[2]) - 3.0;
}
CB_HD double exp_barrier_dual(const double* z) {                           // expcone.rs:252-262
  const double l = lsafe(-z[2] / z[0]);
  return -lsafe(-z[2] * z[0]) - lsafe(z[1] - z[0] - z[0] * l);
}
// gradient and Hessian of the dual barrier at z (expcone.rs:343-367)
CB_HD void exp_dual_grad_H(const double* z, double* g, Sym3& H) {
  const double l = lsafe(-z[2] / z[0]);
  const double r = -z[0] * l - z[0] + z[1];
  const double ri = 1.0 / r, r2 = r * r;
  g[0] = ri * l - 1.0 / z[0];
  g[1] = -ri;
  g[2] = (ri * z[0] - 1.0) / z[2];
  H.d[0] = (r2 - z[0] * r + l * l * z[0] * z[0]) / (r * z[0] * z[0] * r);
  H.d[1] = -l / r2;
  H.d[2] = 1.0 / r2;
  H.d[3] = (z[1] - z[0]) / (r2 * z[2]);
  H.d[4] = -z[0] / (r2 * z[2]);
  H.d[5] = (r2 - z[0] * r + z[0] * z[0]) / (r2 * z[2] * z[2]);
}
// gradient of the primal barrier at s (expcone.rs:375-387)
CB_HD void exp_grad_primal(const double* s, double* g) {
  const double w = wright_omega(1.0 - s[0] / s[1] - lsafe(s[1] / s[2]));
  g[0] = 1.0 / ((w - 1.0) * s[1]);
  g[1] = g[0] + g[0] * lsafe(w * s[1] / s[2]) - 1.0 / s[1];
  g[2] = w / ((1.0 - w) * s[2]);
}
// third-order correction eta at the scaling point z for the directions ds (primal) and v (dual)
// (expcone.rs:264-321)
CB_HD void exp_higher_correction(const Sym3& H, const double* z, const double* ds, const double* v, double* eta) {
  double u[3];
  if (!chol3_solve(H, u, ds)) { eta[0] = eta[1] = eta[2] = 0.0; return; }
  double gp[3];                                   // gradient of psi
  gp[1] = 1.0;
  gp[2] = -z[0] / z[2];
  gp[0] = lsafe(gp[2]);
  const double psi = z[0] * gp[0] - z[0] + z[1];
  const double du = dot3(u, gp), dv = dot3(v, gp);
  const double z0 = z[0], z2 = z[2], z22 = z2 * z2;
  const double coef = ((u[0] * (v[0] / z0 - v[2] / z2) + u[2] * (z0 * v[2] / z2 - v[0]) / z2) * psi - 2.0 * du * dv) /
                      (psi * psi * psi);
  const double ip2 = 1.0 / (psi * psi);
  double e0 = gp[0] * coef, e1 = gp[1] * coef, e2 = gp[2] * coef;
  e0 += (1.0 / psi - 2.0 / z0) * u[0] * v[0] / (z0 * z0) - u[2] * v[2] / z22 / psi +
        du * ip2 * (v[0] / z0 - v[2] / z2) + dv * ip2 * (u[0] / z0 - u[2] / z2);
  e2 += 2.0 * (z0 / psi - 1.0) * u[2] * v[2] / (z22 * z2) - (u[2] * v[0] + u[0] * v[2]) / z22 / psi +
        du * ip2 * (z0 * v[2] / z22 - v[0] / z2) + dv * ip2 * (z0 * u[2] / z22 - u[0] / z2);
  eta[0] = 0.5 * e0; eta[1] = 0.5 * e1; eta[2] = 0.5 * e2;
}

// ------------------------------------------------------------------------------------------ 3-D power cone
// s1^a s2^(1-a) >= |s3|, s1, s2 > 0 (powcone.rs:198-212)
CB_HD bool pow_primal_feasible(const double* s, double a) {
  return s[0] > 0.0 && s[1] > 0.0 && (exp(2.0 * a * lsafe(s[0]) + 2.0 * (1.0 - a) * lsafe(s[1])) - s[2] * s[2]) > 0.0;
}
// (z1/a)^a (z2/(1-a))^(1-a) >= |z3| (powcone.rs:215-232)
CB_HD bool pow_dual_feasible(const double* z, double a) {
  return z[0] > 0.0 && z[1] > 0.0 &&
         (exp(2.0 * a * lsafe(z[0] / a) + 2.0 * (1.0 - a) * lsafe(z[1] / (1.0 - a))) - z[2] * z[2]) > 0.0;
}
// Start of the one-sided Newton iterations of the power and generalised power cones' primal gradients: a point left
// of the root x of  r (phi(x) - x^2) = 2x,  r = |w| the norm of the cone's w-part, psi = 1 / sum(alpha_i^2).  It is
// genpowcone.rs:451-459's  -1/r + (psi r + sqrt((phi/r^2 + psi^2 - 1) phi)) / (phi - r^2)  with the -1/r cancelled
// against the square root, which otherwise leaves 0 or a negative start for r below about 1e-9 sqrt(phi).
CB_HD double newton_start(double r, double phi, double psi) {
  const double p1 = psi * psi - 1.0;
  return r * (psi + 1.0 + p1 / (1.0 + sqrt(1.0 + p1 * r * r / phi))) / (phi - r * r);
}
// Newton stopping rule shared by both cones (nonsymmetric_common.rs:191-219 stops BEFORE taking a step below
// sqrt(eps) relative, which leaves an error of that size): a step that is not positive is rounding noise and is not
// taken; a step below sqrt(eps) relative is taken and ends the iteration, the convergence being quadratic.
CB_HD bool newton_step(double& x, double dx, double f1) {
  if (!(dx >= EPS * x) || fabs(f1) < EPS) return false;
  x += dx;
  return dx >= SQRT_EPS * x;
}
// third component of the primal gradient: root of a scalar equation by a one-sided Newton iteration started to
// the left of it (powcone.rs:440-490, nonsymmetric_common.rs:191-219).  The start is the generalised power cone's
// with psi = 1 / (a^2 + (1-a)^2): powcone.rs:446 fixes psi = 2, which is left of the root only at a = 1/2.
CB_HD double pow_newton(double s3, double phi, double a) {
  const double b = 1.0 - a;
  double x = newton_start(s3, phi, 1.0 / (a * a + b * b));
  const double t0 = -2.0 * a * lsafe(a) - 2.0 * b * lsafe(b);
  const double lphi = lsafe(phi);
  for (int it = 0; it < 100; it++) {
    const double t1 = x * x, t2 = 2.0 * x / s3;
    const double f1 = 2.0 * a * a / (a * x + (1.0 + a) / s3) + 2.0 * b * b / (b * x + (2.0 - a) / s3) -
                      2.0 * (x + 1.0 / s3) / (t1 + t2);
    const double f0 = 2.0 * a * lsafe(2.0 * a * t1 + (1.0 + a) * t2) + 2.0 * b * lsafe(2.0 * b * t1 + (2.0 - a) * t2) -
                      lphi - lsafe(t1 + t2) - 2.0 * lsafe(t2) + t0;
    if (!newton_step(x, -f0 / f1, f1)) break;
  }
  return x;
}
CB_HD void pow_grad_primal(const double* s, double a, double* g) {          // powcone.rs:389-414
  const double phi = pow(s[0], 2.0 * a) * pow(s[1], 2.0 - 2.0 * a);
  const double as = fabs(s[2]);
  if (as > EPS) {
    double g2 = pow_newton(as, phi, a);
    if (s[2] < 0.0) g2 = -g2;
    g[2] = g2;
    g[0] = -(a * g2 * s[2] + 1.0 + a) / s[0];
    g[1] = -((1.0 - a) * g2 * s[2] + 2.0 - a) / s[1];
  } else {
    g[2] = 0.0;
    g[0] = -(1.0 + a) / s[0];
    g[1] = -(2.0 - a) / s[1];
  }
}
CB_HD double pow_barrier_primal(const double* s, double a) {                // powcone.rs:234-255
  double g[3];
  pow_grad_primal(s, a, g);
  return lsafe(pow(-g[0] / a, 2.0 * a) * pow(-g[1] / (1.0 - a), 2.0 - 2.0 * a) - g[2] * g[2]) +
         (1.0 - a) * lsafe(-g[0]) + a * lsafe(-g[1]) - 3.0;
}
CB_HD double pow_barrier_dual(const double* z, double a) {                  // powcone.rs:257-270
  const double arg = pow(z[0] / a, 2.0 * a) * pow(z[1] / (1.0 - a), 2.0 - 2.0 * a) - z[2] * z[2];
  return -lsafe(arg) - (1.0 - a) * lsafe(z[0]) - a * lsafe(z[1]);
}
CB_HD void pow_dual_grad_H(const double* z, double a, double* g, Sym3& H) {  // powcone.rs:350-381
  const double b = 1.0 - a;
  const double phi = pow(z[0] / a, 2.0 * a) * pow(z[1] / b, 2.0 - 2.0 * a);
  const double psi = phi - z[2] * z[2];
  const double p0 = 2.0 * a * phi / (z[0] * psi), p1 = 2.0 * b * phi / (z[1] * psi), p2 = -2.0 * z[2] / psi;
  H.d[0] = p0 * p0 - 2.0 * a * (2.0 * a - 1.0) * phi / (z[0] * z[0] * psi) + b / (z[0] * z[0]);
  H.d[1] = p0 * p1 - 4.0 * a * b * phi / (z[0] * z[1] * psi);
  H.d[2] = p1 * p1 - 2.0 * b * (1.0 - 2.0 * a) * phi / (z[1] * z[1] * psi) + a / (z[1] * z[1]);
  H.d[3] = p0 * p2;
  H.d[4] = p1 * p2;
  H.d[5] = p2 * p2 + 2.0 / psi;
  g[0] = -p0 - b / z[0];
  g[1] = -p1 - a / z[1];
  g[2] = -p2;
}
CB_HD void pow_higher_correction(const Sym3& H, const double* z, double a, const double* ds, const double* v,
                                 double* eta) {                              // powcone.rs:272-348
  double u[3];
  if (!chol3_solve(H, u, ds)) { eta[0] = eta[1] = eta[2] = 0.0; return; }
  const double b = 1.0 - a;
  const double phi = pow(z[0] / a, 2.0 * a) * pow(z[1] / b, 2.0 - 2.0 * a);
  const double psi = phi - z[2] * z[2];
  const double gp[3] = {2.0 * a * phi / z[0], 2.0 * b * phi / z[1], -2.0 * z[2]};
  Sym3 Hp;                                         // Hessian of psi
  Hp.d[0] = 2.0 * a * (2.0 * a - 1.0) * phi / (z[0] * z[0]);
  Hp.d[1] = 4.0 * a * b * phi / (z[0] * z[1]);
  Hp.d[2] = 2.0 * b * (1.0 - 2.0 * a) * phi / (z[1] * z[1]);
  Hp.d[3] = 0.0; Hp.d[4] = 0.0; Hp.d[5] = -2.0;
  const double du = dot3(u, gp), dv = dot3(v, gp);
  double Hv[3], Hu[3];
  Hp.mul(Hv, v);
  Hp.mul(Hu, u);
  const double coef = (dot3(u, Hv) * psi - 2.0 * du * dv) / (psi * psi * psi);
  const double coef2 = 4.0 * a * (2.0 * a - 1.0) * b * phi * (u[0] / z[0] - u[1] / z[1]) * (v[0] / z[0] - v[1] / z[1]) / psi;
  const double ip2 = 1.0 / (psi * psi);
  const double e0 = coef * gp[0] - 2.0 * b * u[0] * v[0] / (z[0] * z[0] * z[0]) + coef2 / z[0] + Hv[0] * du * ip2;
  const double e1 = coef * gp[1] - 2.0 * a * u[1] * v[1] / (z[1] * z[1] * z[1]) - coef2 / z[1] + Hv[1] * du * ip2;
  const double e2 = coef * gp[2] + Hv[2] * du * ip2;
  eta[0] = 0.5 * (e0 + dv * ip2 * Hu[0]);
  eta[1] = 0.5 * (e1 + dv * ip2 * Hu[1]);
  eta[2] = 0.5 * (e2 + dv * ip2 * Hu[2]);
}

// ------------------------------------------------------------------------------------------ both cones
CB_HD bool feasible(int kind, double a, const double* q, bool dual) {
  if (kind == KIND_EXP) return dual ? exp_dual_feasible(q) : exp_primal_feasible(q);
  return dual ? pow_dual_feasible(q, a) : pow_primal_feasible(q, a);
}
CB_HD void unit_init(int kind, double a, double* z, double* s) {            // expcone.rs:88-94, powcone.rs:79-87
  if (kind == KIND_EXP) { s[0] = -1.051383945322714; s[1] = 0.556409619469370; s[2] = 1.258967884768947; }
  else { s[0] = sqrt(1.0 + a); s[1] = sqrt(1.0 + (1.0 - a)); s[2] = 0.0; }
  z[0] = s[0]; z[1] = s[1]; z[2] = s[2];
}

// Hs for the primal-dual (Tuncel / MOSEK-style) scaling, falling back to mu H when (s, z) sit on the central
// path or the update would be ill conditioned (nonsymmetric_common.rs:72-143).  st = dual gradient at z,
// zt = primal gradient at s.
CB_HD void primal_dual_Hs(const double* s, const double* z, const double* st, const double* zt, const Sym3& Hd,
                          Sym3& Hs) {
  const double dsz = dot3(s, z);
  const double mu = dsz / 3.0, mut = dot3(st, zt) / 3.0;
  double ds[3], dz[3];
CB_UNROLL
  for (int i = 0; i < 3; i++) { ds[i] = s[i] + mu * st[i]; dz[i] = z[i] + mu * zt[i]; }
  const double ddsz = dot3(ds, dz);
  const double de1 = mu * mut - 1.0;
  const double de2 = Hd.quad(zt, zt) - 3.0 * mut * mut;
  if (fabs(de1) > SQRT_EPS && fabs(de2) > EPS && dsz > 0.0 && ddsz > 0.0) {
    double tmp[3];
    Hd.mul(tmp, zt);
CB_UNROLL
    for (int i = 0; i < 3; i++) tmp[i] = mut * st[i] - tmp[i];
    Sym3 W = Hd;
    int k = 0;
CB_UNROLL
    for (int j = 0; j < 3; j++)
CB_UNROLL
      for (int i = 0; i <= j; i++) W.d[k++] -= st[i] * st[j] / 3.0 + tmp[i] * tmp[j] / de2;
    const double t = mu * W.fro();
    double ax[3] = {z[1] * zt[2] - z[2] * zt[1], z[2] * zt[0] - z[0] * zt[2], z[0] * zt[1] - z[1] * zt[0]};
    // 2-norm with the scaling of vecmath.rs:206-226 so that tiny cross products do not underflow
    const double amax = fmax(fabs(ax[0]), fmax(fabs(ax[1]), fabs(ax[2])));
    if (amax > 0.0) {
      const double q0 = ax[0] / amax, q1 = ax[1] / amax, q2 = ax[2] / amax;
      const double inv = 1.0 / (amax * sqrt(q0 * q0 + q1 * q1 + q2 * q2));
      ax[0] *= inv; ax[1] *= inv; ax[2] *= inv;
    }
    k = 0;
CB_UNROLL
    for (int j = 0; j < 3; j++)
CB_UNROLL
      for (int i = 0; i <= j; i++) Hs.d[k++] = s[i] * s[j] / dsz + ds[i] * ds[j] / ddsz + t * ax[i] * ax[j];
  } else {
CB_UNROLL
    for (int i = 0; i < 6; i++) Hs.d[i] = mu * Hd.d[i];
  }
}

// Cone::update_scaling (expcone.rs:103-120, powcone.rs:96-113)
CB_HD void update_scaling(int kind, double a, const double* s, const double* z, double mu, int strategy,
                          Sym3& Hd, Sym3& Hs, double* g) {
  if (kind == KIND_EXP) exp_dual_grad_H(z, g, Hd); else pow_dual_grad_H(z, a, g, Hd);
  if (strategy == STRAT_DUAL) {
CB_UNROLL
    for (int i = 0; i < 6; i++) Hs.d[i] = mu * Hd.d[i];
    return;
  }
  double zt[3];
  if (kind == KIND_EXP) exp_grad_primal(s, zt); else pow_grad_primal(s, a, zt);
  primal_dual_Hs(s, z, g, zt, Hd, Hs);
}

// Cone::combined_ds_shift (expcone.rs:139-148): shift = sigma*mu*grad - eta
CB_HD void combined_shift(int kind, double a, const Sym3& Hd, const double* zc, const double* g, const double* step_s,
                          const double* step_z, double sigmamu, double* shift) {
  double eta[3];
  if (kind == KIND_EXP) exp_higher_correction(Hd, zc, step_s, step_z, eta);
  else pow_higher_correction(Hd, zc, a, step_s, step_z, eta);
CB_UNROLL
  for (int i = 0; i < 3; i++) shift[i] = g[i] * sigmamu - eta[i];
}

// Number of backtracking steps (a <- a*step) before q + a*dq is inside the cone, J_ZERO if the step falls
// below a_min first (nonsymmetric_common.rs:160-189).  Every cone walks the same sequence a0, a0*step, ... so
// the composite step of compositecone.rs:289-332 is the largest count over the cones.
CB_HD int backtrack_count(int kind, double a, const double* q, const double* dq, bool dual, double a0, double a_min,
                          double step) {
  double al = a0;
  for (int j = 0; j < 4096; j++) {
    const double w[3] = {q[0] + al * dq[0], q[1] + al * dq[1], q[2] + al * dq[2]};
    if (feasible(kind, a, w, dual)) return j;
    al *= step;
    if (al < a_min) return J_ZERO;
  }
  return J_ZERO;
}
CB_HD double backtrack_value(double a0, int count, double step) {
  if (count >= J_ZERO) return 0.0;
  double al = a0;
  for (int j = 0; j < count; j++) al *= step;
  return al;
}

// Cone::compute_barrier (expcone.rs:176-187)
CB_HD double barrier(int kind, double a, const double* z, const double* s, const double* dz, const double* ds,
                     double al) {
  const double cz[3] = {z[0] + al * dz[0], z[1] + al * dz[1], z[2] + al * dz[2]};
  const double cs[3] = {s[0] + al * ds[0], s[1] + al * ds[1], s[2] + al * ds[2]};
  return kind == KIND_EXP ? exp_barrier_dual(cz) + exp_barrier_primal(cs)
                          : pow_barrier_dual(cz, a) + pow_barrier_primal(cs, a);
}

// ---- barriers of the symmetric cones, needed by the same line search when a problem mixes cone types ----
// second-order cone (socone.rs:304-314, 410-417); one thread walks the cone
CB_HD double soc_barrier(const double* z, const double* s, const double* dz, const double* ds, int n, double al) {
  double qs = 0.0, qz = 0.0;
  for (int i = 1; i < n; i++) {
    const double si = s[i] + al * ds[i], zi = z[i] + al * dz[i];
    qs += si * si; qz += zi * zi;
  }
  const double s0 = s[0] + al * ds[0], z0 = z[0] + al * dz[0];
  const double ns = sqrt(qs), nz = sqrt(qz);
  const double rs = (s0 - ns) * (s0 + ns), rz = (z0 - nz) * (z0 + nz);
  return (rs > 0.0 && rz > 0.0) ? -0.5 * lsafe(rs * rz) : INFINITY;
}
// -logdet of the n x n matrix whose svec is x + al*dx (psdtrianglecone.rs:281-305); W is caller scratch of n*n
// doubles.  When the matrix is not positive definite the reference's logdet_barrier returns +inf and
// compute_barrier SUBTRACTS it, so the term is -inf there; kept as is (the step-length rule has already kept the
// point inside the cone, the branch is not reached in practice).
CB_HD double psd_neg_logdet(const double* x, const double* dx, int n, double al, double* W) {
  const double isq2 = 0.70710678118654752440;
  int t = 0;
  for (int c = 0; c < n; c++)
    for (int r = 0; r <= c; r++, t++) {
      const double v = x[t] + al * dx[t];
      W[c * n + r] = W[r * n + c] = (r == c) ? v : v * isq2;
    }
  double ld = 0.0;
  for (int j = 0; j < n; j++) {
    double d = W[j * n + j];
    for (int k = 0; k < j; k++) d -= W[k * n + j] * W[k * n + j];
    if (!(d > 0.0)) return -INFINITY;
    d = sqrt(d);
    W[j * n + j] = d;
    ld += log(d);
    for (int i = j + 1; i < n; i++) {
      double v = W[j * n + i];
      for (int k = 0; k < j; k++) v -= W[k * n + i] * W[k * n + j];
      W[j * n + i] = v / d;
    }
  }
  return -2.0 * ld;
}

// ------------------------------------------------------------------------------------------ thread bodies
// What thread k of the kernels in cones_nonsym.cu does.  The view holds the composite cone's index arrays and the
// per-cone state in structure-of-arrays form (component j of the k-th nonsymmetric cone at [j*n + k]).
struct View {
  int n;                 // number of nonsymmetric cones
  const int* list;       // [n] cone ids
  const int* type;       // [ncones] cone types
  const int* off;        // [ncones] first row
  const int* boff;       // [ncones] first entry of the Hs block
  const double* alpha;   // [n] power cone exponents
  double *Hd, *Hs;       // [6*n]
  double *grad, *zc;     // [3*n]
};
CB_HD void ld3(double* v, const double* p) { v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; }
CB_HD void ld_soa(const double* base, int n, int k, double* v, int cnt) { for (int j = 0; j < cnt; j++) v[j] = base[(size_t)j * n + k]; }
CB_HD void st_soa(double* base, int n, int k, const double* v, int cnt) { for (int j = 0; j < cnt; j++) base[(size_t)j * n + k] = v[j]; }

CB_HD void body_unit_init(const View& c, int k, double* z, double* s) {
  const int id = c.list[k], o = c.off[id];
  double zz[3], ss[3];
  unit_init(c.type[id], c.alpha[k], zz, ss);
  for (int i = 0; i < 3; i++) { z[o + i] = zz[i]; s[o + i] = ss[i]; }
}
CB_HD void body_update_scaling(const View& c, int k, const double* s_, const double* z_, double mu, int strategy) {
  const int id = c.list[k], o = c.off[id];
  double s[3], z[3], g[3];
  ld3(s, s_ + o); ld3(z, z_ + o);
  Sym3 Hd, Hs;
  update_scaling(c.type[id], c.alpha[k], s, z, mu, strategy, Hd, Hs, g);
  st_soa(c.Hd, c.n, k, Hd.d, 6);
  st_soa(c.Hs, c.n, k, Hs.d, 6);
  st_soa(c.grad, c.n, k, g, 3);
  st_soa(c.zc, c.n, k, z, 3);
}
CB_HD void body_get_Hs(const View& c, int k, double* Hs, double sign) {
  const int b = c.boff[c.list[k]];
  for (int j = 0; j < 6; j++) Hs[b + j] = sign * c.Hs[(size_t)j * c.n + k];
}
CB_HD void body_mul_Hs(const View& c, int k, double* y, const double* x) {
  const int o = c.off[c.list[k]];
  Sym3 H;
  ld_soa(c.Hs, c.n, k, H.d, 6);
  double xx[3], yy[3];
  ld3(xx, x + o);
  H.mul(yy, xx);
  y[o] = yy[0]; y[o + 1] = yy[1]; y[o + 2] = yy[2];
}
// affine_ds = s and ds_from_dz_offset = ds are copies of the cone's three rows (expcone.rs:135-137, 150-152)
CB_HD void body_copy_rows(const View& c, int k, double* out, const double* in) {
  const int o = c.off[c.list[k]];
  out[o] = in[o]; out[o + 1] = in[o + 1]; out[o + 2] = in[o + 2];
}
CB_HD void body_combined_shift(const View& c, int k, double* shift, const double* step_z, const double* step_s,
                               double sigmamu) {
  const int id = c.list[k], o = c.off[id];
  Sym3 Hd;
  double zc[3], g[3], ss[3], sz[3], sh[3];
  ld_soa(c.Hd, c.n, k, Hd.d, 6);
  ld_soa(c.zc, c.n, k, zc, 3);
  ld_soa(c.grad, c.n, k, g, 3);
  ld3(ss, step_s + o); ld3(sz, step_z + o);
  combined_shift(c.type[id], c.alpha[k], Hd, zc, g, ss, sz, sigmamu, sh);
  shift[o] = sh[0]; shift[o + 1] = sh[1]; shift[o + 2] = sh[2];
}
// backtracking count of cone k starting from a0 = min(alpha_sym, 1 - sqrt(eps)) (compositecone.rs:318-325)
CB_HD int body_step_count(const View& c, int k, const double* dz_, const double* ds_, const double* z_, const double* s_,
                          double alpha_sym, double a_min, double step) {
  const int id = c.list[k], o = c.off[id];
  const double a0 = fmin(alpha_sym, 1.0 - SQRT_EPS);
  double q[3], dq[3];
  ld3(q, z_ + o); ld3(dq, dz_ + o);
  const int jz = backtrack_count(c.type[id], c.alpha[k], q, dq, true, a0, a_min, step);
  ld3(q, s_ + o); ld3(dq, ds_ + o);
  const int js = backtrack_count(c.type[id], c.alpha[k], q, dq, false, a0, a_min, step);
  return jz > js ? jz : js;
}
CB_HD double body_step_final(double alpha_sym, int jmax, double step) {
  return backtrack_value(fmin(alpha_sym, 1.0 - SQRT_EPS), jmax, step);
}
CB_HD double body_barrier(const View& c, int k, const double* z, const double* s, const double* dz, const double* ds,
                          double al) {
  const int id = c.list[k], o = c.off[id];
  double zz[3], ss[3], dzz[3], dss[3];
  ld3(zz, z + o); ld3(ss, s + o); ld3(dzz, dz + o); ld3(dss, ds + o);
  return barrier(c.type[id], c.alpha[k], zz, ss, dzz, dss, al);
}

}  // namespace ns3

// ------------------------------------------------------------------------------------------------------------
// Generalised power cone { (u, w) : prod u_i^alpha_i >= ||w|| }, u in R^dim1, w in R^dim2
// (/root/reference/src/solver/core/cones/genpowcone.rs).  Hs = mu (D + p p' - q q' - r r') is never formed: its
// diagonal D goes into the KKT block, p, q, r into three extra KKT columns (datamaps.rs:226-337).  One thread per
// cone walks the cone's rows; all per-row state lives in m-length arrays indexed by row (q in the cone's first dim1
// rows of `qr`, r in the remaining dim2 rows), so no per-cone offsets beyond off[] are needed.
namespace gp {

struct View {
  int n;                 // number of generalised power cones
  const int* list;       // [n] cone ids
  const int* off;        // [ncones] first row
  const int* dim;        // [ncones] rows
  const int* boff;       // [ncones] first entry of the (diagonal) Hs block
  const int* dim1;       // [n]
  const double* alpha;   // [m] exponents, at the cone's first dim1 rows
  const double* psi;     // [n] 1 / sum(alpha^2)
  double *grad, *p, *qr, *d1, *zc;   // [m]
  double *d2, *mu;       // [n]
};
using ns3::lsafe;
using ns3::EPS;
using ns3::SQRT_EPS;
using ns3::J_ZERO;

// 2-norm with the scaling of vecmath.rs:206-226
CB_HD double norm2(const double* x, int n) {
  double mx = 0.0;
  for (int i = 0; i < n; i++) mx = fmax(mx, fabs(x[i]));
  if (!(mx > 0.0)) return 0.0;
  double ss = 0.0;
  for (int i = 0; i < n; i++) { const double t = x[i] / mx; ss += t * t; }
  return mx * sqrt(ss);
}

CB_HD void body_unit_init(const View& c, int k, double* z, double* s) {         // genpowcone.rs:132-141
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  for (int i = 0; i < n; i++) { const double v = i < d1 ? sqrt(1.0 + c.alpha[o + i]) : 0.0; s[o + i] = v; z[o + i] = v; }
}

// Cone::update_scaling = update_dual_grad_H + mu + copy of z (genpowcone.rs:149-163, 360-399); false where the
// reference asserts zeta > 0
CB_HD bool body_update_scaling(const View& c, int k, const double* z_, double mu) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k], d2n = n - d1;
  const double* z = z_ + o;
  const double* al = c.alpha + o;
  double phi = 1.0;
  for (int i = 0; i < d1; i++) phi *= pow(z[i] / al[i], 2.0 * al[i]);
  double norm2w = 0.0;
  for (int i = 0; i < d2n; i++) norm2w += z[d1 + i] * z[d1 + i];
  const double zeta = phi - norm2w;
  if (!(zeta > 0.0)) return false;
  const double p0 = sqrt(phi * (phi + norm2w) / 2.0);
  const double p1 = -2.0 * phi / p0;
  const double q0 = sqrt(zeta * phi / 2.0);
  const double r1 = 2.0 * sqrt(zeta / (phi + norm2w));
  for (int i = 0; i < d1; i++) {
    const double tau = 2.0 * al[i] / z[i];
    c.grad[o + i] = -tau * phi / zeta - (1.0 - al[i]) / z[i];
    c.d1[o + i] = tau * phi / (zeta * z[i]) + (1.0 - al[i]) / (z[i] * z[i]);
    c.p[o + i] = (p0 / zeta) * tau;
    c.qr[o + i] = tau * (q0 / zeta);
  }
  for (int i = d1; i < n; i++) {
    c.grad[o + i] = (2.0 / zeta) * z[i];
    c.p[o + i] = (p1 / zeta) * z[i];
    c.qr[o + i] = (r1 / zeta) * z[i];
  }
  c.d2[k] = 2.0 / zeta;
  c.mu[k] = mu;
  for (int i = 0; i < n; i++) c.zc[o + i] = z[i];
  return true;
}
CB_HD void body_get_Hs(const View& c, int k, double* Hs, double sign) {          // genpowcone.rs:169-175
  const int id = c.list[k], o = c.off[id], b = c.boff[id], n = c.dim[id], d1 = c.dim1[k];
  const double mu = c.mu[k], d2 = c.d2[k];
  for (int i = 0; i < n; i++) Hs[b + i] = sign * (mu * (i < d1 ? c.d1[o + i] : d2));
}
CB_HD void body_mul_Hs(const View& c, int k, double* y_, const double* x_) {     // genpowcone.rs:177-202
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  const double* x = x_ + o;
  double cp = 0.0, cq = 0.0, cr = 0.0;
  for (int i = 0; i < n; i++) cp += c.p[o + i] * x[i];
  for (int i = 0; i < d1; i++) cq += c.qr[o + i] * x[i];
  for (int i = d1; i < n; i++) cr += c.qr[o + i] * x[i];
  const double mu = c.mu[k], d2 = c.d2[k];
  for (int i = 0; i < n; i++) {
    const double base = i < d1 ? c.d1[o + i] * x[i] - cq * c.qr[o + i] : d2 * x[i] - cr * c.qr[o + i];
    y_[o + i] = (cp * c.p[o + i] + base) * mu;
  }
}
CB_HD void body_copy_rows(const View& c, int k, double* out, const double* in) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id];
  for (int i = 0; i < n; i++) out[o + i] = in[o + i];
}
CB_HD void body_combined_shift(const View& c, int k, double* shift, double sigmamu) {   // genpowcone.rs:208-213
  const int id = c.list[k], o = c.off[id], n = c.dim[id];
  for (int i = 0; i < n; i++) shift[o + i] = c.grad[o + i] * sigmamu;
}
// the three KKT columns and their diagonal entries (datamaps.rs:314-337): -sqrt(mu) q, -sqrt(mu) r, -sqrt(mu) p,
// diag (-1, -1, +1)
CB_HD void body_kkt_fill(const View& c, int k, double* vals, const int* map_qr, const int* map_p, const int* map_D) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id];
  const double sq = -sqrt(c.mu[k]);
  for (int i = 0; i < n; i++) { vals[map_qr[o + i]] = c.qr[o + i] * sq; vals[map_p[o + i]] = c.p[o + i] * sq; }
  vals[map_D[3 * k]] = -1.0; vals[map_D[3 * k + 1]] = -1.0; vals[map_D[3 * k + 2]] = 1.0;
}
// q + a*dq inside the primal / dual cone (genpowcone.rs:267-308)
CB_HD bool feasible(const double* al, const double* q, const double* dq, double a, int d1, int n, bool dual) {
  double res = 0.0;
  for (int i = 0; i < d1; i++) {
    const double v = q[i] + a * dq[i];
    if (!(v > 0.0)) return false;
    res += 2.0 * al[i] * lsafe(dual ? v / al[i] : v);
  }
  double ss = 0.0;
  for (int i = d1; i < n; i++) { const double v = q[i] + a * dq[i]; ss += v * v; }
  return exp(res) - ss > 0.0;
}
CB_HD int backtrack_count(const double* al, const double* q, const double* dq, int d1, int n, bool dual, double a0,
                          double a_min, double step) {
  double a = a0;
  for (int j = 0; j < 4096; j++) {
    if (feasible(al, q, dq, a, d1, n, dual)) return j;
    a *= step;
    if (a < a_min) return J_ZERO;
  }
  return J_ZERO;
}
CB_HD int body_step_count(const View& c, int k, const double* dz, const double* ds, const double* z, const double* s,
                          double alpha_sym, double a_min, double step) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  const double a0 = fmin(alpha_sym, 1.0 - SQRT_EPS);
  const int jz = backtrack_count(c.alpha + o, z + o, dz + o, d1, n, true, a0, a_min, step);
  const int js = backtrack_count(c.alpha + o, s + o, ds + o, d1, n, false, a0, a_min, step);
  return jz > js ? jz : js;
}
// dual barrier at q + a*dq (genpowcone.rs:333-354)
CB_HD double barrier_dual_at(const double* al, const double* q, const double* dq, double a, int d1, int n) {
  double res = 0.0, extra = 0.0, ss = 0.0;
  for (int i = 0; i < d1; i++) { const double v = q[i] + a * dq[i]; res += 2.0 * al[i] * lsafe(v / al[i]); extra += lsafe(v) * (1.0 - al[i]); }
  for (int i = d1; i < n; i++) { const double v = q[i] + a * dq[i]; ss += v * v; }
  return -lsafe(exp(res) - ss) - extra;
}
// The primal gradient at s + a*ds (genpowcone.rs:404-485) is g = (-(1 + al_i + al_i x |w|) / u_i, (x / |w|) w) for
// (u, w) = s + a*ds, with x = 0 when |w| <= eps and otherwise the root of a scalar equation, found by a one-sided
// Newton iteration (genpowcone.rs:451-485, nonsymmetric_common.rs:191-219).  Returns x, and |w| in *norm_w.
CB_HD double primal_grad_scalar(const View& c, int k, const double* s, const double* ds, double a, double* norm_w) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  const double* al = c.alpha + o;
  double phi = 1.0;
  for (int i = 0; i < d1; i++) phi *= pow(s[o + i] + a * ds[o + i], 2.0 * al[i]);
  double mx = 0.0;
  for (int i = d1; i < n; i++) mx = fmax(mx, fabs(s[o + i] + a * ds[o + i]));
  double norm_r = 0.0;
  if (mx > 0.0) {
    double ss = 0.0;
    for (int i = d1; i < n; i++) { const double t = (s[o + i] + a * ds[o + i]) / mx; ss += t * t; }
    norm_r = mx * sqrt(ss);
  }
  *norm_w = norm_r;
  if (!(norm_r > EPS)) return 0.0;
  double x = ns3::newton_start(norm_r, phi, c.psi[k]);
  for (int it = 0; it < 100; it++) {
    double f1 = -(2.0 * x + 2.0 / norm_r) / (x * x + 2.0 * x / norm_r);
    double f0 = -lsafe(2.0 * x / norm_r + x * x);
    for (int i = 0; i < d1; i++) {
      f1 += 2.0 * al[i] * norm_r / (norm_r * x + (1.0 + al[i]) / al[i]);
      f0 += 2.0 * al[i] * (lsafe(x * norm_r + (1.0 + al[i]) / al[i]) - lsafe(s[o + i] + a * ds[o + i]));
    }
    if (!ns3::newton_step(x, -f0 / f1, f1)) break;
  }
  return x;
}
// primal barrier at s + a*ds = -f*(-g(s)) - degree (genpowcone.rs:310-331).  The w-part of g is formed from the
// argument's own w-part; genpowcone.rs:426 takes the cone's stored Hessian vector r there, a shadowed name.
CB_HD double barrier_primal_at(const View& c, int k, const double* s, const double* ds, double a) {
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  const double* al = c.alpha + o;
  double norm_r;
  const double g1 = primal_grad_scalar(c, k, s, ds, a, &norm_r);
  const bool far = norm_r > EPS;
  // -f*(-g): dual barrier of the negated gradient, streamed
  double res = 0.0, extra = 0.0, ss = 0.0;
  for (int i = 0; i < d1; i++) {
    const double si = s[o + i] + a * ds[o + i];
    const double gi = far ? -(1.0 + al[i] + al[i] * g1 * norm_r) / si : -(1.0 + al[i]) / si;
    res += 2.0 * al[i] * lsafe(-gi / al[i]);
    extra += lsafe(-gi) * (1.0 - al[i]);
  }
  if (far) for (int i = d1; i < n; i++) { const double gi = (g1 / norm_r) * (s[o + i] + a * ds[o + i]); ss += gi * gi; }
  const double bd = -lsafe(exp(res) - ss) - extra;
  return -bd - (double)(d1 + 1);
}
CB_HD double body_barrier(const View& c, int k, const double* z, const double* s, const double* dz, const double* ds,
                          double a) {                                            // genpowcone.rs:249-263
  const int id = c.list[k], o = c.off[id], n = c.dim[id], d1 = c.dim1[k];
  return barrier_primal_at(c, k, s, ds, a) + barrier_dual_at(c.alpha + o, z + o, dz + o, a, d1, n);
}

}  // namespace gp
}  // namespace cb
