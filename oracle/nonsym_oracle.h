/* ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called by the product library.
 *
 * CPU restatement of the reference's nonsymmetric 3-dimensional cones: the exponential cone
 * (src/solver/core/cones/expcone.rs), the 3-D power cone (powcone.rs) and the scaling shared by the two
 * (nonsymmetric_common.rs), on top of the fixed 3x3 symmetric matrix type
 * (src/algebra/dense/fixed/dense3x3/{core,cholesky}.rs).  Included by ipm_oracle.c after its vector helpers
 * (vnorm = the overflow-safe 2-norm of vecmath.rs:206-226).
 *
 * Pinned on the reference's own tests: tests/basic_expcone.rs, tests/basic_powcone.rs, tests/mixed_conic.rs
 * (end to end, tests/test_oracle_nonsym.py) and the Wright-omega points of expcone.rs:459-472.
 */
#ifndef NONSYM_ORACLE_H
#define NONSYM_ORACLE_H

#define NS_EPS 2.220446049250313e-16

/* scalarmath.rs:14-20 */
static inline double logsafe(double x) { return x <= 0.0 ? -INFINITY : log(x); }

/* packed upper triangle of a symmetric 3x3: (0,0) (0,1) (1,1) (0,2) (1,2) (2,2)  (dense3x3/core.rs:66-78) */
#define S3(H, i, j) (H)[((j) >= (i)) ? ((j) * ((j) + 1) / 2 + (i)) : ((i) * ((i) + 1) / 2 + (j))]

/* dense3x3/core.rs:20-27 */
static inline void sym3_mul(const double *H, double *y, const double *x)
{
    y[0] = (H[0] * x[0]) + (H[1] * x[1]) + (H[3] * x[2]);
    y[1] = (H[1] * x[0]) + (H[2] * x[1]) + (H[4] * x[2]);
    y[2] = (H[3] * x[0]) + (H[4] * x[1]) + (H[5] * x[2]);
}
/* dense3x3/core.rs:29-37 */
static inline double sym3_norm_fro(const double *d)
{
    double sumsq = 0.0;
    sumsq += d[0] * d[0] + d[2] * d[2] + d[5] * d[5];
    sumsq += (d[1] * d[1] + d[3] * d[3] + d[4] * d[4]) * 2.0;
    return sqrt(sumsq);
}
/* dense3x3/core.rs:39-46 */
static inline double sym3_quad_form(const double *H, const double *y, const double *x)
{
    double out = 0.0;
    out += y[0] * (H[0] * x[0] + H[1] * x[1] + H[3] * x[2]);
    out += y[1] * (H[1] * x[0] + H[2] * x[1] + H[4] * x[2]);
    out += y[2] * (H[3] * x[0] + H[4] * x[1] + H[5] * x[2]);
    return out;
}
/* dense3x3/cholesky.rs:13-47: L overwrites a packed symmetric store (lower entries alias the upper ones) */
static inline int chol3_factor(double *L, const double *A)
{
    double t = S3(A, 0, 0);
    if (t <= 0.0) return 0;
    S3(L, 0, 0) = sqrt(t);
    S3(L, 1, 0) = S3(A, 1, 0) / S3(L, 0, 0);
    t = S3(A, 1, 1) - S3(L, 1, 0) * S3(L, 1, 0);
    if (t <= 0.0) return 0;
    S3(L, 1, 1) = sqrt(t);
    S3(L, 2, 0) = S3(A, 2, 0) / S3(L, 0, 0);
    S3(L, 2, 1) = (S3(A, 2, 1) - S3(L, 1, 0) * S3(L, 2, 0)) / S3(L, 1, 1);
    t = S3(A, 2, 2) - S3(L, 2, 0) * S3(L, 2, 0) - S3(L, 2, 1) * S3(L, 2, 1);
    if (t <= 0.0) return 0;
    S3(L, 2, 2) = sqrt(t);
    return 1;
}
/* dense3x3/cholesky.rs:50-60 */
static inline void chol3_solve(const double *L, double *x, const double *b)
{
    double c0 = b[0] / S3(L, 0, 0);
    double c1 = (b[1] - S3(L, 1, 0) * c0) / S3(L, 1, 1);
    double c2 = (b[2] - S3(L, 2, 0) * c0 - S3(L, 2, 1) * c1) / S3(L, 2, 2);
    x[2] = c2 / S3(L, 2, 2);
    x[1] = (c1 - S3(L, 2, 1) * x[2]) / S3(L, 1, 1);
    x[0] = (c0 - S3(L, 1, 0) * x[1] - S3(L, 2, 0) * x[2]) / S3(L, 0, 0);
}
static inline double dot3(const double *a, const double *b) { return ((0.0 + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]; }

/* per-cone state of ExponentialCone / PowerCone (expcone.rs:18-30, powcone.rs:17-33) */
typedef struct { double alpha; double H_dual[6], Hs[6], grad[3], z[3]; } ns3_t;

/* ------------------------------------------------------------------ exponential cone */
/* expcone.rs:397-456 (Wright omega, two refinement steps) */
static double wright_omega(double z)
{
    double p, w;
    if (z < 0.0) return NAN;   /* the reference panics */
    if (z < 1.0 + 3.14159265358979323846) {
        double zm1 = z - 1.0;
        p = zm1;
        w = 1.0 + p * 0.5;
        p *= zm1; w += p * (1.0 / 16.0);
        p *= zm1; w -= p * (1.0 / 192.0);
        p *= zm1; w -= p * (1.0 / 3072.0);
        p *= zm1; w += p * (13.0 / 61440.0);
    } else {
        double logz = logsafe(z), zinv = 1.0 / z;
        w = z - logz;
        double q = logz * zinv;
        w += q;
        q *= zinv;
        w += q * (logz / 2.0 - 1.0);
        q *= zinv;
        w += q * (logz * logz / 3.0 - logz * 1.5 + 1.0);
    }
    double r = z - w - logsafe(w);
    for (int it = 0; it < 2; it++) {
        double wp1 = w + 1.0;
        double t = wp1 * (wp1 + (r * 2.0) / 3.0);
        w *= 1.0 + (r / wp1) * (t - r * 0.5) / (t - r);
        double r4 = r * r * r * r;
        double wp16 = wp1 * wp1 * wp1 * wp1 * wp1 * wp1;
        r = (w * w * 2.0 - w * 8.0 - 1.0) / (wp16 * 72.0) * r4;
    }
    return w;
}
/* expcone.rs:205-217 */
static int exp_is_primal_feasible(const double *s)
{
    if (s[2] > 0.0 && s[1] > 0.0) {
        double res = s[1] * logsafe(s[2] / s[1]) - s[0];
        if (res > 0.0) return 1;
    }
    return 0;
}
/* expcone.rs:220-231 */
static int exp_is_dual_feasible(const double *z)
{
    if (z[2] > 0.0 && z[0] < 0.0) {
        double res = z[1] - z[0] - z[0] * logsafe(-z[2] / z[0]);
        if (res > 0.0) return 1;
    }
    return 0;
}
/* expcone.rs:233-250 */
static double exp_barrier_primal(const double *s)
{
    double w = wright_omega(1.0 - s[0] / s[1] - logsafe(s[1] / s[2]));
    w = (w - 1.0) * (w - 1.0) / w;
    return -logsafe(w) - logsafe(s[1]) * 2.0 - logsafe(s[2]) - 3.0;
}
/* expcone.rs:252-262 */
static double exp_barrier_dual(const double *z)
{
    double l = logsafe(-z[2] / z[0]);
    return -logsafe(-z[2] * z[0]) - logsafe(z[1] - z[0] - z[0] * l);
}
/* expcone.rs:343-367 */
static void exp_update_dual_grad_H(ns3_t *K, const double *z)
{
    double *grad = K->grad, *H = K->H_dual;
    double l = logsafe(-z[2] / z[0]);
    double r = -z[0] * l - z[0] + z[1];
    double c2 = 1.0 / r;
    grad[0] = c2 * l - 1.0 / z[0];
    grad[1] = -c2;
    grad[2] = (c2 * z[0] - 1.0) / z[2];
    S3(H, 0, 0) = (r * r - z[0] * r + l * l * z[0] * z[0]) / (r * z[0] * z[0] * r);
    S3(H, 0, 1) = -l / (r * r);
    S3(H, 1, 1) = 1.0 / (r * r);
    S3(H, 0, 2) = (z[1] - z[0]) / (r * r * z[2]);
    S3(H, 1, 2) = -z[0] / (r * r * z[2]);
    S3(H, 2, 2) = (r * r - z[0] * r + z[0] * z[0]) / (r * r * z[2] * z[2]);
}
/* expcone.rs:375-387 */
static void exp_gradient_primal(const double *s, double *g)
{
    double w = wright_omega(1.0 - s[0] / s[1] - logsafe(s[1] / s[2]));
    g[0] = 1.0 / ((w - 1.0) * s[1]);
    g[1] = g[0] + g[0] * logsafe(w * s[1] / s[2]) - 1.0 / s[1];
    g[2] = w / ((1.0 - w) * s[2]);
}
/* expcone.rs:264-321 */
static void exp_higher_correction(const ns3_t *K, double *eta, const double *ds, const double *v)
{
    const double *H = K->H_dual, *z = K->z;
    double u[3] = {0, 0, 0}, cholH[6] = {0, 0, 0, 0, 0, 0};
    if (chol3_factor(cholH, H)) chol3_solve(cholH, u, ds);
    else { eta[0] = eta[1] = eta[2] = 0.0; return; }
    eta[1] = 1.0;
    eta[2] = -z[0] / z[2];
    eta[0] = logsafe(eta[2]);
    double psi = z[0] * eta[0] - z[0] + z[1];
    double dotpsiu = dot3(u, eta), dotpsiv = dot3(v, eta);
    double coef = ((u[0] * (v[0] / z[0] - v[2] / z[2]) + u[2] * (z[0] * v[2] / z[2] - v[0]) / z[2]) * psi
                   - 2.0 * dotpsiu * dotpsiv) / (psi * psi * psi);
    for (int i = 0; i < 3; i++) eta[i] *= coef;
    double inv_psi2 = 1.0 / (psi * psi);
    eta[0] += (1.0 / psi - 2.0 / z[0]) * u[0] * v[0] / (z[0] * z[0])
            - u[2] * v[2] / (z[2] * z[2]) / psi
            + dotpsiu * inv_psi2 * (v[0] / z[0] - v[2] / z[2])
            + dotpsiv * inv_psi2 * (u[0] / z[0] - u[2] / z[2]);
    eta[2] += 2.0 * (z[0] / psi - 1.0) * u[2] * v[2] / (z[2] * z[2] * z[2])
            - (u[2] * v[0] + u[0] * v[2]) / (z[2] * z[2]) / psi
            + dotpsiu * inv_psi2 * (z[0] * v[2] / (z[2] * z[2]) - v[0] / z[2])
            + dotpsiv * inv_psi2 * (z[0] * u[2] / (z[2] * z[2]) - u[0] / z[2]);
    for (int i = 0; i < 3; i++) eta[i] *= 0.5;
}

/* ------------------------------------------------------------------ 3-D power cone */
/* powcone.rs:198-212 */
static int pow_is_primal_feasible(const double *s, double a)
{
    if (s[0] > 0.0 && s[1] > 0.0) {
        double res = exp(2.0 * a * logsafe(s[0]) + 2.0 * (1.0 - a) * logsafe(s[1])) - s[2] * s[2];
        if (res > 0.0) return 1;
    }
    return 0;
}
/* powcone.rs:215-232 */
static int pow_is_dual_feasible(const double *z, double a)
{
    if (z[0] > 0.0 && z[1] > 0.0) {
        double res = exp((a * 2.0) * logsafe(z[0] / a) + (1.0 - a) * logsafe(z[1] / (1.0 - a)) * 2.0) - z[2] * z[2];
        if (res > 0.0) return 1;
    }
    return 0;
}
/* Start of the one-sided Newton iterations of the power and generalised power cones: genpowcone.rs:451-459's
   -1/r + (psi r + sqrt((phi/r^2 + psi^2 - 1) phi)) / (phi - r^2) with the -1/r cancelled against the square root,
   which otherwise gives 0 or a negative start for r below about 1e-9 sqrt(phi). */
static double newton_onesided_start(double r, double phi, double psi)
{
    double p1 = psi * psi - 1.0;
    return r * (psi + 1.0 + p1 / (1.0 + sqrt(1.0 + p1 * r * r / phi))) / (phi - r * r);
}
/* Stopping rule of nonsymmetric_common.rs:191-219, except that a step below sqrt(eps) relative is taken before the
   iteration ends (the reference stops before it and keeps an error of that size), and a step is rounding noise when
   it is below eps relative rather than absolute. */
static int newton_onesided_step(double *x, double dx, double f1)
{
    if (!(dx >= NS_EPS * *x) || fabs(f1) < NS_EPS) return 0;
    *x += dx;
    return dx >= sqrt(NS_EPS) * *x;
}
/* nonsymmetric_common.rs:191-219 */
static double newton_raphson_onesided_pow(double x0, double s3, double phi, double a, double t0)
{
    double x = x0;
    for (int iter = 0; iter < 100; iter++) {
        /* powcone.rs:476-488 (f1) */
        double t1 = x * x, t2 = (2.0 * x) / s3;
        double dfdx = (a * a * 2.0) / (a * x + (1.0 + a) / s3)
                    + ((1.0 - a) * 2.0) * (1.0 - a) / ((1.0 - a) * x + (2.0 - a) / s3)
                    - ((x + 1.0 / s3) * 2.0) / (t1 + t2);
        /* powcone.rs:460-473 (f0) */
        double u1 = x * x, u2 = (x * 2.0) / s3;
        double f0 = 2.0 * a * logsafe(2.0 * a * u1 + (1.0 + a) * u2)
                  + 2.0 * (1.0 - a) * logsafe(2.0 * (1.0 - a) * u1 + (2.0 - a) * u2)
                  - logsafe(phi) - logsafe(u1 + u2) - 2.0 * logsafe(u2) + t0;
        if (!newton_onesided_step(&x, -f0 / dfdx, dfdx)) break;
    }
    return x;
}
/* powcone.rs:440-490, started like the generalised power cone with psi = 1 / (a^2 + (1-a)^2); powcone.rs:446 fixes
   psi = 2, which starts left of the root only at a = 1/2 */
static double newton_raphson_powcone(double s3, double phi, double a)
{
    double x0 = newton_onesided_start(s3, phi, 1.0 / (a * a + (1.0 - a) * (1.0 - a)));
    double t0 = -2.0 * a * logsafe(a) - 2.0 * (1.0 - a) * logsafe(1.0 - a);
    return newton_raphson_onesided_pow(x0, s3, phi, a, t0);
}
/* powcone.rs:389-414 */
static void pow_gradient_primal(const double *s, double a, double *g)
{
    double phi = pow(s[0], 2.0 * a) * pow(s[1], 2.0 - a * 2.0);
    double abs_s = fabs(s[2]);
    if (abs_s > NS_EPS) {
        g[2] = newton_raphson_powcone(abs_s, phi, a);
        if (s[2] < 0.0) g[2] = -g[2];
        g[0] = -(a * g[2] * s[2] + 1.0 + a) / s[0];
        g[1] = -((1.0 - a) * g[2] * s[2] + 2.0 - a) / s[1];
    } else {
        g[2] = 0.0;
        g[0] = -(1.0 + a) / s[0];
        g[1] = -(2.0 - a) / s[1];
    }
}
/* powcone.rs:234-255 */
static double pow_barrier_primal(const double *s, double a)
{
    double g[3];
    pow_gradient_primal(s, a, g);
    double out = 0.0;
    out += logsafe(pow(-g[0] / a, 2.0 * a) * pow(-g[1] / (1.0 - a), 2.0 - a * 2.0) - g[2] * g[2]);
    out += (1.0 - a) * logsafe(-g[0]);
    out += a * logsafe(-g[1]) - 3.0;
    return out;
}
/* powcone.rs:257-270 */
static double pow_barrier_dual(const double *z, double a)
{
    double arg1 = pow(z[0] / a, 2.0 * a) * pow(z[1] / (1.0 - a), 2.0 - 2.0 * a) - z[2] * z[2];
    return -logsafe(arg1) - (1.0 - a) * logsafe(z[0]) - a * logsafe(z[1]);
}
/* powcone.rs:350-381 */
static void pow_update_dual_grad_H(ns3_t *K, const double *z)
{
    double *H = K->H_dual, *g = K->grad; double a = K->alpha;
    double phi = pow(z[0] / a, 2.0 * a) * pow(z[1] / (1.0 - a), 2.0 - 2.0 * a);
    double psi = phi - z[2] * z[2];
    g[0] = 2.0 * a * phi / (z[0] * psi);
    g[1] = 2.0 * (1.0 - a) * phi / (z[1] * psi);
    g[2] = -2.0 * z[2] / psi;
    S3(H, 0, 0) = g[0] * g[0] - 2.0 * a * (2.0 * a - 1.0) * phi / (z[0] * z[0] * psi) + (1.0 - a) / (z[0] * z[0]);
    S3(H, 0, 1) = g[0] * g[1] - 4.0 * a * (1.0 - a) * phi / (z[0] * z[1] * psi);
    S3(H, 1, 1) = g[1] * g[1] - 2.0 * (1.0 - a) * (1.0 - 2.0 * a) * phi / (z[1] * z[1] * psi) + a / (z[1] * z[1]);
    S3(H, 0, 2) = g[0] * g[2];
    S3(H, 1, 2) = g[1] * g[2];
    S3(H, 2, 2) = g[2] * g[2] + 2.0 / psi;
    g[0] = -2.0 * a * phi / (z[0] * psi) - (1.0 - a) / z[0];
    g[1] = -2.0 * (1.0 - a) * phi / (z[1] * psi) - a / z[1];
    g[2] = 2.0 * z[2] / psi;
}
/* powcone.rs:272-348 */
static void pow_higher_correction(const ns3_t *K, double *eta, const double *ds, const double *v)
{
    const double *H = K->H_dual, *z = K->z; double a = K->alpha;
    double u[3] = {0, 0, 0}, M[6] = {0, 0, 0, 0, 0, 0};
    if (chol3_factor(M, H)) chol3_solve(M, u, ds);
    else { eta[0] = eta[1] = eta[2] = 0.0; return; }
    double phi = pow(z[0] / a, 2.0 * a) * pow(z[1] / (1.0 - a), 2.0 - 2.0 * a);
    double psi = phi - z[2] * z[2];
    eta[0] = 2.0 * a * phi / z[0];
    eta[1] = 2.0 * (1.0 - a) * phi / z[1];
    eta[2] = -2.0 * z[2];
    S3(M, 0, 1) = 4.0 * a * (1.0 - a) * phi / (z[0] * z[1]);
    S3(M, 0, 0) = 2.0 * a * (2.0 * a - 1.0) * phi / (z[0] * z[0]);
    S3(M, 0, 2) = 0.0;
    S3(M, 1, 1) = 2.0 * (1.0 - a) * (1.0 - 2.0 * a) * phi / (z[1] * z[1]);
    S3(M, 1, 2) = 0.0;
    S3(M, 2, 2) = -2.0;
    double dotpsiu = dot3(u, eta), dotpsiv = dot3(v, eta);
    double Hv[3];
    sym3_mul(M, Hv, v);
    double coef = (dot3(u, Hv) * psi - 2.0 * dotpsiu * dotpsiv) / (psi * psi * psi);
    double coef2 = 4.0 * a * (2.0 * a - 1.0) * (1.0 - a) * phi * (u[0] / z[0] - u[1] / z[1]) * (v[0] / z[0] - v[1] / z[1]) / psi;
    double inv_psi2 = 1.0 / (psi * psi);
    eta[0] = coef * eta[0] - 2.0 * (1.0 - a) * u[0] * v[0] / (z[0] * z[0] * z[0]) + coef2 / z[0] + Hv[0] * dotpsiu * inv_psi2;
    eta[1] = coef * eta[1] - 2.0 * a * u[1] * v[1] / (z[1] * z[1] * z[1]) - coef2 / z[1] + Hv[1] * dotpsiu * inv_psi2;
    eta[2] = coef * eta[2] + Hv[2] * dotpsiu * inv_psi2;
    double Hu[3];
    sym3_mul(M, Hu, u);
    for (int i = 0; i < 3; i++) eta[i] = (dotpsiv * inv_psi2) * Hu[i] + 1.0 * eta[i];   /* axpby(a, x, 1) */
    for (int i = 0; i < 3; i++) eta[i] *= 0.5;
}

/* ------------------------------------------------------------------ shared scaling */
/* nonsymmetric_common.rs:66-70 */
static void ns3_use_dual_scaling(ns3_t *K, double mu) { for (int i = 0; i < 6; i++) K->Hs[i] = mu * K->H_dual[i]; }

/* nonsymmetric_common.rs:72-143; zt = primal gradient at s (cone specific) */
static void ns3_use_primal_dual_scaling(ns3_t *K, const double *s, const double *z, const double *zt)
{
    double *H_dual = K->H_dual, *Hs = K->Hs, *st = K->grad;
    double ds_[3] = {0, 0, 0}, tmp[3] = {0, 0, 0}, dz_[3];
    double dot_sz = dot3(s, z);
    double mu = dot_sz / 3.0;
    double mut = dot3(st, zt) / 3.0;
    for (int i = 0; i < 3; i++) { ds_[i] = s[i] + mu * st[i]; dz_[i] = z[i] + mu * zt[i]; }
    double dot_dsz = dot3(ds_, dz_);
    double de1 = mu * mut - 1.0;
    double de2 = sym3_quad_form(H_dual, zt, zt) - 3.0 * mut * mut;
    if (fabs(de1) > sqrt(NS_EPS) && fabs(de2) > NS_EPS && dot_sz > 0.0 && dot_dsz > 0.0) {
        sym3_mul(H_dual, tmp, zt);
        for (int i = 0; i < 3; i++) tmp[i] = mut * st[i] - tmp[i];
        for (int i = 0; i < 6; i++) Hs[i] = H_dual[i];
        for (int i = 0; i < 3; i++)
            for (int j = i; j < 3; j++) S3(Hs, i, j) -= st[i] * st[j] / 3.0 + tmp[i] * tmp[j] / de2;
        double t = mu * sym3_norm_fro(Hs);
        double ax[3];
        ax[0] = z[1] * zt[2] - z[2] * zt[1];
        ax[1] = z[2] * zt[0] - z[0] * zt[2];
        ax[2] = z[0] * zt[1] - z[1] * zt[0];
        double nrm = vnorm(ax, 3);           /* normalize(): vecmath.rs:74-81 */
        if (nrm != 0.0) { double r = 1.0 / nrm; for (int i = 0; i < 3; i++) ax[i] *= r; }
        for (int i = 0; i < 3; i++)
            for (int j = i; j < 3; j++)
                S3(Hs, i, j) = s[i] * s[j] / dot_sz + ds_[i] * ds_[j] / dot_dsz + t * ax[i] * ax[j];
    } else {
        ns3_use_dual_scaling(K, mu);
    }
}


/* ------------------------------------------------------------------ generalised power cone (genpowcone.rs) */
/* { (u, w) : prod u_i^alpha_i >= ||w|| }, u in R^dim1, w in R^dim2.  State of GenPowerConeData (genpowcone.rs:10-60)
   plus the KKT maps of its rank-3 sparse expansion (datamaps.rs:226-243). */
typedef struct {
    idx dim1, dim2;
    double *alpha;
    double *grad, *z;           /* dual gradient, z at the scaling point */
    double mu;
    double *p, *q, *r, *d1;     /* Hs = mu (D + p p' - q q' - r r'),  D = diag(d1, d2 I) */
    double d2, psi;
    double *work, *work_pb;
    idx *map_p, *map_q, *map_r; idx map_D[3];
} gp_t;

static double gp_sumsq(const double *x, idx n) { double s = 0.0; for (idx i = 0; i < n; i++) s += x[i] * x[i]; return s; }

/* genpowcone.rs:267-286 */
static int gp_is_primal_feasible(const gp_t *K, const double *s)
{
    for (idx i = 0; i < K->dim1; i++) if (!(s[i] > 0.0)) return 0;
    double res = 0.0;
    for (idx i = 0; i < K->dim1; i++) res = res + 2.0 * K->alpha[i] * logsafe(s[i]);
    res = exp(res) - gp_sumsq(s + K->dim1, K->dim2);
    return res > 0.0;
}
/* genpowcone.rs:289-308 */
static int gp_is_dual_feasible(const gp_t *K, const double *z)
{
    for (idx i = 0; i < K->dim1; i++) if (!(z[i] > 0.0)) return 0;
    double res = 0.0;
    for (idx i = 0; i < K->dim1; i++) res = res + 2.0 * K->alpha[i] * logsafe(z[i] / K->alpha[i]);
    res = exp(res) - gp_sumsq(z + K->dim1, K->dim2);
    return res > 0.0;
}
/* genpowcone.rs:333-354 */
static double gp_barrier_dual(const gp_t *K, const double *z)
{
    double res = 0.0;
    for (idx i = 0; i < K->dim1; i++) res += 2.0 * K->alpha[i] * logsafe(z[i] / K->alpha[i]);
    res = exp(res) - gp_sumsq(z + K->dim1, K->dim2);
    double barrier = -logsafe(res);
    for (idx i = 0; i < K->dim1; i++) barrier -= logsafe(z[i]) * (1.0 - K->alpha[i]);
    return barrier;
}
/* genpowcone.rs:451-485 + nonsymmetric_common.rs:191-219 */
static double gp_newton_raphson(double norm_r, const double *p, double phi, const double *alpha, idx dim1, double psi)
{
    double x = newton_onesided_start(norm_r, phi, psi);
    for (int iter = 0; iter < 100; iter++) {
        double f1 = -(2.0 * x + 2.0 / norm_r) / (x * x + 2.0 * x / norm_r);
        for (idx i = 0; i < dim1; i++) f1 = f1 + 2.0 * alpha[i] * norm_r / (norm_r * x + (1.0 + alpha[i]) / alpha[i]);
        double f0 = -logsafe(2.0 * x / norm_r + x * x);
        for (idx i = 0; i < dim1; i++) f0 = f0 + 2.0 * alpha[i] * (logsafe(x * norm_r + (1.0 + alpha[i]) / alpha[i]) - logsafe(p[i]));
        if (!newton_onesided_step(&x, -f0 / f1, f1)) break;
    }
    return x;
}
/* genpowcone.rs:404-441, with the w-part of the gradient formed from the argument's own w-part: genpowcone.rs:426
   takes the cone's stored Hessian vector data.r there (a shadowed name), which is the gradient only when w || r. */
static void gp_gradient_primal(const gp_t *K, double *g, const double *s)
{
    idx dim1 = K->dim1, dim2 = K->dim2;
    double phi = 1.0;
    for (idx i = 0; i < dim1; i++) phi = phi * pow(s[i], 2.0 * K->alpha[i]);
    double norm_r = vnorm(s + dim1, dim2);
    if (norm_r > NS_EPS) {
        double g1 = gp_newton_raphson(norm_r, s, phi, K->alpha, dim1, K->psi);
        for (idx i = 0; i < dim2; i++) g[dim1 + i] = (g1 / norm_r) * s[dim1 + i];
        for (idx i = 0; i < dim1; i++) g[i] = -(1.0 + K->alpha[i] + K->alpha[i] * g1 * norm_r) / s[i];
    } else {
        for (idx i = 0; i < dim2; i++) g[dim1 + i] = 0.0;
        for (idx i = 0; i < dim1; i++) g[i] = -(1.0 + K->alpha[i]) / s[i];
    }
}
/* genpowcone.rs:310-331 */
static double gp_barrier_primal(gp_t *K, const double *s)
{
    double *g = K->work_pb; idx n = K->dim1 + K->dim2;
    gp_gradient_primal(K, g, s);
    for (idx i = 0; i < n; i++) g[i] = -g[i];
    return -gp_barrier_dual(K, g) - (double)(K->dim1 + 1);
}
/* genpowcone.rs:360-399; returns 0 where the reference asserts zeta > 0 */
static int gp_update_dual_grad_H(gp_t *K, const double *z)
{
    idx dim1 = K->dim1, dim2 = K->dim2;
    double phi = 1.0;
    for (idx i = 0; i < dim1; i++) phi = phi * pow(z[i] / K->alpha[i], 2.0 * K->alpha[i]);
    double norm2w = gp_sumsq(z + dim1, dim2);
    double zeta = phi - norm2w;
    if (!(zeta > 0.0)) return 0;
    double *tau = K->q;
    for (idx i = 0; i < dim1; i++) {
        tau[i] = 2.0 * K->alpha[i] / z[i];
        K->grad[i] = -tau[i] * phi / zeta - (1.0 - K->alpha[i]) / z[i];
    }
    for (idx i = 0; i < dim2; i++) K->grad[dim1 + i] = (2.0 / zeta) * z[dim1 + i];
    double p0 = sqrt(phi * (phi + norm2w) / 2.0);
    double p1 = -2.0 * phi / p0;
    double q0 = sqrt(zeta * phi / 2.0);
    double r1 = 2.0 * sqrt(zeta / (phi + norm2w));
    for (idx i = 0; i < dim1; i++) K->d1[i] = tau[i] * phi / (zeta * z[i]) + (1.0 - K->alpha[i]) / (z[i] * z[i]);
    K->d2 = 2.0 / zeta;
    for (idx i = 0; i < dim1; i++) K->p[i] = (p0 / zeta) * tau[i];
    for (idx i = 0; i < dim2; i++) K->p[dim1 + i] = (p1 / zeta) * z[dim1 + i];
    for (idx i = 0; i < dim1; i++) K->q[i] *= q0 / zeta;
    for (idx i = 0; i < dim2; i++) K->r[i] = (r1 / zeta) * z[dim1 + i];
    return 1;
}
/* genpowcone.rs:177-202 */
static void gp_mul_Hs(const gp_t *K, double *y, const double *x)
{
    idx dim1 = K->dim1, dim2 = K->dim2, n = dim1 + dim2;
    double coef_p = 0.0, coef_q = 0.0, coef_r = 0.0;
    for (idx i = 0; i < n; i++) coef_p += K->p[i] * x[i];
    for (idx i = 0; i < dim1; i++) coef_q += K->q[i] * x[i];
    for (idx i = 0; i < dim2; i++) coef_r += K->r[i] * x[dim1 + i];
    for (idx i = 0; i < dim1; i++) y[i] = K->d1[i] * x[i] - coef_q * K->q[i];
    for (idx i = 0; i < dim2; i++) y[dim1 + i] = K->d2 * x[dim1 + i] - coef_r * K->r[i];
    for (idx i = 0; i < n; i++) y[i] = coef_p * K->p[i] + 1.0 * y[i];
    for (idx i = 0; i < n; i++) y[i] *= K->mu;
}

#endif
