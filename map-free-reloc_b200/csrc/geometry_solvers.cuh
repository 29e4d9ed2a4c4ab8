// Minimal solvers of the pose back end, written as __host__ __device__ double-precision functions so
// the very same code runs inside the RANSAC kernels and in CPU unit tests (through the host test
// hooks of the C ABI). They replace the minimal solvers inside the OpenCV calls of the reference:
//   cv.findEssentialMat 5-point   (lib/models/matching/pose_solver.py:46-48)
//   cv.solvePnPRansac SOLVEPNP_P3P (pose_solver.py:209-213)
//   cv.recoverPose decomposition    (pose_solver.py:57)
// Algorithms: Nister's five-point formulation (null space -> 10 cubic constraints -> Gauss-Jordan ->
// degree-10 polynomial in z), P3P by eliminating the depth ratios to a quartic, real roots by
// derivative-interlaced bracketing + safeguarded Newton (no complex arithmetic, fixed work bound).
#pragma once

#include <math.h>

#ifdef __CUDACC__
#define MFR_HD __host__ __device__ __forceinline__
#define MFR_HDN __host__ __device__
#else
#define MFR_HD inline
#define MFR_HDN
#endif

namespace mfr {
namespace geo {

// ------------------------------------------------------------------------------------------------
// small linear algebra (row-major 3x3)
// ------------------------------------------------------------------------------------------------
MFR_HD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
MFR_HD void mat3_mul_bt(const double* A, const double* B, double* C) {  // A * B^T
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}
MFR_HD void mat3_vec(const double* A, const double* x, double* y) {
  for (int i = 0; i < 3; ++i) y[i] = A[3 * i] * x[0] + A[3 * i + 1] * x[1] + A[3 * i + 2] * x[2];
}
MFR_HD double det3(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) +
         A[2] * (A[3] * A[7] - A[4] * A[6]);
}
MFR_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
MFR_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
MFR_HD double norm3(const double* a) { return sqrt(dot3(a, a)); }

// R = exp([w]x)
MFR_HD void so3_exp(const double* w, double* R) {
  const double th2 = dot3(w, w);
  const double th = sqrt(th2);
  double a, b;  // sin(th)/th, (1-cos(th))/th^2
  if (th < 1e-8) {
    a = 1.0 - th2 / 6.0;
    b = 0.5 - th2 / 24.0;
  } else {
    a = sin(th) / th;
    b = (1.0 - cos(th)) / th2;
  }
  const double x = w[0], y = w[1], z = w[2];
  R[0] = 1.0 - b * (y * y + z * z); R[1] = -a * z + b * x * y;        R[2] = a * y + b * x * z;
  R[3] = a * z + b * x * y;         R[4] = 1.0 - b * (x * x + z * z); R[5] = -a * x + b * y * z;
  R[6] = -a * y + b * x * z;        R[7] = a * x + b * y * z;         R[8] = 1.0 - b * (x * x + y * y);
}

// E = [t]x R
MFR_HD void essential_from_rt(const double* R, const double* t, double* E) {
  const double tx[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
  mat3_mul(tx, R, E);
}

// Symmetric 3x3 eigen-decomposition by cyclic Jacobi (fixed sweep count). A is overwritten; V's
// columns are eigenvectors, eigenvalues returned in w (unsorted).
MFR_HD void jacobi_eig3(double* A, double* V, double* w) {
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 12; ++sweep) {
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[3 * p + q];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
        const double tt = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
        for (int k = 0; k < 3; ++k) {  // A <- A J
          const double akp = A[3 * k + p], akq = A[3 * k + q];
          A[3 * k + p] = c * akp - s * akq;
          A[3 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {  // A <- J^T A
          const double apk = A[3 * p + k], aqk = A[3 * q + k];
          A[3 * p + k] = c * apk - s * aqk;
          A[3 * q + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[3 * k + p], vkq = V[3 * k + q];
          V[3 * k + p] = c * vkp - s * vkq;
          V[3 * k + q] = s * vkp + c * vkq;
        }
      }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
}

// Decomposition of an essential matrix into the two rotations and the unit translation
// (the four (R, +-t) candidates of cv.recoverPose / cv.decomposeEssentialMat).
MFR_HD void decompose_essential(const double* E, double* R1, double* R2, double* t) {
  // E^T E = V diag(s^2) V^T
  double M[9], V[9], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[3 * i + j] = E[i] * E[j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
  jacobi_eig3(M, V, w);
  // order eigenvalues descending
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (w[o[b]] > w[o[a]]) { const int tmp = o[a]; o[a] = o[b]; o[b] = tmp; }
  double v0[3], v1[3], v2[3];
  for (int k = 0; k < 3; ++k) { v0[k] = V[3 * k + o[0]]; v1[k] = V[3 * k + o[1]]; }
  cross3(v0, v1, v2);  // right-handed V
  double u0[3], u1[3], u2[3];
  mat3_vec(E, v0, u0);
  mat3_vec(E, v1, u1);
  double n0 = norm3(u0);
  for (int k = 0; k < 3; ++k) u0[k] /= (n0 > 0 ? n0 : 1.0);
  // Gram-Schmidt u1 against u0 (exact for a true essential matrix)
  const double d01 = dot3(u0, u1);
  for (int k = 0; k < 3; ++k) u1[k] -= d01 * u0[k];
  double n1 = norm3(u1);
  for (int k = 0; k < 3; ++k) u1[k] /= (n1 > 0 ? n1 : 1.0);
  cross3(u0, u1, u2);  // right-handed U (det U = det V = +1)
  // R1 = U W V^T, R2 = U W^T V^T with W = [0 -1 0; 1 0 0; 0 0 1]
  //   U W   = [u1, -u0, u2],  U W^T = [-u1, u0, u2]   (as columns)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      R1[3 * i + j] = u1[i] * v0[j] - u0[i] * v1[j] + u2[i] * v2[j];
      R2[3 * i + j] = -u1[i] * v0[j] + u0[i] * v1[j] + u2[i] * v2[j];
    }
  for (int k = 0; k < 3; ++k) t[k] = u2[k];
}

// Least-squares rigid transform (Kabsch): R, t minimising sum |R p + t - q|^2 from the moment sums n, sum p, sum q,
// sum p q^T (row-major). H = sum (p - pb)(q - qb)^T = U S V^T by one-sided Jacobi on H's columns (accurate relative to
// the smaller singular values, unlike an eigen-decomposition of H^T H, which squares H's condition: near-collinear point
// sets lose the rotation about their line there); U, V right-handed, so R = V U^T is a rotation (for a reflection
// optimum, the rotation that flips the weakest direction, as SVD-based Kabsch does with its sign correction). false:
// n < 3, or H of rank < 2 (coincident or collinear points) above the rounding noise of the sums, 1e-13 of their scale.
MFR_HD bool kabsch_from_sums(double n, const double* sp, const double* sq, const double* spq, double* R, double* t) {
  if (n < 3.0) return false;
  double pb[3], qb[3], B[9], V[9];
  for (int k = 0; k < 3; ++k) { pb[k] = sp[k] / n; qb[k] = sq[k] / n; }
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) B[3 * a + b] = spq[3 * a + b] - n * pb[a] * qb[b];
  const double noise = 1e-13 * (n * norm3(pb) * norm3(qb) + sqrt(dot3(spq, spq) + dot3(spq + 3, spq + 3) +
                                                                   dot3(spq + 6, spq + 6)));
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  // B <- H V with orthogonal columns (fixed sweep count)
  for (int sweep = 0; sweep < 8; ++sweep)
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double al = 0.0, be = 0.0, ga = 0.0;
        for (int k = 0; k < 3; ++k) {
          al += B[3 * k + p] * B[3 * k + p]; be += B[3 * k + q] * B[3 * k + q]; ga += B[3 * k + p] * B[3 * k + q];
        }
        if (fabs(ga) < 1e-300) continue;
        const double ze = (be - al) / (2.0 * ga);
        const double tt = (ze >= 0 ? 1.0 : -1.0) / (fabs(ze) + sqrt(ze * ze + 1.0));
        const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
        for (int k = 0; k < 3; ++k) {
          const double bp = B[3 * k + p], bq = B[3 * k + q];
          B[3 * k + p] = c * bp - s * bq; B[3 * k + q] = s * bp + c * bq;
          const double vp = V[3 * k + p], vq = V[3 * k + q];
          V[3 * k + p] = c * vp - s * vq; V[3 * k + q] = s * vp + c * vq;
        }
      }
  double w[3];
  for (int j = 0; j < 3; ++j) w[j] = B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j];   // singular values^2
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (w[o[b]] > w[o[a]]) { const int tmp = o[a]; o[a] = o[b]; o[b] = tmp; }
  double v0[3], v1[3], v2[3], u0[3], u1[3], u2[3];
  for (int k = 0; k < 3; ++k) { v0[k] = V[3 * k + o[0]]; v1[k] = V[3 * k + o[1]]; u0[k] = B[3 * k + o[0]]; u1[k] = B[3 * k + o[1]]; }
  cross3(v0, v1, v2);
  const double n0 = norm3(u0);
  if (!(n0 > noise) || !(n0 > 1e-300)) return false;                   // coincident points
  for (int k = 0; k < 3; ++k) u0[k] /= n0;
  const double d01 = dot3(u0, u1);
  for (int k = 0; k < 3; ++k) u1[k] -= d01 * u0[k];
  const double n1 = norm3(u1);
  if (!(n1 > 1e-12 * n0 + noise)) return false;                        // collinear points
  for (int k = 0; k < 3; ++k) u1[k] /= n1;
  cross3(u0, u1, u2);
  // H = U S V^T  with U's columns u_i, V's columns v_i (both right-handed)  =>  R = V U^T
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) R[3 * a + b] = v0[a] * u0[b] + v1[a] * u1[b] + v2[a] * u2[b];
  double Rp[3];
  mat3_vec(R, pb, Rp);
  for (int k = 0; k < 3; ++k) t[k] = qb[k] - Rp[k];
  return true;
}

// ------------------------------------------------------------------------------------------------
// real roots of a polynomial  c[0] + c[1] x + ... + c[deg] x^deg,  deg <= 10
// Roots of p are bracketed by the roots of p' (recursively down to a quadratic) plus a Cauchy
// bound; every sign-changing bracket is polished by safeguarded Newton. Returns the root count.
// ------------------------------------------------------------------------------------------------
MFR_HD double poly_eval(const double* c, int deg, double x) {
  double r = c[deg];
  for (int i = deg - 1; i >= 0; --i) r = r * x + c[i];
  return r;
}
MFR_HD void poly_eval2(const double* c, int deg, double x, double* p, double* dp) {
  double r = c[deg], d = 0.0;
  for (int i = deg - 1; i >= 0; --i) {
    d = d * x + r;
    r = r * x + c[i];
  }
  *p = r;
  *dp = d;
}
MFR_HD double poly_refine(const double* c, int deg, double lo, double hi, double flo, double fhi) {
  // invariant: flo * fhi <= 0
  if (flo == 0.0) return lo;
  if (fhi == 0.0) return hi;
  double x = 0.5 * (lo + hi);
  for (int it = 0; it < 128; ++it) {
    double p, dp;
    poly_eval2(c, deg, x, &p, &dp);
    if (p == 0.0) return x;
    if ((p < 0.0) == (flo < 0.0)) { lo = x; flo = p; } else { hi = x; fhi = p; }
    double xn = (dp != 0.0) ? x - p / dp : lo - 1.0;
    if (!(xn > lo && xn < hi)) xn = 0.5 * (lo + hi);
    if (fabs(xn - x) <= 1e-15 * fmax(1.0, fabs(x))) { x = xn; break; }
    x = xn;
    if (hi - lo <= 1e-15 * fmax(1.0, fabs(lo))) break;
  }
  return x;
}

constexpr int kMaxDeg = 10;

MFR_HDN inline int poly_real_roots(const double* coef, int deg_in, double* roots) {
  // strip (numerically) vanishing leading coefficients
  double cmax = 0.0;
  for (int i = 0; i <= deg_in; ++i) cmax = fmax(cmax, fabs(coef[i]));
  if (cmax == 0.0 || !(cmax < 1e300)) return 0;
  int deg = deg_in;
  while (deg > 0 && fabs(coef[deg]) <= 1e-14 * cmax) --deg;
  if (deg == 0) return 0;
  // derivative table: d[k] holds the k-th derivative's coefficients (scaled, only roots matter)
  double d[kMaxDeg + 1][kMaxDeg + 1];
  for (int i = 0; i <= deg; ++i) d[0][i] = coef[i] / coef[deg];
  for (int k = 1; k < deg; ++k) {
    const int dk = deg - k;
    for (int i = 0; i <= dk; ++i) d[k][i] = d[k - 1][i + 1] * (i + 1) / (dk + 1.0);  // keep monic
  }
  // Cauchy bound for the monic polynomial (valid for all its derivatives after monic scaling? no:
  // compute one bound per level)
  double prev[kMaxDeg], cur[kMaxDeg];
  int nprev = 0;
  // level deg-1 is linear: x + d0 = 0
  {
    const double* c = d[deg - 1];
    prev[0] = -c[0] / c[1];
    nprev = 1;
  }
  for (int k = deg - 2; k >= 0; --k) {
    const int dk = deg - k;
    const double* c = d[k];
    // Fujiwara's bound for a monic polynomial: 2 max_k |c_{n-k}|^(1/k)
    double bound = 0.0;
    for (int i = 0; i < dk; ++i) bound = fmax(bound, pow(fabs(c[i]), 1.0 / (dk - i)));
    bound = 2.0 * bound + 1e-12;
    int ncur = 0;
    double lo = -bound, flo = poly_eval(c, dk, lo);
    for (int i = 0; i <= nprev; ++i) {
      double hi = (i < nprev) ? prev[i] : bound;
      if (hi < lo) hi = lo;  // guards against slightly unordered critical points
      const double fhi = poly_eval(c, dk, hi);
      if ((flo <= 0.0 && fhi >= 0.0) || (flo >= 0.0 && fhi <= 0.0)) {
        if (!(flo == 0.0 && fhi == 0.0) && ncur < dk) {
          const double r = poly_refine(c, dk, lo, hi, flo, fhi);
          if (ncur == 0 || r > cur[ncur - 1] + 1e-14 * fmax(1.0, fabs(r))) cur[ncur++] = r;
        }
      }
      lo = hi;
      flo = fhi;
    }
    for (int i = 0; i < ncur; ++i) prev[i] = cur[i];
    nprev = ncur;
    if (nprev == 0 && k > 0) {
      // derivative without real roots: polynomial at the next level is monotone; keep going with
      // an empty critical set (single bracket [-bound, bound]).
    }
  }
  for (int i = 0; i < nprev; ++i) roots[i] = prev[i];
  return nprev;
}

// ------------------------------------------------------------------------------------------------
// five-point relative pose (Nister). x0, x1: 5 normalised image points each; x1^T E x0 = 0.
// Writes up to 10 essential matrices (row-major 9 doubles each); returns their number.
// ------------------------------------------------------------------------------------------------
MFR_HDN inline int five_point(const double (*x0)[2], const double (*x1)[2], double (*Eout)[9]) {
  // ---- null space of the 5x9 epipolar constraint matrix (Gauss-Jordan, full pivoting)
  double A[5][9];
  for (int i = 0; i < 5; ++i) {
    const double a = x1[i][0], b = x1[i][1], c = x0[i][0], d = x0[i][1];
    A[i][0] = a * c; A[i][1] = a * d; A[i][2] = a;
    A[i][3] = b * c; A[i][4] = b * d; A[i][5] = b;
    A[i][6] = c;     A[i][7] = d;     A[i][8] = 1.0;
  }
  int perm[9];
  for (int j = 0; j < 9; ++j) perm[j] = j;
  for (int k = 0; k < 5; ++k) {
    int pr = k, pc = k;
    double best = -1.0;
    for (int i = k; i < 5; ++i)
      for (int j = k; j < 9; ++j)
        if (fabs(A[i][j]) > best) { best = fabs(A[i][j]); pr = i; pc = j; }
    if (best < 1e-13) return 0;  // degenerate sample
    if (pr != k)
      for (int j = 0; j < 9; ++j) { const double t = A[k][j]; A[k][j] = A[pr][j]; A[pr][j] = t; }
    if (pc != k) {
      for (int i = 0; i < 5; ++i) { const double t = A[i][k]; A[i][k] = A[i][pc]; A[i][pc] = t; }
      const int t = perm[k]; perm[k] = perm[pc]; perm[pc] = t;
    }
    const double inv = 1.0 / A[k][k];
    for (int j = 0; j < 9; ++j) A[k][j] *= inv;
    for (int i = 0; i < 5; ++i)
      if (i != k) {
        const double f = A[i][k];
        if (f != 0.0)
          for (int j = 0; j < 9; ++j) A[i][j] -= f * A[k][j];
      }
  }
  // basis vectors: for free column f (5..8): v[perm[f]] = 1, v[perm[k]] = -A[k][f]
  double N[4][9];
  for (int f = 0; f < 4; ++f) {
    for (int j = 0; j < 9; ++j) N[f][j] = 0.0;
    N[f][perm[5 + f]] = 1.0;
    for (int k = 0; k < 5; ++k) N[f][perm[k]] = -A[k][5 + f];
  }
  // modified Gram-Schmidt for conditioning
  for (int f = 0; f < 4; ++f) {
    for (int g = 0; g < f; ++g) {
      double dd = 0.0;
      for (int j = 0; j < 9; ++j) dd += N[f][j] * N[g][j];
      for (int j = 0; j < 9; ++j) N[f][j] -= dd * N[g][j];
    }
    double nn = 0.0;
    for (int j = 0; j < 9; ++j) nn += N[f][j] * N[f][j];
    nn = 1.0 / sqrt(nn);
    for (int j = 0; j < 9; ++j) N[f][j] *= nn;
  }
  // E(x,y,z) = x N0 + y N1 + z N2 + N3 ; entry e of E is the linear form L[e][0..3] over (x,y,z,1)

  // monomial bookkeeping. degree-1 index: x,y,z,1 = 0..3.
  // degree<=2 monomials (10): x2 y2 z2 xy xz yz x y z 1
  // degree<=3 monomials (20), Nister's elimination order:
  //   x3 y3 x2y xy2 x2z x2 y2z y2 xyz xy | xz2 xz x yz2 yz y z3 z2 z 1
  // t12[a][b]: index of (deg-1 a)*(deg-1 b) among the degree<=2 set; t23[a][b]: (deg<=2 a)*(deg-1 b)
  const int t12[4][4] = {{0, 3, 4, 6}, {3, 1, 5, 7}, {4, 5, 2, 8}, {6, 7, 8, 9}};
  const int t23[10][4] = {{0, 2, 4, 5}, {3, 1, 6, 7}, {10, 13, 16, 17}, {2, 3, 8, 9}, {4, 8, 10, 11}, {8, 6, 13, 14}, {5, 9, 11, 12}, {9, 7, 14, 15}, {11, 14, 17, 18}, {12, 15, 18, 19}};
  // L[e][v]: coefficient of variable v (x,y,z,1) in entry e
  // EEt[i][j] (quadratic, 10 coeffs), symmetric
  double EEt[3][3][10];
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) {
      double q[10];
      for (int m = 0; m < 10; ++m) q[m] = 0.0;
      for (int k = 0; k < 3; ++k)
        for (int a = 0; a < 4; ++a) {
          const double la = N[a][3 * i + k];
          for (int b = 0; b < 4; ++b) q[t12[a][b]] += la * N[b][3 * j + k];
        }
      for (int m = 0; m < 10; ++m) { EEt[i][j][m] = q[m]; EEt[j][i][m] = q[m]; }
    }
  // Lambda = EEt - 0.5 trace(EEt) I
  double tr[10];
  for (int m = 0; m < 10; ++m) tr[m] = 0.5 * (EEt[0][0][m] + EEt[1][1][m] + EEt[2][2][m]);
  for (int i = 0; i < 3; ++i)
    for (int m = 0; m < 10; ++m) EEt[i][i][m] -= tr[m];
  double M[10][20];
  for (int r = 0; r < 10; ++r)
    for (int m = 0; m < 20; ++m) M[r][m] = 0.0;
  // rows 0..8: (Lambda E)[i][j] = sum_k Lambda[i][k] E[k][j]
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double* row = M[3 * i + j];
      for (int k = 0; k < 3; ++k)
        for (int a = 0; a < 10; ++a) {
          const double la = EEt[i][k][a];
          if (la == 0.0) continue;
          for (int b = 0; b < 4; ++b) row[t23[a][b]] += la * N[b][3 * k + j];
        }
    }
  // row 9: det(E) = E00 (E11 E22 - E12 E21) - E01 (E10 E22 - E12 E20) + E02 (E10 E21 - E11 E20)
  {
    const int mn[3][2][2] = {{{4, 8}, {5, 7}}, {{3, 8}, {5, 6}}, {{3, 7}, {4, 6}}};
    const double sg[3] = {1.0, -1.0, 1.0};
    for (int c = 0; c < 3; ++c) {
      double q[10];
      for (int m = 0; m < 10; ++m) q[m] = 0.0;
      for (int a = 0; a < 4; ++a)
        for (int b = 0; b < 4; ++b)
          q[t12[a][b]] += N[a][mn[c][0][0]] * N[b][mn[c][0][1]] - N[a][mn[c][1][0]] * N[b][mn[c][1][1]];
      for (int a = 0; a < 10; ++a)
        for (int b = 0; b < 4; ++b) M[9][t23[a][b]] += sg[c] * q[a] * N[b][c];
    }
  }
  // ---- Gauss-Jordan on the first 10 columns (partial pivoting)
  for (int k = 0; k < 10; ++k) {
    int pr = k;
    double best = fabs(M[k][k]);
    for (int i = k + 1; i < 10; ++i)
      if (fabs(M[i][k]) > best) { best = fabs(M[i][k]); pr = i; }
    if (best < 1e-14) return 0;
    if (pr != k)
      for (int j = 0; j < 20; ++j) { const double t = M[k][j]; M[k][j] = M[pr][j]; M[pr][j] = t; }
    const double inv = 1.0 / M[k][k];
    for (int j = k; j < 20; ++j) M[k][j] *= inv;
    for (int i = 0; i < 10; ++i)
      if (i != k) {
        const double f = M[i][k];
        if (f != 0.0)
          for (int j = k; j < 20; ++j) M[i][j] -= f * M[k][j];
      }
  }
  // rows e..j = 4..9 ; tails live in columns 10..19 = [xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1]
  // B(z) rows: k = e - z f, l = g - z h, m = i - z j ; columns: x-poly (deg 3), y-poly (deg 3), 1-poly (deg 4)
  double Bm[3][3][5];  // coefficients in ascending powers of z
  for (int r = 0; r < 3; ++r) {
    const double* p = &M[4 + 2 * r][10];  // e, g, i
    const double* q = &M[5 + 2 * r][10];  // f, h, j
    // x-poly: -q0 z^3 + (p0 - q1) z^2 + (p1 - q2) z + p2
    Bm[r][0][0] = p[2]; Bm[r][0][1] = p[1] - q[2]; Bm[r][0][2] = p[0] - q[1]; Bm[r][0][3] = -q[0]; Bm[r][0][4] = 0.0;
    Bm[r][1][0] = p[5]; Bm[r][1][1] = p[4] - q[5]; Bm[r][1][2] = p[3] - q[4]; Bm[r][1][3] = -q[3]; Bm[r][1][4] = 0.0;
    Bm[r][2][0] = p[9]; Bm[r][2][1] = p[8] - q[9]; Bm[r][2][2] = p[7] - q[8]; Bm[r][2][3] = p[6] - q[7]; Bm[r][2][4] = -q[6];
  }
  // det B(z): degree 10
  double poly[11];
  for (int i = 0; i <= 10; ++i) poly[i] = 0.0;
  {
    const int perm3[6][3] = {{0, 1, 2}, {1, 2, 0}, {2, 0, 1}, {0, 2, 1}, {1, 0, 2}, {2, 1, 0}};
    const double sgn[6] = {1, 1, 1, -1, -1, -1};
    for (int s = 0; s < 6; ++s) {
      const double* a = Bm[0][perm3[s][0]];
      const double* b = Bm[1][perm3[s][1]];
      const double* c = Bm[2][perm3[s][2]];
      double ab[9];
      for (int i = 0; i < 9; ++i) ab[i] = 0.0;
      for (int i = 0; i < 5; ++i)
        for (int j = 0; j < 5; ++j) ab[i + j] += a[i] * b[j];
      for (int i = 0; i < 9; ++i)
        for (int j = 0; j < 5; ++j)
          if (i + j <= 10) poly[i + j] += sgn[s] * ab[i] * c[j];
    }
  }
  double roots[10];
  const int nr = poly_real_roots(poly, 10, roots);
  int nsol = 0;
  for (int r = 0; r < nr; ++r) {
    const double z = roots[r];
    double b[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) b[i][j] = poly_eval(Bm[i][j], 4, z);
    // solve [b00 b01; b10 b11][x y]^T = -[b02 b12]^T using the best conditioned row pair
    double bestdet = 0.0, x = 0.0, y = 0.0;
    for (int r0 = 0; r0 < 3; ++r0)
      for (int r1 = r0 + 1; r1 < 3; ++r1) {
        const double dd = b[r0][0] * b[r1][1] - b[r0][1] * b[r1][0];
        if (fabs(dd) > fabs(bestdet)) {
          bestdet = dd;
          x = (-b[r0][2] * b[r1][1] + b[r0][1] * b[r1][2]) / dd;
          y = (-b[r0][0] * b[r1][2] + b[r0][2] * b[r1][0]) / dd;
        }
      }
    if (bestdet == 0.0) continue;
    double nn = 0.0;
    double* Eo = Eout[nsol];
    for (int j = 0; j < 9; ++j) {
      Eo[j] = x * N[0][j] + y * N[1][j] + z * N[2][j] + N[3][j];
      nn += Eo[j] * Eo[j];
    }
    if (!(nn > 0.0) || !(nn < 1e300)) continue;
    nn = 1.0 / sqrt(nn);
    for (int j = 0; j < 9; ++j) Eo[j] *= nn;
    ++nsol;
  }
  return nsol;
}

// ------------------------------------------------------------------------------------------------
// P3P: 3 points X (reference frame) with unit bearing vectors f (camera frame), X_cam = R X + t.
// Eliminates the depth ratios u = s2/s1, v = s3/s1 to a quartic in v. Up to 4 solutions.
// ------------------------------------------------------------------------------------------------
MFR_HDN inline int p3p(const double (*X)[3], const double (*f)[3], double (*Rout)[9], double (*tout)[3]) {
  double d12[3], d13[3], d23[3];
  for (int k = 0; k < 3; ++k) {
    d12[k] = X[0][k] - X[1][k];
    d13[k] = X[0][k] - X[2][k];
    d23[k] = X[1][k] - X[2][k];
  }
  const double a2 = dot3(d23, d23), b2 = dot3(d13, d13), c2 = dot3(d12, d12);
  if (a2 < 1e-20 || b2 < 1e-20 || c2 < 1e-20) return 0;
  const double ca = dot3(f[1], f[2]), cb = dot3(f[0], f[2]), cg = dot3(f[0], f[1]);
  // (E1) b2 (u^2 + v^2 - 2 u v ca) - a2 (1 + v^2 - 2 v cb) = 0
  // (E2) b2 (1 + u^2 - 2 u cg)    - c2 (1 + v^2 - 2 v cb) = 0
  // (E1)-(E2) is linear in u:  u * D(v) = Nn(v)
  //   D(v)  = 2 b2 (cg - v ca)
  //   Nn(v) = (a2 - c2)(1 + v^2 - 2 v cb) - b2 (v^2 - 1)
  const double D[2] = {2.0 * b2 * cg, -2.0 * b2 * ca};
  const double q[3] = {1.0, -2.0 * cb, 1.0};  // 1 + v^2 - 2 v cb (ascending)
  const double Nn[3] = {(a2 - c2) * q[0] + b2, (a2 - c2) * q[1], (a2 - c2) * q[2] - b2};
  // quartic: b2 (D^2 + Nn^2 - 2 cg Nn D) - c2 q D^2 = 0
  double D2[3] = {D[0] * D[0], 2.0 * D[0] * D[1], D[1] * D[1]};
  double N2[5] = {0, 0, 0, 0, 0}, ND[4] = {0, 0, 0, 0}, qD2[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      N2[i + j] += Nn[i] * Nn[j];
      qD2[i + j] += q[i] * D2[j];
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 2; ++j) ND[i + j] += Nn[i] * D[j];
  double poly[5];
  for (int i = 0; i < 5; ++i) {
    poly[i] = b2 * N2[i] - c2 * qD2[i];
    if (i < 3) poly[i] += b2 * D2[i];
    if (i < 4) poly[i] -= 2.0 * b2 * cg * ND[i];
  }
  double roots[4];
  const int nr = poly_real_roots(poly, 4, roots);
  int nsol = 0;
  for (int r = 0; r < nr; ++r) {
    const double v = roots[r];
    if (!(v > 0.0)) continue;
    const double Dv = D[0] + D[1] * v;
    if (fabs(Dv) < 1e-14) continue;
    const double u = (Nn[0] + Nn[1] * v + Nn[2] * v * v) / Dv;
    if (!(u > 0.0)) continue;
    const double den = 1.0 + v * v - 2.0 * v * cb;
    if (!(den > 0.0)) continue;
    const double s1 = sqrt(b2 / den), s2 = u * s1, s3 = v * s1;
    // camera-frame points and rigid alignment from two orthonormal frames
    double Y[3][3];
    for (int k = 0; k < 3; ++k) { Y[0][k] = s1 * f[0][k]; Y[1][k] = s2 * f[1][k]; Y[2][k] = s3 * f[2][k]; }
    double ex[3], ey[3], ez[3], gx[3], gy[3], gz[3], tmp[3];
    for (int k = 0; k < 3; ++k) { ex[k] = X[1][k] - X[0][k]; tmp[k] = X[2][k] - X[0][k]; }
    double n = norm3(ex);
    for (int k = 0; k < 3; ++k) ex[k] /= n;
    cross3(ex, tmp, ez);
    n = norm3(ez);
    if (n < 1e-14) continue;
    for (int k = 0; k < 3; ++k) ez[k] /= n;
    cross3(ez, ex, ey);
    for (int k = 0; k < 3; ++k) { gx[k] = Y[1][k] - Y[0][k]; tmp[k] = Y[2][k] - Y[0][k]; }
    n = norm3(gx);
    if (n < 1e-14) continue;
    for (int k = 0; k < 3; ++k) gx[k] /= n;
    cross3(gx, tmp, gz);
    n = norm3(gz);
    if (n < 1e-14) continue;
    for (int k = 0; k < 3; ++k) gz[k] /= n;
    cross3(gz, gx, gy);
    double* R = Rout[nsol];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[3 * i + j] = gx[i] * ex[j] + gy[i] * ey[j] + gz[i] * ez[j];
    double RX[3];
    mat3_vec(R, X[0], RX);
    for (int k = 0; k < 3; ++k) tout[nsol][k] = Y[0][k] - RX[k];
    ++nsol;
  }
  return nsol;
}

// squared Sampson distance of a normalised correspondence under x1^T E x0 = 0
MFR_HD double sampson_sq(const double* E, double x0, double y0, double x1, double y1) {
  const double Ex0 = E[0] * x0 + E[1] * y0 + E[2];
  const double Ex1 = E[3] * x0 + E[4] * y0 + E[5];
  const double Ex2 = E[6] * x0 + E[7] * y0 + E[8];
  const double Et0 = E[0] * x1 + E[3] * y1 + E[6];
  const double Et1 = E[1] * x1 + E[4] * y1 + E[7];
  const double num = x1 * Ex0 + y1 * Ex1 + Ex2;
  const double den = Ex0 * Ex0 + Ex1 * Ex1 + Et0 * Et0 + Et1 * Et1;
  return num * num / den;
}

// ------------------------------------------------------------------------------------------------
// MAGSAC++ loss (Barath et al., CVPR 2020; the objective of cv.findEssentialMat(USAC_MAGSAC)) of a residual with
// nu = 4 degrees of freedom, the Sampson distance r in normalised coordinates, with sigma = sigma_max (the normalised
// RANSAC threshold). With x = r^2 / (2 sigma^2), x_k = k^2 / 2, G_k = Gamma(1.5, x_k) and C = 1 / (2^(nu/2) Gamma(nu/2)):
//   rho(r) = (C 2^2.5 / sigma) [sigma^2 / 2 gamma(2.5, x) + r^2 / 4 (Gamma(1.5, x) - G_k)]
//          = C 2^1.5 sigma [gamma(2.5, x) + x (Gamma(1.5, x) - G_k)]                 for r < k sigma, rho(k sigma) beyond
//   w(r)   = rho'(r) / r = (C 2^1.5 / sigma) (Gamma(1.5, x) - G_k)                  for r < k sigma, 0 beyond
// Closed forms: Gamma(1.5, x) = sqrt(x) e^-x + sqrt(pi)/2 erfc(sqrt(x)),
//               gamma(2.5, x) = 3 sqrt(pi)/4 erf(sqrt(x)) - sqrt(x) e^-x (x + 1.5).
// ------------------------------------------------------------------------------------------------
constexpr double kMagsacK = 3.64;                          // 0.99 quantile of chi_4 (3.6437), as OpenCV's USAC has it
constexpr double kMagsacXk = 0.5 * kMagsacK * kMagsacK;    // 6.6248
constexpr double kMagsacGk = 0.0036572608340910780;        // Gamma(1.5, x_k)
constexpr double kMagsacG25k = 1.3012265540498873;         // gamma(2.5, x_k)
constexpr double kMagsacC2 = 0.70710678118654752;          // C 2^1.5 with C = 0.25
constexpr double kHalfSqrtPi = 0.88622692545275801;        // sqrt(pi) / 2 = Gamma(1.5)
constexpr double kThreeQuarterSqrtPi = 1.3293403881791370; // 3 sqrt(pi) / 4 = Gamma(2.5)

// fp64 rho and w of a residual given as r^2. gamma(2.5, x) comes from its power series below x = 1, where the closed
// form loses digits to cancellation (x^2.5 against 1.5 sqrt(x)).
MFR_HD void magsac_loss_sq(double r2, double sigma, double* rho, double* w) {
  const double x = r2 / (2.0 * sigma * sigma);
  if (!(x < kMagsacXk)) {
    *rho = kMagsacC2 * sigma * kMagsacG25k;
    *w = 0.0;
    return;
  }
  const double sx = sqrt(x), e = exp(-x);
  const double G15 = sx * e + kHalfSqrtPi * erfc(sx);
  double g25;
  if (x < 1.0) {   // gamma(a, x) = x^a e^-x sum_n x^n / (a (a + 1) ... (a + n)); 18 terms reach 1e-17 at x < 1
    double term = 1.0 / 2.5, sum = term;
    for (int n = 1; n < 18; ++n) {
      term *= x / (2.5 + n);
      sum += term;
    }
    g25 = x * x * sx * e * sum;
  } else {
    g25 = kThreeQuarterSqrtPi * erf(sx) - sx * e * (x + 1.5);
  }
  *rho = kMagsacC2 * sigma * (g25 + x * (G15 - kMagsacGk));
  *w = kMagsacC2 / sigma * (G15 - kMagsacGk);
}

// fp32 rho / (C 2^1.5 sigma) of a residual at x = r^2 / (2 sigma^2), for the hypothesis scoring: one erfc and one exp
// per point. With erf = 1 - erfc the two closed forms combine to
//   gamma(2.5, x) + x (Gamma(1.5, x) - G_k) = 3 sqrt(pi)/4 (1 - erfc) - 1.5 sqrt(x) e^-x + x (sqrt(pi)/2 erfc - G_k).
MFR_HD float magsac_rho_unit_f(float x) {
  if (!(x < static_cast<float>(kMagsacXk))) return static_cast<float>(kMagsacG25k);
  const float sx = sqrtf(x), ec = erfcf(sx);
  const float e = expf(-x);
  return fmaf(x, fmaf(static_cast<float>(kHalfSqrtPi), ec, -static_cast<float>(kMagsacGk)),
              fmaf(static_cast<float>(kThreeQuarterSqrtPi), 1.0f - ec, -1.5f * sx * e));
}

// ------------------------------------------------------------------------------------------------
// RANSAC stopping rule of the solver plugins (pose_solver.required_hypotheses and _SolverBase._satisfied), branch for
// branch in fp64: the number of minimal samples after which an all-inlier sample has been drawn with probability
// `confidence`, given the inlier ratio found, capped at 2^31 - 1.
// ------------------------------------------------------------------------------------------------
MFR_HD long long ransac_required_hypotheses(double confidence, double inlier_ratio, int sample_size) {
  const double w = pow(fmin(fmax(inlier_ratio, 0.0), 1.0), static_cast<double>(sample_size));
  if (w >= 1.0 - 1e-12) return 1;
  const double c = fmin(fmax(confidence, 0.0), 1.0 - 1e-12);
  if (w < 1e-15) return 2147483647LL;   // no consensus at all: no finite budget reaches the confidence
  const double k = w < 1e-8 ? log(1.0 - c) / -w : log(1.0 - c) / log1p(-w);
  return static_cast<long long>(fmin(2147483647.0, ceil(k)));
}

// Whether a solve at `budget` hypotheses that found n_inliers of n_points stops the escalation. Nothing found
// (n <= 0) stops it only at the cap `max_budget` (the NaN pose stands then).
MFR_HD bool ransac_satisfied(double confidence, int n_inliers, int n_points, int budget, int max_budget,
                             int sample_size) {
  if (n_points <= 0 || n_inliers <= 0) return n_points <= 0 || budget >= max_budget;
  return budget >= ransac_required_hypotheses(confidence, static_cast<double>(n_inliers) / n_points, sample_size);
}

}  // namespace geo
}  // namespace mfr
