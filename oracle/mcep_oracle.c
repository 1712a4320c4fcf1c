/* mcep_oracle.c -- TEST INFRASTRUCTURE (oracle): CPU restatement of the mel-cepstral analysis the reference runs
 * through pysptk (reference wavenet_vocoder/bin/feature_extract.py:33-52 `stft_mcep`: one
 * `pysptk.mcep(frame, mcep_dim, mcep_alpha, eps=1e-10, etype=1)` per periodic-Hamming-windowed frame).
 *
 * pysptk is a Cython wrapper of SPTK 3.11 and is NOT part of the reference or a dependency here, so this file restates
 * the PUBLISHED algorithm of SPTK's `mcep` (Fukada, Tokuda, Kobayashi, Imai: "An adaptive algorithm for mel-cepstral
 * analysis of speech", ICASSP 1992; Tokuda, Kobayashi, Masuko, Imai: "Mel-generalized cepstral analysis -- a unified
 * approach to speech spectral estimation", ICSLP 1994; SPTK reference manual, command mcep): the mel-cepstrum c[0..M] on
 * the alpha-warped axis (z~^-1 = (z^-1 - a) / (1 - a z^-1), warped frequency w~(w) = w + 2 atan(a sin w / (1 - a cos w)))
 * that minimises the unbiased log-spectrum criterion
 *     E(c) = sum_k [ P_k / |H_k|^2 - log(P_k / |H_k|^2) - 1 ],   log|H_k|^2 = 2 sum_m c_m cos(m w~_k),
 * over the L bins of the frame's periodogram P, by Newton-Raphson.  Its stationarity condition is
 *     r(m) = (1/L) sum_k (P_k / |H_k|^2) cos(m w~_k) = (-a)^m,   m = 0 .. M,
 * and its Hessian is 2 L (T + H) with T_ij = r(|i-j|), H_ij = r(i+j): a Toeplitz-plus-Hankel matrix.
 *
 * The steps (itype 0: windowed frame in, etype 1: eps added to the periodogram):
 *   1. P_k = |X_k|^2 + eps for the L-point DFT X of the frame (eps > 0, so P > 0 and no zero check is needed);
 *   2. the real cepstrum of log P: c_n = (1/L) Re DFT(log P)_n, then c[0] and c[L/2] halved (log|H| = sum c_n cos n w);
 *   3. mc = freqt(c[0 .. L/2], M, a): the initial value; s = c[0] (of the halved cepstrum) seeds the convergence test;
 *   4. for j = 1, 2, ...: logH_k = Re DFT(freqt(mc, L/2, -a))_k;  R_k = P_k / exp(logH_k + logH_k);
 *      rho_n = (1/L) Re DFT(R)_n;  r = frqtr(rho[0 .. L/2], 2M, a);  t = r[0];
 *      if j >= miniter: stat_j = |(t - s) / t|; converged if stat_j < threshold (stop BEFORE update j); else s = t;
 *      solve (T + H) d = r[0 .. M] - (-a)^(0 .. M);  mc += d;
 *   5. stop after maxiter updates.
 * Choices this restatement makes (each is stated because it is not pinned against SPTK's source):
 *   - convergence statistic: |(r0_j - s) / r0_j| with s the r0 of the previous checked iteration, initialised to the
 *     halved cepstrum's c[0]; the check runs from iteration miniter on;
 *   - the update is the full Newton step d above (SPTK moves r[0] between its Toeplitz and Hankel halves before `theq`;
 *     T + H is the same matrix);
 *   - the solve is an LL^T Cholesky factorisation of T + H in column order, sums in ascending index; it FAILS when a
 *     pivot A_jj - sum_k L_jk^2 is below min_det (SPTK's theq applies min_det to its own recursion's quantity; the
 *     Hessian of the convex criterion is positive definite, and no pivot of a normal frame comes near 1e-6);
 *   - at maxiter the coefficients after the maxiter-th update are returned (SPTK returns them with code -1; pysptk
 *     does not raise for it); a failed solve returns -j (the iteration) and the caller raises, as pysptk raises on
 *     theq's failure.
 * The returned count is the number of updates applied: j - 1 when the test at iteration j converges, else maxiter.
 * force >= 0 runs exactly `force` updates with no convergence exit (statistics are still recorded), so a frame can be
 * recomputed at any iteration count.
 *
 * PARITY UNPINNED against pysptk itself (it cannot be imported here).  What pins this restatement is what mel-cepstral
 * analysis IS, checked in tests/test_mcep_oracle.py with direct numpy cosines, independent of freqt, frqtr and the
 * solve: exact recovery of a c* whose spectrum the frame carries, the stationarity condition above at the returned c,
 * E(c +- h e_m) > E(c), digital silence, the gain law of c[0], and a comparison with pysptk when it is importable.
 *
 * Only tests/, __graft_entry__.smoke() and tools/ may use this file.  Compiled without FMA contraction
 * (-ffp-contract=off).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* in-place forward DFT (e^{-2 pi i n k / n}) of length n = 2^p: bit reversal, then radix-2 butterflies */
static void fft(double* re, double* im, int n) {
  for (int i = 1, j = 0; i < n; i++) {
    int bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) {
      double t = re[i]; re[i] = re[j]; re[j] = t;
      t = im[i]; im[i] = im[j]; im[j] = t;
    }
  }
  const double pi = 3.14159265358979323846;
  for (int len = 2; len <= n; len <<= 1) {
    const int h = len >> 1;
    for (int k = 0; k < h; k++) {
      const double ang = -2.0 * pi * (double)k / (double)len;
      const double wr = cos(ang), wi = sin(ang);
      for (int i = 0; i < n; i += len) {
        const double br = re[i + k + h], bi = im[i + k + h];
        const double tr = br * wr - bi * wi, ti = br * wi + bi * wr;
        re[i + k + h] = re[i + k] - tr;
        im[i + k + h] = im[i + k] - ti;
        re[i + k] += tr;
        im[i + k] += ti;
      }
    }
  }
}

/* SPTK freqt: c1[0..m1] (one-sided cepstrum) -> c2[0..m2] on the axis warped by a (Oppenheim's recursion) */
void mcep_freqt(const double* c1, int m1, double* c2, int m2, double a) {
  double* g = (double*)calloc((size_t)(m2 + 1) * 2, sizeof(double));
  double* d = g + (m2 + 1);
  const double b = 1 - a * a;
  for (int i = -m1; i <= 0; i++) {
    memcpy(d, g, sizeof(double) * (size_t)(m2 + 1));
    g[0] = c1[-i] + a * d[0];
    if (m2 >= 1) g[1] = b * d[0] + a * d[1];
    for (int j = 2; j <= m2; j++) g[j] = d[j - 1] + a * (d[j] - g[j - 1]);
  }
  memcpy(c2, g, sizeof(double) * (size_t)(m2 + 1));
  free(g);
}

/* SPTK frqtr: rho[0..m1] (one side of a real symmetric sequence) -> r[0..m2], r(j) = (1/L) sum_k R_k cos(j w~_k) */
void mcep_frqtr(const double* c1, int m1, double* c2, int m2, double a) {
  double* g = (double*)calloc((size_t)(m2 + 1) * 2, sizeof(double));
  double* d = g + (m2 + 1);
  for (int i = -m1; i <= 0; i++) {
    memcpy(d, g, sizeof(double) * (size_t)(m2 + 1));
    g[0] = c1[-i];
    for (int j = 1; j <= m2; j++) g[j] = d[j - 1] + a * (d[j] - g[j - 1]);
  }
  memcpy(c2, g, sizeof(double) * (size_t)(m2 + 1));
  free(g);
}

/* Cholesky solve of the n x n symmetric A (row-major, overwritten by L) for x (b is kept); 0, or -1 on a pivot below
 * min_det */
static int chol_solve(double* A, const double* b, double* x, int n, double min_det) {
  for (int j = 0; j < n; j++) {
    double s = A[j * n + j];
    for (int k = 0; k < j; k++) s -= A[j * n + k] * A[j * n + k];
    if (!(s >= min_det)) return -1;
    const double ljj = sqrt(s);
    A[j * n + j] = ljj;
    for (int i = j + 1; i < n; i++) {
      double v = A[i * n + j];
      for (int k = 0; k < j; k++) v -= A[i * n + k] * A[j * n + k];
      A[i * n + j] = v / ljj;
    }
  }
  for (int i = 0; i < n; i++) {
    double v = b[i];
    for (int k = 0; k < i; k++) v -= A[i * n + k] * x[k];
    x[i] = v / A[i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    double v = x[i];
    for (int k = i + 1; k < n; k++) v -= A[k * n + i] * x[k];
    x[i] = v / A[i * n + i];
  }
  return 0;
}

/* the initial value alone (steps 1-3): mc[0..M] and the halved cepstrum's c[0] in *s0 */
static void initial_value(const double* xw, int L, int M, double a, double eps, double* P, double* re, double* im,
                          double* mc, double* s0) {
  for (int i = 0; i < L; i++) { re[i] = xw[i]; im[i] = 0.0; }
  fft(re, im, L);
  for (int i = 0; i < L; i++) P[i] = re[i] * re[i] + im[i] * im[i] + eps;
  for (int i = 0; i < L; i++) { re[i] = log(P[i]); im[i] = 0.0; }
  fft(re, im, L);
  for (int i = 0; i < L; i++) re[i] /= L;
  re[0] /= 2.0;
  re[L / 2] /= 2.0;
  mcep_freqt(re, L / 2, mc, M, a);
  *s0 = re[0];
}

/* one frame xw[0..L) (already windowed), L = 2^p >= 2: mc[0..M]; stats[j] (j = 0 .. max(maxiter, force)) gets the
 * convergence statistic of iteration j (NAN where none was computed); returns the number of updates applied, or -j when
 * the solve of iteration j fails.  force < 0: the convergence test decides; force >= 0: exactly force updates. */
int mcep_frame(const double* xw, int L, int M, double a, int miniter, int maxiter, double threshold, double eps,
               double min_det, int force, double* mc, double* stats) {
  const int n = M + 1, jmax = force >= 0 ? force : maxiter;
  double* P = (double*)malloc(sizeof(double) * (size_t)(4 * L + 6 * n + 2 * M + 1 + n * n));
  double* re = P + L;
  double* im = re + L;
  double* R = im + L;
  double* al = R + L;
  double* rr = al + n;
  double* b = rr + 2 * M + 1;
  double* d = b + n;
  double* A = d + n;
  double s;
  for (int j = 0; j <= jmax; j++) stats[j] = NAN;
  initial_value(xw, L, M, a, eps, P, re, im, mc, &s);
  al[0] = 1.0;
  for (int i = 1; i <= M; i++) al[i] = -a * al[i - 1];
  int ret = jmax;
  for (int j = 1; j <= jmax; j++) {
    for (int i = 0; i < L; i++) { re[i] = 0.0; im[i] = 0.0; }
    mcep_freqt(mc, M, re, L / 2, -a);
    fft(re, im, L);
    for (int i = 0; i < L; i++) { R[i] = P[i] / exp(re[i] + re[i]); }
    for (int i = 0; i < L; i++) { re[i] = R[i]; im[i] = 0.0; }
    fft(re, im, L);
    for (int i = 0; i <= L / 2; i++) re[i] /= L;
    mcep_frqtr(re, L / 2, rr, 2 * M, a);
    const double t = rr[0];
    if (j >= miniter) {
      stats[j] = fabs((t - s) / t);
      if (force < 0 && stats[j] < threshold) { ret = j - 1; break; }
      s = t;
    }
    for (int i = 0; i < n; i++) {
      b[i] = rr[i] - al[i];
      for (int k = 0; k < n; k++) A[i * n + k] = rr[abs(i - k)] + rr[i + k];
    }
    if (chol_solve(A, b, d, n, min_det)) { ret = -j; break; }
    for (int i = 0; i < n; i++) mc[i] += d[i];
  }
  free(P);
  return ret;
}

/* steps 1-3 only: the initial value mc[0..M] and the seed s of the convergence test */
void mcep_initial(const double* xw, int L, int M, double a, double eps, double* mc, double* s0) {
  double* P = (double*)malloc(sizeof(double) * (size_t)(3 * L));
  initial_value(xw, L, M, a, eps, P, P + L, P + 2 * L, mc, s0);
  free(P);
}
