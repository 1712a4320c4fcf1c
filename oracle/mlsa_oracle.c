/* mlsa_oracle.c -- TEST INFRASTRUCTURE (oracle): CPU restatement of the MLSA noise-shaping filter the reference applies
 * through pysptk (reference wavenet_vocoder/bin/noise_shaping.py:28-43 `pysptk.mc2b`, :57-87
 * `pysptk.synthesis.Synthesizer(pysptk.synthesis.MLSADF(order, alpha), hopsize).synthesis(x, tiled_coef)`).
 *
 * pysptk (requirements: `pysptk>=0.1.17`, reference setup.py) is a Cython wrapper of SPTK 3.11 and is NOT part of
 * the reference or a dependency here, so this file restates the PUBLISHED algorithm of SPTK's `mc2b` and `mlsadf`
 * (Imai, Sumita, Furuichi: "Mel log spectrum approximation (MLSA) filter for speech synthesis", 1983; SPTK reference
 * manual, commands mc2b / mlsadf): a cascade of two Pade approximants (order pd = 4 or 5) of exp(), the first over the
 * b[1] basic filter, the second over the FIR part b[2..m] on a chain of first-order all-pass sections, and pysptk's
 * Synthesizer loop: per sample, `mlsadf(x * exp(b[0]), b)` with b interpolated linearly between frames (constant
 * here: the reference tiles one coefficient vector over all frames).
 *
 * PARITY UNPINNED against pysptk itself (it cannot be imported here); what pins this restatement is the filter's
 * defining property, checked in tests/test_mlsa_oracle.py: its frequency response equals exp(sum_m c_m e^{-j m w~})
 * on the alpha-warped axis to the accuracy of the Pade approximant, and filtering with -coef inverts filtering with coef.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU leg may use this file.  Compiled without FMA contraction
 * (-ffp-contract=off): the operation order below is the contract the CUDA kernel reproduces bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const double kPade[] = {1.0,
                               1.0, 0.0,
                               1.0, 0.0, 0.0,
                               1.0, 0.0, 0.0, 0.0,
                               1.0, 0.4999273, 0.1067005, 0.01170221, 0.0005656279,
                               1.0, 0.4999391, 0.1107098, 0.01369984, 0.0009564853, 0.00003041721};

/* SPTK mc2b: mel-cepstrum -> MLSA filter coefficients */
void mlsa_mc2b(const double* mc, double* b, int m, double a) {
  b[m] = mc[m];
  for (m--; m >= 0; m--) b[m] = mc[m] - a * b[m + 1];
}

static double mlsafir(double x, const double* b, int m, double a, double* d) {
  double y = 0.0, aa = 1 - a * a;
  int i;
  d[0] = x;
  d[1] = aa * d[0] + a * d[1];
  for (i = 2; i <= m; i++) {
    d[i] = d[i] + a * (d[i + 1] - d[i - 1]);
    y += d[i] * b[i];
  }
  for (i = m + 1; i > 1; i--) d[i] = d[i - 1];
  return y;
}

static double mlsadf1(double x, const double* b, double a, int pd, double* d, const double* ppade) {
  double v, out = 0.0, *pt, aa = 1 - a * a;
  int i;
  pt = &d[pd + 1];
  for (i = pd; i >= 1; i--) {
    d[i] = aa * pt[i - 1] + a * d[i];
    pt[i] = d[i] * b[1];
    v = pt[i] * ppade[i];
    x += (1 & i) ? v : -v;
    out += v;
  }
  pt[0] = x;
  out += x;
  return out;
}

static double mlsadf2(double x, const double* b, int m, double a, int pd, double* d, const double* ppade) {
  double v, out = 0.0, *pt;
  int i;
  pt = &d[pd * (m + 2)];
  for (i = pd; i >= 1; i--) {
    pt[i] = mlsafir(pt[i - 1], b, m, a, &d[(i - 1) * (m + 2)]);
    v = pt[i] * ppade[i];
    x += (1 & i) ? v : -v;
    out += v;
  }
  pt[0] = x;
  out += x;
  return out;
}

/* delay line length of one filter instance: 3 (pd + 1) + pd (m + 2) doubles */
int mlsa_delay_len(int m, int pd) { return 3 * (pd + 1) + pd * (m + 2); }

double mlsa_mlsadf(double x, const double* b, int m, double a, int pd, double* d) {
  const double* ppade = &kPade[pd * (pd + 1) / 2];
  x = mlsadf1(x, b, a, pd, d, ppade);
  x = mlsadf2(x, b, m, a, pd, &d[2 * (pd + 1)], ppade);
  return x;
}

/* pysptk Synthesizer.synthesis with one coefficient row per frame (nframes x (m+1)), hop samples per frame, linear
 * interpolation from the previous frame's row to the current one inside a frame.  gain[s] = exp(b0 of sample s) comes
 * from the caller: pysptk's loop is Python and takes numpy's exp, which is not glibc's exp to the last bit, so the Python
 * front end evaluates it (mlsa_oracle.py) and this file never calls exp().  delay: mlsa_delay_len doubles, zeroed by the
 * caller for a fresh filter (the reference keeps ONE filter object per worker process, so its state runs on from file to
 * file: pass the same buffer again to reproduce that).  Returns the number of samples written. */
long mlsa_synthesis(const double* x, long n, const double* coef, long nframes, int m, double a, int pd, int hop,
                    const double* gain, double* delay, double* y) {
  double* cur = (double*)malloc(sizeof(double) * (size_t)(m + 1) * 2);
  double* slope = cur + (m + 1);
  long done = 0;
  for (long f = 0; f < nframes; f++) {
    const double* prev = coef + (size_t)(f > 0 ? f - 1 : 0) * (m + 1);
    const double* curr = coef + (size_t)f * (m + 1);
    long s0 = f * hop, s1 = s0 + hop;
    if (s0 >= n) break;
    if (s1 > n) s1 = n;
    for (int k = 0; k <= m; k++) { cur[k] = prev[k]; slope[k] = (curr[k] - prev[k]) / (double)hop; }
    for (long s = s0; s < s1; s++) {
      y[s] = mlsa_mlsadf(x[s] * gain[s], cur, m, a, pd, delay);
      for (int k = 0; k <= m; k++) cur[k] += slope[k];
    }
    done = s1;
  }
  free(cur);
  return done;
}

/* the reference's time-invariant use: every frame carries the same row; gain = exp(b[0]) from the caller (see above) */
void mlsa_filter_const(const double* x, long n, const double* b, int m, double a, int pd, double gain, double* delay,
                       double* y) {
  for (long s = 0; s < n; s++) y[s] = mlsa_mlsadf(x[s] * gain, b, m, a, pd, delay);
}

/* numpy's float64 -> int16 cast (`np.int16(x_ns)`, noise_shaping.py:87): truncation toward zero, wrap modulo 2^16 */
void mlsa_to_int16(const double* y, long n, int16_t* out) {
  for (long s = 0; s < n; s++) out[s] = (int16_t)(long long)y[s];
}
