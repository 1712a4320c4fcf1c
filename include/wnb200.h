/*
 * wnb200.h -- C ABI of libwnb200.so, the H100 (sm_90a) kernels behind the WaveNet vocoder hot paths.
 *
 * The reference (kan-bayashi/PytorchWaveNetVocoder v0.1.1) is pure Python on top of torch: it has no
 * FFI layer of its own (SURVEY.md 8b).  This header is therefore OUR drop-in boundary: each entry
 * point replaces one piece of reference/wavenet_vocoder/nets/wavenet.py (cited per function) and is
 * what the host-side mirror `pytorchwavenetvocoder_b200.nets.WaveNet` binds through ctypes
 * (INTEGRATION.md shows the stub a reference maintainer would add).
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless named host_*;
 *   - the caller (PyTorch) owns every buffer; nothing is allocated or freed in here;
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*) and never synchronise;
 *   - return value: 0 = WNB_OK, negative = error; wnb_last_error() gives a thread-local message;
 *   - activations are CHANNELS-LAST fp32: (B, T, C) with C contiguous (the reference is (B, C, T));
 *     `Ap` is n_aux rounded up to a multiple of 32 (zero padded);
 *   - weights arrive in the PACKED layouts documented below (built from the reference state_dict by
 *     pytorchwavenetvocoder_b200/nets/packing.py).
 *
 * Packed weight layouts (R=n_resch, S=n_skipch, Q=n_quantize, ks=kernel_size, K1 = ks*R + Ap)
 *   wf   (ks, Q, R)   wf[k][q][r]     = causal.conv.weight[r][q][k]                 (wavenet.py:189)
 *   w1   (2R, K1)     rows 0..R-1 sigmoid branch, R..2R-1 tanh branch; columns j*R+c = tap j
 *                     (j=0 oldest, x[t-(ks-1-j)d]) of dil_{sigmoid,tanh}[l].conv.weight[o][c][j],
 *                     columns ks*R+a = aux_1x1_{sigmoid,tanh}[l].weight[o][a][0] (zero for a>=A)
 *   b1   (2R)         dil bias + aux bias                                            (wavenet.py:527-532)
 *   w2   (R+S, R)     rows 0..R-1 res_1x1[l].weight, rows R.. skip_1x1[l].weight     (wavenet.py:533-534)
 *   b2   (R+S)
 *   wp1  (S, S), bp1 (S), wp2 (Q, S), bp2 (Q)                                        (wavenet.py:209-210)
 *   *_t  the same matrices transposed (K-major), used by the backward and decode kernels.
 */
#ifndef WNB200_H_
#define WNB200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define WNB_API __attribute__((visibility("default")))
#else
#define WNB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define WNB_OK 0
#define WNB_ERR_INVALID (-1)   /* bad argument / unsupported shape */
#define WNB_ERR_CUDA (-2)      /* a CUDA runtime call or launch failed */
#define WNB_ERR_UNSUPPORTED (-3)

#define WNB_MATH_FP32 0        /* SIMT FFMA, fp32 throughout (parity mode) */
#define WNB_MATH_TF32 1        /* wgmma tf32 contractions, fp32 accumulate */
/* wgmma bf16 contractions: both operands of every product rounded to bf16 (nearest even), fp32 accumulate; activations,
 * weights and gradients stay fp32 in memory (the weights a call uses are rounded into a library scratch per call).
 * Covered: wnb_resblock_fwd / wnb_resblock_bwd on the composed path's shapes (wnb_resblock_fwd_supported() == 2) and
 * wnb_post_fwd / wnb_post_bwd with S, Q multiples of 32 up to 256 (or 512); any other shape is an error.  The
 * deferred-skip stack and the fused per-block kernels are tf32 only. */
#define WNB_MATH_BF16 2

#define WNB_MODE_ARGMAX 0
#define WNB_MODE_SAMPLING 1

/* ---- library / device info -------------------------------------------------------------- */
WNB_API int wnb_version(void);
WNB_API const char* wnb_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py "gpu_launches") */
WNB_API int64_t wnb_launch_count(void);

/* ---- a1/a2: mu-law codec (wavenet.py:17-30, 33-47) -- bit exact with numpy ----------------- */
WNB_API int wnb_mulaw_encode_f32(const float* x, int64_t* y, int64_t n, int mu, void* stream);
WNB_API int wnb_mulaw_encode_f64(const double* x, int64_t* y, int64_t n, int mu, void* stream);
WNB_API int wnb_mulaw_decode_f64(const int64_t* y, double* x, int64_t n, int mu, void* stream);

/* a17 (decode driver, bin/decode.py:318-319): generated codes -> PCM_16 samples for a whole batch on the device.  The
 * input domain is the mu codes, so `table` (ntab int16, device) holds decode_mu_law + the writer's quantisation per code
 * (built by nets.mulaw_pcm16_table); out[i] = table[idx[i] mod ntab]. */
WNB_API int wnb_lut_i16(const int32_t* idx, const int16_t* table, int16_t* out, int64_t n, int ntab, void* stream);

/* ---- a4/a5/a9: OneHot + causal conv as an embedding gather (wavenet.py:78-92, 513-516) ----- */
WNB_API int wnb_front_embed_fwd(const int64_t* x /*(B,T)*/, const float* wf, const float* bias /*(R)*/,
                        float* out /*(B,T,R)*/, int B, int T, int Q, int R, int ks, void* stream);
/* dwf (ks,Q,R) and dbias (R) are ACCUMULATED into (caller zeroes) */
WNB_API int wnb_front_embed_bwd(const int64_t* x, const float* dout /*(B,T,R)*/, float* dwf, float* dbias,
                        int B, int T, int Q, int R, int ks, void* stream);

/* ---- a6: UpSampling (wavenet.py:124-154) fused with the (B,A,Tf)->(B,T,Ap) layout change ----
 * U > 0: haux[b][tU+j][a] = h[b][a][t]*w[j] + bias[0];  U == 0: plain transpose (Tf == T). */
WNB_API int wnb_aux_upsample_fwd(const float* h /*(B,A,Tf)*/, const float* w /*(U)*/, const float* bias /*(1)*/,
                         float* haux /*(B,T,Ap)*/, int B, int A, int Ap, int Tf, int U, void* stream);
/* dw (U), dbias (1) accumulated into */
WNB_API int wnb_aux_upsample_bwd(const float* h, const float* dhaux /*(B,T,Ap)*/, float* dw, float* dbias,
                         int B, int A, int Ap, int Tf, int U, void* stream);

/* ---- a10: fused residual block forward (wavenet.py:525-536), one launch per layer ----------
 * xout = res_1x1(z) + xin, skip (+)= skip_1x1(z), z = sigmoid(..)*tanh(..).
 * xout may be NULL (last layer: its residual output is discarded, wavenet.py:230-238).
 * skip_init != 0: skip = value (first layer; python `0 + s0`), else skip += value.
 * zsave (B,T,R) may be NULL; when given, z is also stored (not used by the default backward). */
WNB_API int wnb_resblock_fwd(const float* xin, const float* haux, const float* w1, const float* b1,
                     const float* w2, const float* b2, float* xout, float* skip, float* zsave,
                     int B, int T, int R, int S, int Ap, int ks, int dilation, int skip_init,
                     int math_mode, void* stream);

/* tf32: 1 = fused per-block kernel (no zsave), 2 = composed tensor-core path (zsave optional), 0 = not covered;
   bf16: 2 = composed tensor-core path (zsave optional), 0 = not covered; fp32: 1 = covered, 0 = not;
   an unknown math_mode: 0 */
WNB_API int wnb_resblock_fwd_supported(int R, int S, int Ap, int ks, int math_mode);

/* ---- a5 standalone: CausalConv1d.forward (wavenet.py:95-121), channels-last, fp32 FFMA, forward only.
 * x (B,T,Cin), w (Cout, ks*Cin) with w[o][j*Cin+c] = conv.weight[o][c][j], bias (Cout) or NULL, out (B,T,Cout). */
WNB_API int wnb_causal_conv1d_fwd(const float* x, const float* w, const float* bias, float* out, int B, int T,
                                  int Cin, int Cout, int ks, int dilation, void* stream);

/* ---- a18 / f1: train_generator on the device (bin/train.py:67-312) ------------------------------------------------
 * One launch cuts a whole mini-batch out of device-resident RING buffers: `wave` (cap_s floats) = the concatenated
 * float32 waveforms, `feat` (cap_f rows of D, float32 or float64 as read from the feature file) = the concatenated
 * feature frames; positions are absolute stream positions, ring index = position mod capacity.  Window b starts at
 * sample s0 + b*hop: x[b][i] = encode_mu_law(wave[..+i]), t[b][i] = encode_mu_law(wave[..+i+1]) (bit exact with
 * wnb_mulaw_encode_f32); h[b][d][j] = float32 StandardScaler transform ((v - mean[d]) / scale[d] with sklearn's dtype
 * behaviour; mean == NULL: none) of frame (s0 + b*hop)/U + j (up-sampling layer: Tf = T/U, frame_of_sample NULL) or of
 * frame frame_of_sample[sample] (extend_time mode: Tf = T; an int32 ring parallel to `wave`).
 * feat_f64: 1 = float64 rows; 0 = float32 rows, scaler in float64 arithmetic rounded to float32 after each step
 * (scikit-learn 0.22, the reference's pin); 2 = float32 rows, scaler in float32 arithmetic (scikit-learn >= 1.x).
 * x, t (B,T) int64; h (B,D,Tf) fp32. */
WNB_API int wnb_make_train_batch(const float* wave, const void* feat, const int32_t* frame_of_sample, int64_t s0,
                                 int64_t hop, int U, int64_t cap_s, int64_t cap_f, const double* mean, const double* scale,
                                 int64_t* x, int64_t* t, float* h, int B, int T, int Tf, int D, int feat_f64, int mu,
                                 void* stream);

/* ---- the same batch cut from a device-resident corpus (utils/corpus.py, utils/device_loader.DeviceCorpusGenerator) ---
 * `wave` (int16) and `feat` (rows of D, layout and feat_f64 as above) hold every utterance once, trimmed to whole frames.
 * The stream of concatenated utterances in epoch order is a table of the n_utts non-empty utterances it covers:
 * starts[k] = stream position of the utterance's first sample (strictly increasing), offsets[k] = its first sample in
 * `wave` (a multiple of U; its first frame is row offsets[k] / U).  Stream position p maps to the utterance k with the
 * largest starts[k] <= p (binary search), sample offsets[k] + p - starts[k].  [table_begin, table_end) is the part of the
 * stream the table covers; every window must lie in it.  x[b][i] = encode_mu_law(sample / 32768) of position
 * s0 + b*hop + i, t the next sample, h[b][d][j] = the scaled row of stream frame (s0 + b*hop)/U + j (up-sampling layer). */
WNB_API int wnb_make_train_batch_corpus(const int16_t* wave, const void* feat, const int64_t* starts, const int64_t* offsets,
                                        int n_utts, int64_t table_begin, int64_t table_end, int64_t s0, int64_t hop, int U,
                                        const double* mean, const double* scale, int64_t* x, int64_t* t, float* h, int B,
                                        int T, int Tf, int D, int feat_f64, int mu, void* stream);

/* ---- a12: the optimizer step (bin/train.py:457-460, :539 torch.optim.Adam) as one kernel over flat buffers ----------
 * p, g, m, v: parameters, gradients (the flat buffer wnb_pack_weights' backward direction fills), first and second moment
 * estimates, n floats each, 16-byte aligned, identical layout.  torch's (fused) Adam arithmetic in fp32: g += weight_decay*p;
 * m += (1-beta1)(g-m); v = beta2 v + (1-beta2) g^2; p -= lr/bias_correction1 * m / (sqrt(v)/sqrt(bias_correction2) + eps)
 * with bias_correction_i = 1 - beta_i^step supplied by the caller (step counted from 1); the scalar hyper-parameters are
 * doubles, combined in double and rounded to float once, as torch does. */
WNB_API int wnb_adam_flat(float* p, const float* g, float* m, float* v, int64_t n, double lr, double beta1, double beta2,
                          double eps, double weight_decay, double bias_correction1, double bias_correction2, void* stream);

/* ---- f4: MLSA noise-shaping filter for a batch of utterances (bin/noise_shaping.py:46-87: pysptk
 * Synthesizer(MLSADF(order, alpha), hopsize).synthesis(x, tiled coefficients), i.e. per sample SPTK
 * mlsadf(x * exp(coef[0]), coef, order, alpha, pd) with a time-invariant coefficient vector) -------------------------
 * x: the utterances concatenated, int16 (x_is_i16 = 1: the wav samples, converted like np.float64(x)) or float64;
 * offsets (n_utts + 1 int64, device): utterance u is [offsets[u], offsets[u+1]); coef (order + 1 float64, device) =
 * pysptk.mc2b output (pass -coef for the inverse filter, noise_shaping.py:55-56); pd = Pade order 4 (pysptk's default) or
 * 5; gain = exp(coef[0]) computed by the caller; y: same layout as x, float64 or int16 (y_is_i16 = 1: truncation toward
 * zero like np.int16(y), noise_shaping.py:87).  fp64 arithmetic in SPTK's operation order without FMA contraction;
 * every utterance starts from a zero filter state (the reference lets the state of one file run on into the next file of
 * the same worker process). */
WNB_API int wnb_mlsa_filter(const void* x, int x_is_i16, const long long* offsets, int n_utts, const double* coef, int order,
                            double alpha, int pd, double gain, void* y, int y_is_i16, void* stream);

/* Resumable MLSA filtering: wnb_mlsa_filter over n_segs segments, each carrying its filter state from one call to the
 * next, so that a signal filtered in consecutive chunks gives, bit for bit, what one call over the whole signal gives.
 *   states      caller-owned device table of n_slots slots of wnb_mlsa_state_doubles(order, pd) doubles each; slot s
 *               at states + s * wnb_mlsa_state_doubles(order, pd), laid out as d1[1..pd], pt1[0..pd], pt20,
 *               pt[1..pd] (each Pade stage's previous output), then stage k's all-pass chain e[1..order] for
 *               k = 1..pd (SPTK mlsadf's recursion state in the kernel's form, csrc/mlsa.cu).
 *   slots       host int32 array of n_segs: segment u loads slot slots[u] and stores into it the state after its own last
 *               sample (an empty segment leaves its slot unchanged).  The slots are distinct, 0 <= slots[u] < n_slots.
 *   zero_start  host int32 array of n_segs or NULL: segment u with zero_start[u] != 0 starts from a zero state instead
 *               of loading its slot (a new signal in a reused slot).
 * Everything else as wnb_mlsa_filter; 1 <= n_segs <= WNB_MLSA_MAX_STATE_SEGMENTS.  WNB_ERR_INVALID for a bad shape,
 * pointer or slot, before any device work.  wnb_mlsa_state_doubles returns 0 for an order or pd wnb_mlsa_filter rejects. */
#define WNB_MLSA_MAX_STATE_SEGMENTS 1024
WNB_API size_t wnb_mlsa_state_doubles(int order, int pd);
WNB_API int wnb_mlsa_filter_state(const void* x, int x_is_i16, const long long* offsets, int n_segs, const double* coef,
                                  int order, double alpha, int pd, double gain, void* y, int y_is_i16, double* states,
                                  int n_slots, const int32_t* slots, const int32_t* zero_start, void* stream);

/* ---- f5: mel-spectrogram features for a batch of utterances (bin/feature_extract.py --feature_type melspc:
 * low_cut_filter, then librosa.feature.melspectrogram(x / 32768, power=1.0, center=True) and log10(max(1e-10, .)))
 * in float64 throughout, one float32 rounding at the end; fixed operation order, no atomics: two runs are bit-identical.
 *
 * wnb_melspc_lowcut: the low-cut FIR of every utterance, y[n] = sum_{k < n_taps} taps[k] x[n - k] with x[< 0] = 0
 * (scipy lfilter(taps, 1, x)), one fma chain in ascending k per output sample.
 *   x        the utterances concatenated, int16 (x_is_i16 = 1: the wav samples, converted like np.float64(x)) or float64;
 *   offsets  (n_utts + 1 int64, device): utterance u is [offsets[u], offsets[u+1]); max_len = the longest utterance;
 *   taps     (n_taps float64, device): scipy firwin(255, cutoff / (fs // 2), pass_zero=False) in the recipes;
 *   y        float64, same layout as x;  y16  NULL or int16, same layout: np.int16(y) (truncation toward zero to int32,
 *            out-of-range values giving INT_MIN, then the low 16 bits; the reference's filtered wav).
 *
 * wnb_melspc: log mel-spectrogram of every utterance.  The input is in int16 units (int16 samples, or the float64 output
 * of wnb_melspc_lowcut) and is divided by 32768.  Utterance u has n_u = offsets[u+1] - offsets[u] >= 1 samples and
 * 1 + n_u / hop frames, frames [frame_offsets[u], frame_offsets[u+1]) of out; n_frames = frame_offsets[n_utts] (the host
 * computes both tables).  Frame t reads positions [t hop, t hop + fftl) of np.pad(x, fftl / 2, mode="reflect"), times
 * `window` (fftl float64: scipy get_window("hann", fftl)), real FFT (radix-2 Stockham, float64, `twiddles` = fftl / 2
 * pairs (cos, -sin)(2 pi m / fftl), interleaved), S[k] = hypot(Re, Im) for k <= fftl / 2, then for each mel filter m
 * E = sum_{mel_lo[m] <= k < mel_hi[m]} (double)mel_basis[m][k] S[k] in ascending k (mel_basis (n_mels, fftl / 2 + 1)
 * float32, the filters' nonzero ranges in mel_lo / mel_hi, int32), out[frame][m] = (float)log10(max(1e-10, E)).
 * fftl must be a power of two in [WNB_MELSPC_MIN_FFTL, WNB_MELSPC_MAX_FFTL], else WNB_ERR_UNSUPPORTED.
 *
 * Both: WNB_ERR_INVALID for a bad shape or pointer, before any device work. */
#define WNB_MELSPC_MAX_TAPS 1024
#define WNB_MELSPC_MIN_FFTL 64
#define WNB_MELSPC_MAX_FFTL 4096
WNB_API int wnb_melspc_lowcut(const void* x, int x_is_i16, const long long* offsets, int n_utts, long long max_len,
                              const double* taps, int n_taps, double* y, int16_t* y16, void* stream);
WNB_API int wnb_melspc(const void* x, int x_is_i16, const long long* offsets, const long long* frame_offsets, int n_utts,
                       long long n_frames, int fftl, int hop, const double* window, const double* twiddles,
                       const float* mel_basis, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, float* out,
                       void* stream);

/* ---- f7: streaming mel-spectrogram.  wnb_melspc_stream advances n_segs keyed signals by one chunk each and writes every
 * frame no later sample can change; concatenated, a signal's frames equal wnb_melspc (after wnb_melspc_lowcut when
 * n_taps > 0) of the whole signal bit for bit, whatever the chunking.  Frame t reads signal indices
 * [t hop - fftl / 2, t hop + fftl / 2) through the reflect map of the signal's length; the host decides which frames
 * are final and which filtered samples to keep (utils/melspc.py melspc_frames_ready, melspc_carry_start).
 *   states   device table of n_slots slots of wnb_melspc_stream_state_doubles(fftl, n_taps) doubles: the last
 *            n_taps - 1 input samples (FIR history), then the carry, filtered samples [carry start, n) of a signal that
 *            has had n samples (at most fftl - 1).
 *   segs     host table of n_segs rows of WNB_MELSPC_SEG_FIELDS int64, and segs_dev, the same table in device memory
 *            (the kernels read segs_dev; the library validates segs):
 *              SLOT      the slot; distinct within a call.
 *              FLAGS     NEW: exactly when N_BEFORE = 0 (zero history, no carry); STORE: store the new state (a key
 *                        that does not end with this chunk and has samples in it).
 *              X_OFF, X_LEN  the chunk, x[X_OFF, X_OFF + X_LEN) (int16 when x_is_i16, else float64, int16 units).
 *              N_BEFORE  samples the key had before this chunk;  CARRY0  the carry's start index before it.
 *              SCRATCH   offset of the segment's scratch region (doubles): [old carry | filtered chunk | new history
 *                        when STORE], N_BEFORE - CARRY0 + X_LEN (+ n_taps - 1) doubles.
 *              R0, R1    frames [R0, R1) to write, rows OUT_ROW .. OUT_ROW + R1 - R0 of out; OUT_ROW is the running sum
 *                        of R1 - R0 over the previous segments, n_frames the total.
 *              CARRY1    the carry's new start index (STORE).
 *   out      (n_frames, n_mels) float32 raw features.  aux NULL or float32: segment u's frames scaled,
 *            (x - mean) / scale, transposed to (n_mels, R1 - R0) at aux + OUT_ROW n_mels.  scaler_mode 0: float64
 *            subtract, round to float32, float64 divide, round; 2: float32 subtract and divide with mean and scale
 *            rounded to float32 (StandardScaler.transform of float32 features, scikit-learn 0.22 and >= 1.x).
 * Two launches (the first reads slots and writes scratch, the second reads scratch and writes frames and slots, so no
 * block reads a slot another block of the call has stored), none when no segment has frames or state to store; no host
 * synchronisation, no atomics.  WNB_ERR_INVALID for a bad table or pointer, WNB_ERR_UNSUPPORTED for an fftl wnb_melspc
 * rejects, both before any device work.  wnb_melspc_stream_state_doubles returns 0 for such an fftl or n_taps outside
 * [0, WNB_MELSPC_MAX_TAPS]. */
#define WNB_MELSPC_MAX_STREAM_SEGMENTS 1024
#define WNB_MELSPC_SEG_SLOT 0
#define WNB_MELSPC_SEG_FLAGS 1
#define WNB_MELSPC_SEG_X_OFF 2
#define WNB_MELSPC_SEG_X_LEN 3
#define WNB_MELSPC_SEG_N_BEFORE 4
#define WNB_MELSPC_SEG_CARRY0 5
#define WNB_MELSPC_SEG_SCRATCH 6
#define WNB_MELSPC_SEG_R0 7
#define WNB_MELSPC_SEG_R1 8
#define WNB_MELSPC_SEG_OUT_ROW 9
#define WNB_MELSPC_SEG_CARRY1 10
#define WNB_MELSPC_SEG_FIELDS 11
#define WNB_MELSPC_SEG_NEW 1
#define WNB_MELSPC_SEG_STORE 2
WNB_API size_t wnb_melspc_stream_state_doubles(int fftl, int n_taps);
WNB_API int wnb_melspc_stream(const void* x, int x_is_i16, int n_segs, const long long* segs, const long long* segs_dev,
                              long long n_frames, int fftl, int hop, const double* taps, int n_taps,
                              const double* window, const double* twiddles, const float* mel_basis,
                              const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, double* states, int n_slots,
                              double* scratch, long long scratch_doubles, float* out, const double* mean,
                              const double* scale, int scaler_mode, float* aux, void* stream);

/* ---- f6: STFT mel-cepstra for a batch of utterances (bin/feature_extract.py --feature_type mcep: stft_mcep, then
 * pysptk.mcep(frame, order, alpha, eps=1e-10, etype=1) per frame) in float64 throughout, one float32 rounding at the end;
 * fixed operation order, no atomics: two runs are bit-identical.
 *
 * wnb_mcep: the input is in int16 units (int16 samples, or the float64 output of wnb_melspc_lowcut), NOT divided by
 * 32768.  Utterance u has n_u = offsets[u+1] - offsets[u] >= fftl samples and (n_u - fftl) / hop + 1 frames, frames
 * [frame_offsets[u], frame_offsets[u+1]) of out; n_frames = frame_offsets[n_utts] (the host computes both tables).
 * Frame t is x[t hop, t hop + fftl) (no padding) times `window` (fftl float64: scipy get_window("hamming", fftl)), real
 * FFT (the Stockham FFT of wnb_melspc, same `twiddles` layout), P_k = |X_k|^2 + eps for k <= fftl / 2, then SPTK mcep's
 * Newton-Raphson for the mel-cepstrum of order `order` on the axis warped by alpha, every warp a sum over the bins:
 *   warp_cos      (fftl / 2 + 1 float64): cos w~_k, w~_k = w_k + 2 atan(alpha sin w_k / (1 - alpha cos w_k)),
 *                 w_k = 2 pi k / fftl;
 *   init_map      ((order + 2) x (fftl / 2 + 1) float64): rows 0 .. order map log P to SPTK's initial value (real
 *                 cepstrum of log P, c[0] and c[fftl/2] halved, freqt to the order); row order + 1 gives the halved
 *                 c[0] that seeds the convergence test;
 *   neg_alpha_pow (order + 1 float64): (-alpha)^m.
 * From iteration miniter on, |(r0 - s) / r0| < threshold (r0 the zeroth warped autocorrelation of P / |H|^2, s the
 * previous checked r0) stops before that iteration's update; at most maxiter updates.  out[frame][m] = (float)c_m,
 * iters[frame] = the number of updates applied, or -j when iteration j's Cholesky pivot falls below min_det.
 * Supported: fftl a power of two in [WNB_MCEP_MIN_FFTL, WNB_MCEP_MAX_FFTL], 1 <= order <= WNB_MCEP_MAX_ORDER,
 * 0 <= alpha <= WNB_MCEP_MAX_ALPHA (there the bin sums equal SPTK's truncated recursions to 1e-13), else
 * WNB_ERR_UNSUPPORTED.  WNB_ERR_INVALID for a bad shape or pointer, before any device work. */
#define WNB_MCEP_MIN_FFTL 1024
#define WNB_MCEP_MAX_FFTL 4096
#define WNB_MCEP_MAX_ORDER 40
#define WNB_MCEP_MAX_ALPHA 0.6
#define WNB_MCEP_MAX_ITER 1000
WNB_API int wnb_mcep(const void* x, int x_is_i16, const long long* offsets, const long long* frame_offsets, int n_utts,
                     long long n_frames, int fftl, int hop, int order, double alpha, const double* window,
                     const double* twiddles, const double* warp_cos, const double* init_map,
                     const double* neg_alpha_pow, int miniter, int maxiter, double threshold, double eps,
                     double min_det, float* out, int32_t* iters, void* stream);

/* ---- pack_weights: state_dict layout <-> kernel layout as one launch per direction (SURVEY.md 8b) ----------
 * A table of strided 3-D copies dst[i0*ds0 + i1*ds1 + i2*ds2] = scale * f(src[i0*ss0 + i1*ss1 + i2*ss2]) executed by
 * one kernel (one block row per entry).  `src` / `src2` are absolute device pointers (WNB_PACK_SRC_ABS: the
 * reference-shaped nn.Parameters of wavenet.py:188-210) or element offsets from `src_base`; `dst` is an element
 * offset from `dst_base`.  Ops: COPY; ADD2 = src + src2 (dilated-conv bias + aux bias, wavenet.py:527-532);
 * SUMPTR = sum over a device table (at `src`) of `nsum` equally shaped tensors (the summed skip biases).
 * Forward: parameters -> packed buffer (layouts above, plus the transposes the backward wants).  Backward: packed
 * gradient buffer -> one flat buffer holding every parameter's .grad, scaled by the device scalar `scale` (NULL = 1). */
#define WNB_PACK_COPY 0
#define WNB_PACK_ADD2 1
#define WNB_PACK_SUMPTR 2
#define WNB_PACK_SRC_ABS 1
typedef struct WnbPackDesc {
  int64_t src, src2, dst;
  int32_t n0, n1, n2;
  int32_t ss0, ss1, ss2;
  int32_t ds0, ds1, ds2;
  int32_t op, flags, nsum;
} WnbPackDesc;
WNB_API int wnb_pack_weights(const WnbPackDesc* descs /*device*/, int ndesc, const float* src_base, float* dst_base,
                             const float* scale /*device scalar or NULL*/, void* stream);
/* cudaMemsetAsync(p, 0, bytes) on `stream`: gradient accumulators the kernels add into */
WNB_API int wnb_zero(void* p, size_t bytes, void* stream);

/* ---- per-launch timing of the stack kernels (measurement aid for bench.py's roofline block) ----
 * While enabled, wnb_stack_fwd / wnb_stack_bwd bracket every kernel launch with CUDA events on the launching stream;
 * wnb_profile_read() waits for them and returns the summed duration and launch count of one kind since the last
 * wnb_profile_enable().  Single-threaded use. */
#define WNB_PROF_FWD_BLOCK 0   /* resblock_fwd_z: one residual block, deferred-skip form */
#define WNB_PROF_SKIP_GEMM 1   /* skip = Z_all Wskip^T */
#define WNB_PROF_DZALL_GEMM 2  /* dZ_all = dskip Wskip */
#define WNB_PROF_GATE_BWD 3    /* the stack backward's block chain: last gate backward, dx_l + gate backward of block l-1, dx_0 */
#define WNB_PROF_DX_GEMM 4     /* dx (+ dhaux) (no longer launched on its own: part of WNB_PROF_GATE_BWD) */
#define WNB_PROF_DW1 5         /* dW1, db1 (no longer launched on its own: part of WNB_PROF_WGRAD) */
#define WNB_PROF_DW2RES 6      /* dW2res, db2res (part of WNB_PROF_WGRAD) */
#define WNB_PROF_DWSKIP 7      /* dWskip, dbskip (part of WNB_PROF_WGRAD) */
#define WNB_PROF_WGRAD 8       /* every weight gradient of the stack (dW1, dW2res, dWskip + biases): one launch + reduce */
#define WNB_PROF_KINDS 9
WNB_API int wnb_profile_enable(int on);
WNB_API int wnb_profile_read(int kind, double* total_ms, int* launches);

/* The static work split of the weight-gradient kernel (a host function; no device needed): problem i has stages[i]
 * stages of cost[i] each, cut into nchunk[i] time chunks of ceil(stages / nchunk) stages (one CTA sums a chunk from
 * zero, so the chunks fix the summation order); lock[i] != 0 marks problems that share operands through L2, whose chunks
 * run side by side.  CTA j (of sms) runs the pieces cta_first[j] .. cta_first[j+1]-1; piece q is the stages
 * pieces[3q+1] .. pieces[3q+2]-1 of problem pieces[3q].  Returns the number of pieces (pieces may be NULL to count
 * them), or WNB_ERR_INVALID (bad input, or more than max_pieces). */
WNB_API int wnb_wgrad_partition(const int* stages, const int* nchunk, const double* cost, const int* lock, int nprob,
                                int sms, int* cta_first, int* pieces, int max_pieces);
/* How the consumer threads of the weight-gradient kernel transpose the nB (1..7) B sub-tiles of one tf32 stage (a host
 * function; no device needed): one row of 10 ints per 4 x 4 unit, {thread, iteration, 4 load offsets from the first B
 * sub-tile, 4 store offsets into the transposed tile}, in bytes; load i holds time row i of the unit's 4 channels, store
 * j channel j of its 4 time rows.  map holds 640 nB ints.  Returns the number of units (64 nB) or WNB_ERR_INVALID. */
WNB_API int wnb_wgrad_transpose_map(int nB, int* map);

/* ---- residual stack in deferred-skip form (training path of WaveNet.forward, wavenet.py:229-236 over :525-536) ----
 * The skip sum over all L blocks is one GEMM over the concatenated gate outputs,
 *     skip = [z_0 | ... | z_{L-1}] Wskip^T + bskip,   Wskip[s][l*R+c] = skip_1x1_l.weight[s][c],  bskip = sum_l skip bias_l
 * so a block only writes z_l into Z_all (B,T,L*R) and its residual output (no read-modify-write of skip per block),
 * and the backward hoists dZ_all = dskip Wskip and dWskip = dskip^T Z_all out of the block loop the same way.
 * WNB_MATH_TF32 only (0 for any other math_mode); wnb_stack_supported() says whether the shape is covered (else use the
 * per-block entries). */
WNB_API int wnb_stack_supported(int R, int S, int Ap, int ks, int L, int math_mode);

/* one block: xout (B,T,R) = xin + res_1x1(z) (NULL for the last block), z -> zall[:, :, zcol0:zcol0+R] (row pitch ldz).
 * w1 (2R,K1), b1 (2R) as for wnb_resblock_fwd; w2res (R,R) = res_1x1.weight[o][c], b2res (R). */
WNB_API int wnb_resblock_fwd_z(const float* xin, const float* haux, const float* w1, const float* b1,
                               const float* w2res, const float* b2res, float* xout, float* zall, int ldz, int zcol0,
                               int B, int T, int R, int Ap, int ks, int dilation, void* stream);

/* skip (B,T,S) = zall (B,T,K) wskip^T + bskip (relu != 0: rectified, the form wnb_post_fwd consumes);
 * wskip (S,K) row-major, bskip (S) or NULL */
WNB_API int wnb_skip_gemm(const float* zall, const float* wskip, const float* bskip, float* skip, int B, int T,
                          int K, int S, int relu, void* stream);

/* whole stack: xs (nxs,B,T,R) holds the block inputs, xs[0] filled by the caller (wnb_front_embed_fwd); block l reads
 * xs[l % nxs] and writes xs[(l+1) % nxs] (nxs = L keeps every input for the backward, nxs = 2 ping-pongs).
 * w1 (L,2R,K1), b1 (L,2R), w2res (L,R,R), b2res (L,R), wskip (S,L*R), bskip (S); dilations: L host ints.
 * Outputs zall (B,T,L*R) and skip (B,T,S) (rectified when skip_relu != 0). */
WNB_API int wnb_stack_fwd(float* xs, int nxs, const float* haux, const float* w1, const float* b1,
                          const float* w2res, const float* b2res, const float* wskip, const float* bskip,
                          float* zall, float* skip, const int* dilations, int L, int B, int T, int R, int S,
                          int Ap, int ks, int skip_relu, void* stream);

/* backward of wnb_stack_fwd.  xs (L,B,T,R) and zall from the forward; dskip (B,T,S) = d loss / d skip.
 * w1t (L,K1,2R) as for wnb_resblock_bwd; wgate (L,3R,K1+R) = block matrix [[w1, 0], [0, w2res^T]] per block (gate
 * recompute and the residual part of dz share one GEMM); wskip_t (L*R,S) = wskip^T.
 * dx0 (B,T,R) = gradient of xs[0]; dhaux (B,T,Ap) accumulated into (or NULL); dw1, db1, dw2res, db2res, dwskip
 * (S,L*R), dbskip (S) are ACCUMULATED into (the last block's dw2res / db2res are left untouched: that conv has no
 * gradient, like the reference).  workspace: wnb_stack_bwd_workspace() bytes. */
WNB_API size_t wnb_stack_bwd_workspace(int L, int B, int T, int R, int S, int Ap, int ks);
WNB_API int wnb_stack_bwd(const float* xs, const float* haux, const float* zall, const float* dskip, const float* w1,
                          const float* b1, const float* w1t, const float* wgate, const float* wskip_t, float* dx0,
                          float* dhaux, float* dw1, float* db1, float* dw2res, float* db2res, float* dwskip,
                          float* dbskip, void* workspace, const int* dilations, int L, int B, int T, int R, int S,
                          int Ap, int ks, void* stream);

/* ---- a10 backward --------------------------------------------------------------------------
 * Recomputes the gate from xin/haux, then produces dxin and accumulates weight gradients.
 * dout = d(loss)/d(xout) (NULL for the last layer), dskip = d(loss)/d(skip_sum) (same for all layers).
 * dhaux (B,T,Ap) accumulated into (NULL when the aux path has no trainable producer).
 * dw1 (2R,K1), db1 (2R), dw2 (R+S,R), db2 (R+S) are ACCUMULATED into.
 * w1t = (ks+1 blocks) transposed W1: block j<ks is (R, 2R): w1t[j][c][o] = w1[o][j*R+c];
 *        block ks is (Ap, 2R): w1[o][ks*R+a];  w2t (R, R+S): w2t[c][o] = w2[o][c].
 * workspace: wnb_resblock_bwd_workspace() bytes. */
WNB_API size_t wnb_resblock_bwd_workspace(int B, int T, int R, int S, int Ap, int ks);
WNB_API int wnb_resblock_bwd(const float* xin, const float* haux, const float* dout, const float* dskip,
                     const float* w1, const float* b1, const float* w1t, const float* w2t,
                     float* dxin, float* dhaux, float* dw1, float* db1, float* dw2, float* db2,
                     void* workspace, int B, int T, int R, int S, int Ap, int ks, int dilation,
                     int math_mode, void* stream);

/* ---- a11: post network (wavenet.py:518-523) -------------------------------------------------
 * logits (B,T,Q) = wp2 * relu(wp1 * relu(skip) + bp1) + bp2 ; r1 (B,T,S) = relu(h1) is kept (needed by the
 * backward).  With WNB_MATH_TF32 `skip` is rectified IN PLACE first (its sign pattern -- all that
 * wnb_post_bwd needs from it -- is unchanged; wnb_post_bwd in tf32 mode relies on it); skip_rectified != 0
 * (tf32 only) says the producer already did that (wnb_skip_gemm / wnb_stack_fwd with relu) and skips the pass. */
WNB_API int wnb_post_fwd(float* skip, const float* wp1, const float* bp1, const float* wp2,
                 const float* bp2, float* r1, float* logits, int B, int T, int S, int Q,
                 int math_mode, int skip_rectified, void* stream);
/* dskip (B,T,S) out; dwp1,dbp1,dwp2,dbp2 accumulated into; workspace (B,T,S) floats */
WNB_API int wnb_post_bwd(const float* skip, const float* r1, const float* dlogits, const float* wp1t /*(S,S) [c][o]*/,
                 const float* wp2t /*(S,Q) [c][o]*/, float* dskip, float* dwp1, float* dbp1, float* dwp2,
                 float* dbp2, float* workspace, int B, int T, int S, int Q, int math_mode, void* stream);

/* ---- a12: CrossEntropyLoss(mean) on [:, start:] fused with its gradient (bin/train.py:534-536)
 * loss_sum (1 double, accumulated into; caller zeroes) receives the MEAN loss;
 * dlogits (B,T,Q) may be NULL (loss only); rows t < start get zero gradient. */
WNB_API int wnb_cross_entropy(const float* logits, const int64_t* target /*(B,T)*/, double* loss_sum,
                      float* dlogits, int B, int T, int Q, int start, void* stream);
/* ---- held-out scoring (WaveNet.score, DESIGN.md section 6): per-row summed cross entropy, one launch, no atomics.
 * For each row b, adds -log softmax(logits[b, t])[target[b, t]] over start <= t < min(lengths[b], T) to nll[b]
 * (accumulated into; the caller zeroes it) and that number of positions to count[b] (may be NULL).  A row with
 * lengths[b] <= start is left untouched.  The value of each position is the one wnb_cross_entropy computes (its Q == 256
 * register path when logits is 16-byte aligned).  The row is summed in one order that depends on the row alone
 * (csrc/score.cu): segments [32 j, 32 j + 32) of its columns, each summed as a fixed lane tree, then added to nll[b]
 * in ascending j.  So a row's result does not depend on B, T beyond its length, the other rows or the run, and chaining
 * calls over windows whose first column is a multiple of 32 reproduces one call over the whole row bit for bit. */
WNB_API int wnb_cross_entropy_rows(const float* logits /*(B,T,Q)*/, const int64_t* target /*(B,T)*/,
                                   const int64_t* lengths /*(B)*/, int start, double* nll /*(B)*/,
                                   int64_t* count /*(B)*/, int B, int T, int Q, void* stream);

/* ---- a14/a15/a16: persistent fast-generate kernels (wavenet.py:309-395, 397-511, 538-549) ----------------------------
 * Four decoders, one entry point each: wnb_decode_at (weights read directly from L2), wnb_decode_stream_at,
 * wnb_decode_warp_at and wnb_decode_bf16_at.  One launch generates the samples of every utterance over one window of
 * padded positions, pos0 .. max(pos0, P - 1) + max_n - 1.  pos0 = xs_base = h_frame0 = 0 runs the whole range in one
 * call: the P - 1 teacher-forced warm-up positions, then every sample.  A chain of calls, each starting where the previous
 * one stopped, computes exactly what one call over the whole range computes, bit for bit, whatever the chunk boundaries,
 * so a session can decode an utterance chunk by chunk as its aux frames arrive.  The arguments the four share:
 *   P, n_pad   keep their absolute meaning: P - 1 warm-up positions, then sample i at position P - 1 + i; n_pad is the
 *              number of left-replicated aux columns (wavenet.py:334): aux at padded position p is h_up[max(p - n_pad, 0)];
 *   pos0       0 (the first call: it runs the whole warm-up) or >= P - 1.  A call generates at least one sample, so a
 *              chain never starts a call inside the warm-up; 0 < pos0 < P - 1 is rejected;
 *   i0         = max(pos0 - (P - 1), 0), the first sample index of the call;
 *   n_samples  (B) int32, the samples to generate in this call per utterance (sample indices i0 .. i0 + n_b - 1),
 *              max_n >= every n_b; the call stops after max_n samples;
 *   xs         (B, max(pos0, P - 1) + max_n + 1 - xs_base) int32: column c is absolute position xs_base + c.  The call
 *              reads positions pos0 - (ks - 1) .. (those >= 0; so xs_base <= max(pos0 - (ks - 1), 0)), which must hold the
 *              padded seed prefix (wavenet.py:330-334) or what earlier calls generated, and writes position P + i with
 *              sample i;
 *   h          (B, A, Th) aux features BEFORE upsampling (U > 0, with up_w / up_b) or at sample rate (U == 0): column c is
 *              absolute frame h_frame0 + c (aux column max(p - n_pad, 0), divided by U when U > 0); h_frame0 <= the frame
 *              of pos0.  Lookups past the last column are clamped to it;
 *   mode       WNB_MODE_*; uniforms (B, max_n) optional externally supplied U[0,1) draws (tests), else
 *              Philox4x32-10(seed, utterance, step);
 *   logits_out (B, max_n, Q) optional teacher-check output (NULL in production).  It and uniforms are indexed by the
 *              call's own sample index i - i0; the in-kernel Philox counter keeps the absolute i, so a sampled stream does
 *              not depend on the chunk boundaries;
 *   queues     the dilation queues, caller-allocated (wnb_decode_workspace() bytes, need not be zeroed; the bf16 decoder
 *              has its own size).  Between the calls of one chain the caller keeps them untouched and the same B (hence the
 *              same launch form: NU / W / CL of wnb_decode_warp_at, the utterances per CTA of wnb_decode_stream_at /
 *              wnb_decode_at, the cluster split of wnb_decode_bf16_at); the fp32 decoders never need cleared queues,
 *              wnb_decode_bf16_at clears them when pos0 == 0 only.
 * Positions are int: the last position written must stay below 2^31 - 1.  WNB_ERR_INVALID for an inconsistent window. */
WNB_API size_t wnb_decode_workspace(int B, int R, int ks, const int32_t* host_dilations, int L);

/* Decode weights of wnb_decode_at are K-major: wf (ks,Q,R), w1d (L,K1,2R), b1 (L,2R), w2d (L,R,R+S), b2 (L,R+S),
 * wp1d (S,S) [c][o], wp2d (S,Q) [c][o]. */
WNB_API int wnb_decode_at(int32_t* xs, const float* h, const float* up_w, const float* up_b,
                          const float* wf, const float* bf, const float* w1d, const float* b1, const float* w2d,
                          const float* b2, const float* wp1d, const float* bp1, const float* wp2d, const float* bp2,
                          const int32_t* host_dilations, int L, void* queues, const int32_t* n_samples,
                          const float* uniforms, float* logits_out, int B, int P, int max_n, int n_pad, int Th,
                          int Q, int A, int Ap, int R, int S, int ks, int U, int mode, uint64_t seed,
                          int pos0, int xs_base, int h_frame0, void* stream);

/* ---- a14-a16, streaming variant: same contract as wnb_decode_at, but the K-major matrices arrive as ONE
 * packed stream consumed in order every step (a producer warp pushes it through a shared-memory ring
 * with cp.async.bulk while the consumer warps run the recurrence):
 *   per layer l: W1d [K1][O1] | W2res [R][Or] | W2skip [R][Os]   then  wp1d [S][Sp] | wp2d [S][Qp]
 * with O1 = 2R, Or = R, Os = Sp = S, Qp = Q each rounded up to a multiple of 4 (zero padded).
 * Returns WNB_ERR_UNSUPPORTED when the shape does not fit, before any device work (the caller may run wnb_decode_at).
 * wnb_decode_stream_supported answers the same question without a device: 1 when covered (every padded width fits the
 * consumer threads and a 32 KB ring chunk, R, S and Ap are multiples of 4, L <= 64, and the work area of one utterance
 * plus two ring slots fits shared memory), else 0.  Whether it is covered does not depend on B. */
WNB_API size_t wnb_decode_stream_floats(int Q, int Ap, int R, int S, int ks, int L);
WNB_API int wnb_decode_stream_supported(int Q, int Ap, int R, int S, int ks, int L);
WNB_API int wnb_decode_stream_at(int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                 const float* wf, const float* bf, const float* stream, const float* b1,
                                 const float* b2, const float* bp1, const float* bp2,
                                 const int32_t* host_dilations, int L, void* queues, const int32_t* n_samples,
                                 const float* uniforms, float* logits_out, int B, int P, int max_n, int n_pad,
                                 int Th, int Q, int A, int Ap, int R, int S, int ks, int U, int mode,
                                 uint64_t seed, int pos0, int xs_base, int h_frame0, void* stream_handle);

/* ---- a14-a16, warp-tiled variant for the BASELINE shape (R 64, S 512, Q 256, Ap 32, ks 2): same contract,
 * weights as ONE stream in warp-tile order (layout documented in csrc/decode_warp.cu; built by
 * nets/wavenet.py::_decode_warp_pack).  Batches of <= 74 utterances run ONE UTTERANCE PER 2-CTA CLUSTER (CL = 2):
 * each CTA streams its half of every matrix and the two exchange their halves of every activation vector through
 * distributed shared memory; the stream then holds the two per-CTA streams back to back. */
WNB_API size_t wnb_decode_warp_floats(int L, int CL);
/* debug aid: per-phase cycle counters of the free-running steps (16 int64 per CTA; NULL = off) */
WNB_API void wnb_decode_warp_set_timing(long long* device_buf);
WNB_API int wnb_decode_warp_supported(int Q, int Ap, int R, int S, int ks, int L);
WNB_API int wnb_decode_warp_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                               const float* bf, const float* stream, const float* b1, const float* b2,
                               const float* bp1, const float* bp2, const int32_t* host_dilations, int L,
                               void* queues, const int32_t* n_samples, const float* uniforms, float* logits_out,
                               int B, int P, int max_n, int n_pad, int Th, int A, int U, int mode, uint64_t seed,
                               int W, int CL, int pos0, int xs_base, int h_frame0, void* stream_handle);
/* consumer warps (8 or 16) / CTAs per utterance (1 or 2) the launcher uses for B utterances; the stream layout depends
 * on both */
WNB_API int wnb_decode_warp_plan(int B);
WNB_API int wnb_decode_warp_cluster(int B);
/* the kernel instantiation decode_warp_kernel<NU, W, BIG, CL> that wnb_decode_warp_at runs for B utterances of L layers,
 * under the current WNB_DECODE_BIG: form[0..3] = NU (utterances per CTA), W (consumer warps), CL (CTAs per cluster),
 * BIG (1: three 64 KB ring slots, 0: up to six 32 KB slots).  WNB_ERR_UNSUPPORTED when no ring fits. */
WNB_API int wnb_decode_warp_form(int B, int L, int32_t* form);

/* ---- a14-a16, opt-in bf16 tensor-core variant for the recipe sizes (WaveNet.decode_math = "bf16"): same contract as
 * wnb_decode_stream_at (xs, pre-upsampling h with up_w / up_b, n_pad, ragged n_samples, supplied uniforms or in-kernel
 * Philox with counter (step, batch index, 0, 0), optional logits_out, xs[b][P + n_b ..] untouched), but every product
 * multiplies bf16 operands (fp32 accumulation) and the batch runs as ceil(B / 64) clusters of 8 CTAs (csrc/decode_bf16.cu).
 * `weights` is the packed bf16 stream of wnb_decode_bf16_weights() 16-bit elements (layout in csrc/decode_bf16.cu,
 * built by nets/wavenet.py::_decode_bf16_pack; the biases ride inside it); `queues` holds
 * wnb_decode_bf16_workspace() bytes and is cleared by a call with pos0 == 0.  Covered (wnb_decode_bf16_supported): Q 256,
 * ks 2 or 3, Ap <= 256, R/S 256/256, 512/256 or 512/512, L <= 64; otherwise WNB_ERR_UNSUPPORTED (no fallback). */
WNB_API int wnb_decode_bf16_supported(int Q, int Ap, int R, int S, int ks, int L);
WNB_API size_t wnb_decode_bf16_weights(int Q, int Ap, int R, int S, int ks, int L);
WNB_API size_t wnb_decode_bf16_workspace(int B, int R, int ks, const int32_t* host_dilations, int L);
WNB_API int wnb_decode_bf16_at(int32_t* xs, const float* h, const float* up_w, const float* up_b, const float* wf,
                               const float* bf, const void* weights, const int32_t* host_dilations, int L, void* queues,
                               const int32_t* n_samples, const float* uniforms, float* logits_out, int B, int P,
                               int max_n, int n_pad, int Th, int Q, int A, int Ap, int R, int S, int ks, int U, int mode,
                               uint64_t seed, int pos0, int xs_base, int h_frame0, void* stream_handle);

/* ---- the teacher-forced warm-up computed in parallel over time (csrc/decode_prefill.cu) ------------------------------
 * wnb_decode_warp_prefill writes into `queues` (the workspace of wnb_decode_warp_at, same B) exactly what
 * wnb_decode_warp_at(pos0 = 0) leaves there after the warm-up positions 0 .. P - 2, bit for bit, without running them one
 * by one; the caller then runs wnb_decode_warp_at with pos0 = P - 1, xs_base = 0, h_frame0 = 0 and the same xs, h, CL.
 * Only layer l's last S_l = (ks - 1) * (d_l + ... + d_{L-1}) warm-up positions are computed, so the cost does not depend
 * on the seed length.  Queue slots of positions < 0 are left as they are, like the sequential warm-up leaves them.
 *   xs      (B, P) int32, the padded seed prefix (columns 0 .. P - 1 of the xs of wnb_decode_warp_at);
 *   h, up_w, up_b, n_pad, Th, A, U   as for wnb_decode_warp_at (h_frame0 = 0);
 *   w1d (L,160,128), b1 (L,128), w2d (L,64,576), b2 (L,576)   the plain K-major decode weights of wnb_decode_at, 16-byte
 *           aligned (the arithmetic is fixed per element, not per layout, so the warp-tiled stream is not needed);
 *   CL      wnb_decode_warp_cluster(B): the 2-CTA form sums half of the residual products in another order;
 *   scratch wnb_decode_prefill_workspace(B, P, 64, 2, dilations, L) bytes (two fp32 copies of x_l over the largest
 *           window; 0 bytes, and scratch may be NULL, when P == 1).
 * Covers the shapes of wnb_decode_warp_supported; WNB_ERR_INVALID for a bad shape or pointer, before any device work. */
/* the pruned windows: windows[l] = S_l = (ks - 1) * (d_l + ... + d_{L-1}), the warm-up positions before P - 1 on which
 * layer l's input is needed (the prefill computes layer l's input on max(0, P - 1 - S_l) .. P - 2); WNB_ERR_INVALID for a
 * dilation < 1.  wnb_decode_prefill_workspace returns 0 for such dilations. */
WNB_API int wnb_decode_prefill_windows(const int32_t* host_dilations, int L, int ks, int64_t* windows);
WNB_API size_t wnb_decode_prefill_workspace(int B, int P, int R, int ks, const int32_t* host_dilations, int L);
WNB_API int wnb_decode_warp_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                    const float* wf, const float* bf, const float* w1d, const float* b1,
                                    const float* w2d, const float* b2, const int32_t* host_dilations, int L,
                                    void* queues, void* scratch, int B, int P, int n_pad, int Th, int A, int U, int CL,
                                    void* stream_handle);
/* wnb_decode_stream_prefill: the same for the streaming decoder (csrc/decode_stream_prefill.cu).  After the call `queues`
 * (the workspace of wnb_decode_stream_at, same B, wnb_decode_workspace() bytes) holds exactly what
 * wnb_decode_stream_at(pos0 = 0) leaves there after the warm-up positions 0 .. P - 2, bit for bit; the caller then runs
 * wnb_decode_stream_at with pos0 = P - 1, xs_base = 0, h_frame0 = 0 and the same xs, h, stream.  Slots of positions < 0
 * are left as they are.
 *   xs      (B, P) int32, the padded seed prefix;
 *   h, up_w, up_b, wf, bf, b1, b2, n_pad, Th, Q, A, Ap, R, S, ks, U   as for wnb_decode_stream_at (h_frame0 = 0);
 *   stream  the packed stream of wnb_decode_stream_at (its W1d and W2res are read), 16-byte aligned;
 *   scratch wnb_decode_prefill_workspace(min(B, 64), P, R, ks, dilations, L) bytes: batches run in groups of at most 64
 *           utterances (0 bytes, and scratch may be NULL, when P == 1 or ks == 1).
 * Launches 1 + (L - 1) kernels per group of 64.  Covers every shape of wnb_decode_stream_supported and any dilations >= 1;
 * WNB_ERR_UNSUPPORTED for another shape and WNB_ERR_INVALID for a bad shape or pointer, before any device work. */
WNB_API int wnb_decode_stream_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                      const float* wf, const float* bf, const float* stream, const float* b1,
                                      const float* b2, const int32_t* host_dilations, int L, void* queues,
                                      void* scratch, int B, int P, int n_pad, int Th, int Q, int A, int Ap, int R,
                                      int S, int ks, int U, void* stream_handle);
/* wnb_decode_bf16_prefill: the same for the bf16 decoder (csrc/decode_bf16_prefill.cu).  After the call `queues` (the
 * workspace of wnb_decode_bf16_at, same B, wnb_decode_bf16_workspace() bytes) holds exactly what wnb_decode_bf16_at(pos0 = 0)
 * leaves there after the warm-up positions 0 .. P - 2, bit for bit, padding rows of each cluster included; the caller
 * then runs wnb_decode_bf16_at with pos0 = P - 1, xs_base = 0, h_frame0 = 0 and the same xs, h, weights.  The call clears
 * the queues first, as the pos0 = 0 call does.
 *   xs      (B, P) int32, the padded seed prefix (columns 0 .. P - 1 of the xs of wnb_decode_bf16_at);
 *   h, up_w, up_b, wf, bf, weights, n_pad, Th, A, Ap, R, S, ks, U   as for wnb_decode_bf16_at (h_frame0 = 0);
 *   scratch wnb_decode_bf16_prefill_workspace(B, P, R, ks, dilations, L) bytes (x_l as fp32 and bf16 and the gate output
 *           z as bf16 over the largest window; 0 bytes, and scratch may be NULL, when P == 1).
 * WNB_ERR_INVALID for a bad shape or pointer and WNB_ERR_UNSUPPORTED for a shape outside wnb_decode_bf16_supported, both
 * before any device work.  wnb_decode_bf16_prefill_workspace returns 0 for a bad shape or a dilation < 1. */
WNB_API size_t wnb_decode_bf16_prefill_workspace(int B, int P, int R, int ks, const int32_t* host_dilations, int L);
WNB_API int wnb_decode_bf16_prefill(const int32_t* xs, const float* h, const float* up_w, const float* up_b,
                                    const float* wf, const float* bf, const void* weights,
                                    const int32_t* host_dilations, int L, void* queues, void* scratch, int B, int P,
                                    int n_pad, int Th, int A, int Ap, int R, int S, int ks, int U,
                                    void* stream_handle);

/* ---- continuous batching on the bf16 decoder (csrc/decode_bf16_pool.cu, nets/wavenet.py::DecodePool) ----------------
 * A pool of `capacity` rows runs wnb_decode_bf16_at unchanged on B = capacity with P = 1, n_pad = 0, U = 0, a global
 * step counter g as the window (pos0 = g0 >= ks - 1, xs_base = g0 - (ks - 1), h_frame0 = g0, Th = max_n = n) and its
 * queues allocated zeroed (pos0 is never 0, so the launcher never clears them).  Every row then reads queue slot
 * g mod (ks-1) d_l, xs column g, aux column g and uniform column g, and the two calls below fill those with what one-shot
 * decoding gives the stream in that row, so each stream's codes equal one-shot decoding bit for bit.
 *
 * wnb_decode_bf16_pool_transplant moves n admitted streams into the pool: row src_rows[i] of `src_queues` (a workspace
 * of wnb_decode_bf16_at for src_B utterances, after wnb_decode_bf16_prefill) goes to row dst_slots[i] of `dst_queues`
 * (the pool's workspace, B = capacity), layer l's slot s to slot (s + rotations[i]) mod (ks-1) d_l, with
 * rotations[i] = g_a - (P - 1) for a stream whose first sample is the pool's step g_a.  Every slot of the row is written.
 *   src_rows, dst_slots, rotations   host int32 arrays of n (1 <= n <= 64); the slots must be distinct.
 * WNB_ERR_INVALID for a bad shape, row, slot, dilation or pointer, before any device work.
 *
 * wnb_decode_bf16_pool_inputs writes the call's aux window and uniforms for wnb_decode_bf16_at:
 *   frames   (B, A, F) fp32, each row's aux frames as given (before up-sampling when U > 0);
 *   table    (5, B) int32 device, per row: [0] the absolute frame of frames[b][.][0], [1] the aux column of the row's
 *            first step, [2] its first sample index, [3] its stream id (the Philox counter's second word), [4] its samples
 *            in this call (0: an idle row), which is also the n_samples of wnb_decode_bf16_at;
 *   aux      (B, A, n) out: column k of row b = fmaf(frames[b][a][j / U - [0]], up_w[j % U], up_b[0]) with j = [1] + k
 *            (frames[b][a][j - [0]] when U = 0), the fp32 value the decoder computes in-kernel; 0 for k >= [4];
 *   uniforms (B, n) out, or NULL (argmax): column k = (r0 >> 8) * 2^-24 of Philox4x32-10((sample [2] + k, stream id [3],
 *            0, 0), seed), the decoder's own draw; 0 for k >= [4].
 * WNB_ERR_INVALID for a bad shape or pointer, before any device work.
 * wnb_decode_bf16_pool_inputs does not depend on the decoder: the fp32 decoders compute the same fmaf up-sampling and
 * the same draw in-kernel, and the pool on the fp32 warp decoder (below) uses it unchanged. */
WNB_API int wnb_decode_bf16_pool_transplant(const void* src_queues, int src_B, const int32_t* src_rows, void* dst_queues,
                                            int capacity, const int32_t* dst_slots, const int32_t* rotations, int n,
                                            int R, int ks, const int32_t* host_dilations, int L, void* stream_handle);
WNB_API int wnb_decode_bf16_pool_inputs(const float* frames, const float* up_w, const float* up_b, const int32_t* table,
                                        float* aux, float* uniforms, int B, int A, int F, int n, int U, uint64_t seed,
                                        void* stream_handle);

/* ---- parking pool streams (csrc/decode_bf16_park.cu, nets/wavenet.py::DecodePool with park_below) -------------------
 * A parked stream's queues live in a store of its own: [sum_l (ks-1) d_l slots][R] bf16, layer l's slots after those
 * of layers 0 .. l-1, slot s of layer l holding x_l of the stream's positions v = s mod (ks-1) d_l (the slots an
 * admission prefill leaves).  wnb_decode_bf16_park_bytes gives its size (0 for a bad shape or a dilation < 1).
 *
 * wnb_decode_bf16_pool_park copies n pool rows into stores: row slots[i] of `queues` (the pool's workspace, B =
 * capacity) goes to stores[i], layer l's row slot s to store slot (s + rotations[i]) mod (ks-1) d_l, with rotations[i] =
 * v - g for a stream whose next position v is the pool's step g.  wnb_decode_bf16_pool_unpark copies stores[i] back into
 * row slots[i], store slot s to row slot (s + rotations[i]) mod (ks-1) d_l, with rotations[i] = g' - v for a stream whose
 * next position v is to be the pool's step g'.  Both copy bit for bit and write every slot of their destination; one
 * launch per call.
 *   slots, rotations   host int32 arrays of n (1 <= n <= 64); the slots must be distinct;
 *   stores             host array of n device pointers, 16-byte aligned, park_bytes each.
 * WNB_ERR_INVALID for a bad shape, slot, dilation or pointer, before any device work. */
WNB_API size_t wnb_decode_bf16_park_bytes(int R, int ks, const int32_t* host_dilations, int L);
WNB_API int wnb_decode_bf16_pool_park(const void* queues, int capacity, const int32_t* slots, void* const* stores,
                                      const int32_t* rotations, int n, int R, int ks, const int32_t* host_dilations,
                                      int L, void* stream_handle);
WNB_API int wnb_decode_bf16_pool_unpark(const void* const* stores, void* queues, int capacity, const int32_t* slots,
                                        const int32_t* rotations, int n, int R, int ks, const int32_t* host_dilations,
                                        int L, void* stream_handle);

/* ---- continuous batching on the fp32 warp decoder (csrc/decode_pool.cu, nets/wavenet.py::DecodePool) ----------------
 * The same pool on wnb_decode_warp_at: B = capacity, P = 1, n_pad = 0, U = 0, pos0 = g0, xs_base = g0 - 1,
 * h_frame0 = g0, Th = max_n = n, W / CL of the capacity, inputs from wnb_decode_bf16_pool_inputs.  The fp32 decoders
 * read a tap of layer l only at positions >= d_l (a zero before, the causal padding), so the pool's step counter stays
 * at or above the longest queue, (ks-1) max_l d_l.  An admitted stream's warm-up runs through wnb_decode_warp_prefill
 * with the pool's CL (not the CL of the admitted group's size: the 2-CTA form sums half of the residual products in
 * another order).
 *
 * The fp32 decoders keep one utterance's queues in one contiguous block of wnb_decode_workspace(1, R, ks, dilations, L)
 * bytes, [sum_l (ks-1) d_l slots][R] fp32, slot t mod (ks-1) d_l of layer l holding x_l(t).  A pool row, a row of an
 * admission workspace and a parked stream's store all have this layout, so admission, parking and resuming are one
 * operation: wnb_decode_pool_move copies n queue blocks src[i] -> dst[i], layer l's slot s to slot
 * (s + rotations[i]) mod (ks-1) d_l, bit for bit, every slot of the destination written, one launch per call.  Admission
 * rotates by g_a - (P - 1) (the stream's first sample is the pool's step g_a), parking by v - g (its next position v is
 * the pool's step g), resuming by g' - v.
 *   src, dst   host arrays of n device pointers to one utterance's block (workspace + b * block bytes) or to a store of
 *              that size, 16-byte aligned;
 *   rotations  host int32 array of n, any sign;  1 <= n <= 64.
 * WNB_ERR_INVALID, before any device work, for a bad shape (R a multiple of 4), a dilation < 1, a null or misaligned
 * pointer, a destination given twice or one that overlaps any source (an in-place rotation would race). */
WNB_API int wnb_decode_pool_move(const void* const* src, void* const* dst, const int32_t* rotations, int n, int R,
                                 int ks, const int32_t* host_dilations, int L, void* stream_handle);

/* ---- mel-cepstral distortion between reference and decoded mel-cepstra (csrc/distortion.cu, utils/distortion.py) -----
 * Inputs are float32 frames of n_cols = D + 1 coefficients (c0 first), as wnb_mcep writes them, widened to float64 in
 * the kernels; every operation is float64 with explicit rounding (__dadd_rn, __dmul_rn, __dsqrt_rn), never an FMA.
 * Pair p is reference frames [ref_offsets[p], ref_offsets[p+1]) of `ref` and decoded frames [dec_offsets[p],
 * dec_offsets[p+1]) of `dec` (n_pairs + 1 int64 each; they need not start at 0).  The offsets are passed twice: on the
 * device for the kernel and on the host (the same values) for the launcher's checks.
 * dist(a, b) = sqrt(sum_{d=1..D} (a_d - b_d)^2), the squares added in ascending d; c0 is left out.  A frame's MCD in dB
 * is K dist with K = fl(10 / ln 10) fl(sqrt 2), applied by the caller: the kernels write sums of dist and counts.
 *
 * wnb_mcd_aligned: frames t < n = min(Tr, Td) compared index by index; sum[p] = their dists added as 32-frame chunks
 * (each chunk an xor butterfly over its 32 lanes, o = 16, 8, 4, 2, 1, frames past n counting 0.0), the chunk sums added
 * in ascending order from 0.0; count[p] = n.
 *
 * wnb_mcd_dtw: C(i, j) = dist(r_i, d_j) + min(C(i-1, j-1), C(i-1, j), C(i, j-1)), C(0, 0) = dist(r_0, d_0); row 0 and
 * column 0 follow their one predecessor; ties go to (i-1, j-1), then (i-1, j), then (i, j-1).  The path runs from
 * (0, 0) to (Tr-1, Td-1); count[p] = its length, sum[p] = C(Tr-1, Td-1), which equals the sum of dist along the path
 * added in forward order.  With `path` (optional), pair p's steps (i, j) as int32 pairs fill the first count[p] entries of
 * its slot of Tr + Td - 1 entries; slot p starts at entry (ref_offsets[p] - ref_offsets[0]) + (dec_offsets[p] -
 * dec_offsets[0]) - p.  Pair p uses wnb_mcd_dtw_workspace(Tr, Td) bytes of `workspace` (16-byte aligned) starting at the
 * sum of that size over the pairs before it: the step directions, one byte per cell laid out per strip of
 * WNB_MCD_DTW_THREADS rows, and, when Td > WNB_MCD_DTW_SMEM_COLS, a row of Td doubles.  wnb_mcd_dtw_workspace returns 0
 * for a length outside [1, WNB_MCD_MAX_FRAMES].  One CTA per pair, the grid strided over the pairs.
 *
 * Both: no allocation, no synchronisation, one launch.  WNB_ERR_UNSUPPORTED for D outside [1, WNB_MCD_MAX_DIM] (wnb_mcep's
 * orders) or a side with no frames (or more than WNB_MCD_MAX_FRAMES); WNB_ERR_INVALID for a null pointer, a misaligned
 * workspace or path, or a workspace smaller than the pairs need; all before any device work. */
#define WNB_MCD_MAX_DIM 40
#define WNB_MCD_MAX_FRAMES (1 << 24)
#define WNB_MCD_DTW_THREADS 256
#define WNB_MCD_DTW_SMEM_COLS 4096
WNB_API int wnb_mcd_aligned(const float* ref, const float* dec, int n_cols, const long long* ref_offsets,
                            const long long* dec_offsets, const long long* host_ref_offsets,
                            const long long* host_dec_offsets, int n_pairs, double* sum, int64_t* count,
                            void* stream);
WNB_API size_t wnb_mcd_dtw_workspace(long long ref_frames, long long dec_frames);
WNB_API int wnb_mcd_dtw(const float* ref, const float* dec, int n_cols, const long long* ref_offsets,
                        const long long* dec_offsets, const long long* host_ref_offsets,
                        const long long* host_dec_offsets, int n_pairs, void* workspace, size_t workspace_bytes,
                        double* sum, int64_t* count, int32_t* path, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WNB200_H_ */
