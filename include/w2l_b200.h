/*
 * w2l_b200.h — C ABI of libw2l_b200.so: the H100-native (sm_90a) implementation of
 * wav2letter's training hot path.  Every entry point below replaces one piece of the
 * un-vendored flashlight-0.3 backend that the reference's Train.cpp loop reaches through
 * fl::pkg::speech::SequenceCriterion / fl::Module (SURVEY.md §8b).  The binding a
 * maintainer adds on the reference side is shown in INTEGRATION.md; include/fl_compat/
 * holds the C++ classes with the reference's own names (ASGLoss, CTCLoss, ...) on top.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - all calls are asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant
 *     across streams, and keep no hidden state: scratch memory is a caller-owned workspace
 *     whose size the matching *_workspace_size() call returns (SURVEY.md §8b "Threading");
 *   - return value: W2L_OK or an error code; w2l_last_error() gives the thread-local text.
 *     The fl_compat C++ layer turns codes into std::invalid_argument / std::runtime_error
 *     like the reference (cpc/SequentialBuilder.cpp:107-109);
 *   - numerical failure is signalled in-band (NaN / Inf in the loss), which the caller
 *     checks exactly as Train.cpp:1686-1698 does.
 *
 * Layouts (ArrayFire column-major dims -> row-major C):
 *   emissions  af [N,T,B]  -> float  emis[B][T][N]
 *   targets    af [L,B]    -> int32  target[B][L], padded with negative values
 *                             (kTargetPadValue = -1, recipes/slimIPL/src/Train.cpp:318-322)
 *   transitions af [N,N]   -> float  trans[N][N], trans[i*N+j] = score of moving FROM j TO i
 *                             (criterion->param(0), tools/StreamingTDSModelConverter.cpp:310-321)
 *   losses     af [B]      -> float  loss[B]           (per sample, not reduced; Train.cpp:1743)
 *   paths      af [T,B]    -> int32  path[B][T]
 */
#ifndef W2L_B200_H_
#define W2L_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define W2L_API __attribute__((visibility("default")))

/* status codes */
enum {
  W2L_OK = 0,
  W2L_ERR_INVALID_ARGUMENT = 1, /* bad shape / null pointer  (-> std::invalid_argument) */
  W2L_ERR_WORKSPACE = 2,        /* workspace too small        (-> std::invalid_argument) */
  W2L_ERR_CUDA = 3,             /* a CUDA runtime call failed (-> std::runtime_error)    */
  W2L_ERR_UNSUPPORTED = 4       /* size outside what the kernels cover                   */
};

/* flashlight/lib/sequence/criterion/Defines.h CriterionScaleMode, selected by
 * getCriterionScaleMode(FLAGS_onorm, FLAGS_sqnorm) at Train.cpp:389 */
enum {
  W2L_SCALE_NONE = 0,
  W2L_SCALE_INPUT_SZ = 1,
  W2L_SCALE_INPUT_SZ_SQRT = 2,
  W2L_SCALE_TARGET_SZ = 3,
  W2L_SCALE_TARGET_SZ_SQRT = 4
};

/* which terms of the ASG criterion a call evaluates */
enum {
  W2L_TERM_FCC = 1, /* FullConnectionCriterion: loss = +FCC                       */
  W2L_TERM_FAC = 2, /* ForceAlignmentCriterion: loss = +FAC                       */
  W2L_TERM_ASG = 3  /* AutoSegmentationCriterion: loss = FCC - FAC                */
};

W2L_API int w2l_version(void);
W2L_API const char* w2l_last_error(void);
/* number of kernels this library launched on the calling thread since the last reset
 * (bench.py's "gpu_launches" claim) */
W2L_API long long w2l_launch_count(void);
W2L_API void w2l_reset_launch_count(void);
/* Measurement hook (bench.py's roofline leg): while set (non-NULL cudaEvent_t handles), every
 * call on this thread records `start` right before and `stop` right after its DOMINANT kernel
 * (asg_chains_kernel, ctc_chains_kernel, the GEMM of a dense op) on the call's stream, so that
 * kernel can be timed live inside a timed region.  Pass NULL, NULL to clear. */
W2L_API void w2l_set_profile_events(void* start_event, void* stop_event);
/* list mode: the k-th dominant-kernel launch of `kind` (0 any, 1 GEMM, 2 criterion chains) records pair k of the
 * caller-owned arrays (n pairs); w2l_profile_events_used() tells how many were consumed.  NULL clears. */
W2L_API int w2l_set_profile_event_list(int kind, void** start_events, void** stop_events, int n);
W2L_API int w2l_profile_events_used(void);
/* Trace mode (measurement only): between begin and end every kernel launched by this thread records one event on
 * `stream` (all work must be on that stream); end synchronises, sums the inter-event time per kernel name and writes
 * "name\tlaunches\tms\n" lines into out.  Returns the byte count needed (call with NULL to size). */
W2L_API int w2l_trace_begin(void* stream, int capacity);
W2L_API long long w2l_trace_end(char* out, long long out_bytes);
/* after w2l_trace_end: every traced launch in order, "name\tms\n" (same sizing convention) */
W2L_API long long w2l_trace_list(char* out, long long out_bytes);

/* ----------------------------------------------------------------------------------------
 * ASG = FullConnectionCriterion - ForceAlignmentCriterion, fused forward + backward.
 * Replaces AutoSegmentationCriterion::forward + its gradFunc (constructed at
 * recipes/slimIPL/src/Train.cpp:408-410, called :1675, backward :1720).
 *
 *   loss[b]   = scale_b * (FCC_b - FAC_b)                         (terms selects the parts)
 *   d_emis    = dloss[b] * d loss[b] / d emis     [B][T][N]
 *   d_trans   = sum_b dloss[b] * d loss[b] / d trans   [N][N]
 * dloss == NULL means ones (what loss.backward() seeds).  d_emis and d_trans may be NULL
 * together for a forward-only call (criterion->forward in eval mode, Train.cpp:977).
 * L is the padded target width; the per-sample size is the index of the last non-negative
 * entry + 1, clamped to T (upstream getTargetSizeArray).  Samples whose target is empty or
 * holds a label outside [0,N) get loss = NaN and zero gradient.
 * Supported: N <= 32 (token sets of the ASG recipes are ~30: conv_glu/.../train.cfg) and
 * targets of at most 1024 positions after the clamp to T (min(L, T) <= 1024: a warp walks a
 * recursion with up to 32 positions per lane); W2L_ERR_UNSUPPORTED beyond.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_asg_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_asg_forward_backward(void* stream, int terms, int B, int T, int N, int L, int scale_mode,
                                     const float* emis, const int32_t* target, const float* trans,
                                     const float* dloss, float* loss, float* d_emis, float* d_trans,
                                     void* workspace, size_t workspace_bytes);

/* ----------------------------------------------------------------------------------------
 * Viterbi decoding.  w2l_fcc_viterbi replaces ASGLoss::viterbiPath (Train.cpp:838, :1375):
 * max-plus FCC + backtrace, fp32 add/compare in ascending-j order, first maximum wins —
 * bit-exact with upstream ViterbiPath.  w2l_fac_viterbi is the forced alignment
 * (upstream ForceAlignmentCriterion::viterbiPath / fl_asr_align): path = label per frame,
 * path_idx (nullable) = position in the target per frame.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_fcc_viterbi_workspace_size(int B, int T, int N);
W2L_API int w2l_fcc_viterbi(void* stream, int B, int T, int N, const float* emis, const float* trans,
                            int32_t* path, void* workspace, size_t workspace_bytes);
W2L_API size_t w2l_fac_viterbi_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_fac_viterbi(void* stream, int B, int T, int N, int L, const float* emis, const int32_t* target,
                            const float* trans, int32_t* path, int32_t* path_idx, void* workspace,
                            size_t workspace_bytes);

/* ----------------------------------------------------------------------------------------
 * CTC, fused forward + backward on RAW activations (internal log-softmax over N, blank =
 * N-1 appended last: Train.cpp:248-251).  Replaces ConnectionistTemporalClassification
 * Criterion::forward (CTCLoss, Train.cpp:406-407; CUDA backend upstream = warp-ctc).
 * Every sample runs over the full padded T (the loop passes no input sizes to CTC/ASG:
 * Train.cpp:1473-1477).  d_emis may be NULL (forward only).  Targets of at most 1023 labels
 * after the clamp to T (2 * min(L, T) + 1 <= 2048 extended states); W2L_ERR_UNSUPPORTED beyond.
 * w2l_argmax_path = CTCLoss::viterbiPath (per-frame argmax, first maximum wins).
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_ctc_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_ctc_forward_backward(void* stream, int B, int T, int N, int L, int scale_mode, const float* emis,
                                     const int32_t* target, const float* dloss, float* loss, float* d_emis,
                                     void* workspace, size_t workspace_bytes);
W2L_API int w2l_argmax_path(void* stream, int B, int T, int N, const float* emis, int32_t* path);

/* LinearSegmentationCriterion's target stretch (Train.cpp:589-617, --linseg): out[b][t] =
 * target[b][floor(t * L_b / T)]; LinSeg = w2l_asg_forward_backward(W2L_TERM_ASG, L = T) on it (loss FCC - FAC). */
W2L_API int w2l_linseg_target(void* stream, int B, int T, int L, const int32_t* target, int32_t* out);

/* ----------------------------------------------------------------------------------------
 * Dense contraction of the acoustic model (replaces fl::Linear's af::matmul -> cuBLAS and the
 * GEMM inside cuDNN's convolutions; forward at Train.cpp:1470, backward at :1720).
 *   C[m][n] = act( sum_k A(m,k) * B(n,k) + bias[n] ),  fp32 storage, wgmma math in the kind the thread's precision
 *   setting selects (TF32 by default, F32X3 under W2L_PRECISION_F32), fp32 accumulation.  a_mn_major = 0: A stored [M][K] (lda), 1: A stored [K][M];  b_mn_major = 0:
 *   B stored [N][K] (ldb), 1: B stored [K][N].  forward Y = X W^T : (0,0); dgrad dX = dY W :
 *   (0,1) with B = W; wgrad dW = dY^T X : (1,1) with A = dY, B = X.  bias nullable; act 0 none,
 *   1 ReLU.  lda/ldb must be multiples of 4 floats and A/B 16-byte aligned (TMA).
 * ---------------------------------------------------------------------------------------- */
/* w2l_gemm_tf32 with OVERLAPPING operand rows allowed (lda / ldb may be smaller than the row length; still % 4):
 * the im2col matrix of a stride-1 time convolution over [T][Cin] activations — row t = the kw*Cin contiguous floats
 * starting at frame t, row stride Cin — is then a zero-copy TMA view.  This is how the large-channel `C` convolutions
 * of the conv_glu archs (recipes/conv_glu/librispeech/network.arch) run on the wgmma GEMM:
 *   fwd   Y[t][co]  = sum_k Xview[t][k] Warr[co][k]            (A = Xview K-major, lda = Cin;  B = Warr K-major)
 *   dgrad dX[t][ci] = sum_k dYview[t][k] Wflip[ci][k]          (A = zero-padded dY view, lda = Cout)
 *   wgrad dWarr[co][k] += sum_t dY[t][co] Xview[t][k]          (A = dY MN-major; B = Xview MN-major, ldb = Cin)
 * (the data gradient's kw-1 frames of left context are kw-1 zero rows in front of dY: the caller pads a copy) */
W2L_API int w2l_gemm_tf32_view(void* stream, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                               const float* B, int ldb, float* C, int ldc, const float* bias, int act, int accumulate);
/* Operand kinds of the wgmma GEMM (csrc/gemm_wgmma.cu) and the precision setting that selects among them.
 *   TF32  : fp32 operands in HBM, TF32 products (10-bit mantissa), fp32 accumulation — what cuDNN/cuBLAS do by default
 *           for fp32 tensors on Ampere+; the default.
 *   F32X3 : fp32 operands in HBM, fp32-ACCURATE contraction: each staged tile is split hi/lo in shared memory and the
 *           tensor core accumulates Al*Bh + Ah*Bl + Ah*Bh (error-compensated 3xTF32, products good to ~2^-21) — the
 *           precision BASELINE.json configs[1] ("fp32") states; the time convolutions use the fp32 SIMT kernels.
 *   BF16  : bf16 operands in HBM (activations / weights cast by their producers), fp32 accumulation — the AMP mode of
 *           the reference (recipes/slimIPL/src/Train.cpp:211-219) with bf16 instead of fp16, configs[2]/[3].
 * w2l_set_precision is thread-local and selects the kind used by the fp32-operand entry points (w2l_gemm_tf32*,
 * w2l_conv_time_*) and by the fl_compat modules (which cast their GEMM operands in BF16 mode). */
enum { W2L_GEMM_TF32 = 0, W2L_GEMM_F32X3 = 1, W2L_GEMM_BF16 = 2 };
enum { W2L_PRECISION_TF32 = 0, W2L_PRECISION_F32 = 1, W2L_PRECISION_BF16 = 2 };
W2L_API int w2l_set_precision(int precision);
W2L_API int w2l_get_precision(void);
/* General form: A / B are fp32 (kinds TF32, F32X3) or bf16 (kind BF16) with lda / ldb in ELEMENTS (rows 16-byte aligned:
 * ld % 4 for fp32, ld % 8 for bf16); C is fp32 or bf16 (c_bf16; no accumulate / split-K then); aux (the backward mask
 * source) fp32 or bf16 (aux_bf16).  allow_overlap: operand rows may overlap (im2col views, see w2l_gemm_tf32_view). */
W2L_API int w2l_gemm(void* stream, int kind, int a_mn_major, int b_mn_major, int M, int N, int K, const void* A, int lda,
                     const void* B, int ldb, void* C, int ldc, int c_bf16, const float* bias, int act, int accumulate,
                     const void* aux, int ld_aux, int aux_bf16, int aux_mode, float aux_scale, float dropout_p,
                     unsigned long long seed, int allow_overlap);
/* fp32 -> bf16 (round to nearest even): flat, and row-wise with zero-padded columns (rows of `cols` floats, row stride
 * ld_in, to rows of cols_padded bf16) */
W2L_API int w2l_cast_bf16(void* stream, long long n, const float* x, void* y);
W2L_API int w2l_cast_bf16_rows(void* stream, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y);
/* Pin the GEMM tile width (128 / 160 / 224 / 256; 0 = choose per shape, the default).  Thread-local; for tests and tuning. */
W2L_API int w2l_gemm_set_tile(int bn);
/* 1 (default): one CTA per SM walking the tiles, so the producer stages the next tile's operands during an epilogue;
 * 0: one CTA per tile.  Thread-local; for tests (the two must agree) and tuning. */
W2L_API int w2l_gemm_set_variant(int variant);
W2L_API int w2l_gemm_tf32(void* stream, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                          const float* B, int ldb, float* C, int ldc, const float* bias, int act);

/* Extended epilogue: after bias/act, (a) forward dropout with keep-scale 1/(1-p) (Philox4x32-10 keyed by
 * (seed, element index)), (b) backward activation mask read back from a stored activation tensor
 * aux[M][ld_aux]: aux_mode 1 multiplies by (aux > 0) * aux_scale (fused ReLU+dropout backward),
 * 2 by (aux != 0) * aux_scale (dropout backward), (c) accumulate != 0: C += result. */
W2L_API int w2l_gemm_tf32_ex(void* stream, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                             const float* B, int ldb, float* C, int ldc, const float* bias, int act, int accumulate,
                             const float* aux, int ld_aux, int aux_mode, float aux_scale, float dropout_p,
                             unsigned long long seed);

/* ----------------------------------------------------------------------------------------
 * Time convolution of the acoustic models: fl::Conv2D with a kw x 1 kernel (TDSBlock's conv,
 * the strided `C2` front-ends; arch parser cpc/SequentialBuilder.cpp:254-301).  Activations are
 * float [B][T][C][W] (W <= 80 innermost), weights float wt[Cout][Cin][K] (= fl's [kw,1,cin,cout]
 * column-major), out frame `to` reads input frames to*stride + dk - pad_left.
 *   fwd   : y = dropout(act(conv(x) + bias)) (+ add)          act 0 none / 1 ReLU
 *   dgrad : dx = conv^T(dy) (+ add)                           add may be dx itself (in-place accumulation;
 *                                                            likewise add == y in fwd)
 *   wgrad : dwt += ..., dbias += ...  (deterministic two-stage reduction)
 * The workspace size call covers all three.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_conv_time_workspace_size(int B, int Tout, int Cin, int Cout, int K);
/* 0 (default): the mma.sync tensor-core kernels where the shape allows (TF32, or 3xTF32 under W2L_PRECISION_F32); 1: always the
 * fp32 SIMT kernels (the fallback for widths that are not multiples of 8); 2: mma.sync; 3: the wgmma / TMA kernel of
 * conv_wgmma.cu for forward and stride-1 data gradients (parity-green, opt-in: see DESIGN.md).  Thread-local. */
W2L_API int w2l_conv_set_path(int path);
W2L_API int w2l_conv_time_fwd(void* stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                              int pad_left, const float* x, const float* wt, const float* bias, const float* add, float* y,
                              int act, float dropout_p, unsigned long long seed, void* ws, size_t ws_bytes);
W2L_API int w2l_conv_time_dgrad(void* stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                int pad_left, const float* dy, const float* wt, const float* add, float* dx, void* ws,
                                size_t ws_bytes);
W2L_API int w2l_conv_time_wgrad(void* stream, int B, int T, int Tout, int W, int Cin, int Cout, int K, int stride,
                                int pad_left, const float* x, const float* dy, float* dwt, float* dbias, void* ws,
                                size_t ws_bytes);

/* ------------------------------------------------------------------------------------------
 * Conv1D + GLU family (recipes/conv_glu/{wsj,librispeech}/network.arch: `WN 3 C cin cout kw 1 pad`, `GLU 2`, `DO p`,
 * `RO 2 0 3 1`, `WN 0 L in out`, `GLU 0`).  Activations are [rows = B*T][C] row-major (internal layout with W = 1).
 *   weightnorm : w[r][:] = g[r] v[r][:] / ||v[r][:]|| per output unit r (rows of the [cout][cin*kw] / [out][in] weight);
 *                bwd ADDS into dv, dg.  inv_norm [rows] is saved by fwd for bwd.
 *   conv1d_arrange : w [cout][cin][kw] (= fl's [kw,1,cin,cout]) -> GEMM operands fwd [cout_p][kw*cin_p] and (nullable)
 *                flip [cin_p][kw*cout_p] (data gradient), bias -> bias_p [cout_p]; padded channels are zero.  glu_split:
 *                the two halves of cout are padded separately (cout_p/2 each) so a following GLU stays aligned.
 *                The convolution itself is w2l_gemm_tf32_view on these operands.
 *   conv1d_unarrange_grad : dw[co][ci][dk] += dfwd[row(co)][dk*cin_p+ci]; dbias[co] += sum_rows dy[row][col(co)]
 *   glu        : y[r][c] = x[r][c] * sigmoid(x[r][half+c]) * dropout-mask(r*half+c)   (x has 2*half columns)
 * ---------------------------------------------------------------------------------------- */
W2L_API int w2l_weightnorm_fwd(void* stream, int rows, int len, const float* v, const float* g, float* w, float* inv_norm);
W2L_API int w2l_weightnorm_bwd(void* stream, int rows, int len, const float* v, const float* g, const float* inv_norm,
                               const float* dw, float* dv, float* dg);
W2L_API int w2l_conv1d_arrange(void* stream, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split, const float* w,
                               const float* bias, float* fwd, float* flip, float* bias_p);
/* the same with bf16 destination operands (out_bf16 != 0; W2L_PRECISION_BF16): fwd / flip are written as bf16 directly */
W2L_API int w2l_conv1d_arrange_ex(void* stream, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split, const float* w,
                                  const float* bias, void* fwd, void* flip, float* bias_p, int out_bf16);
W2L_API int w2l_conv1d_unarrange_grad(void* stream, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split,
                                      const float* dfwd, float* dw, long long rows, const float* dy, float* dbias);
W2L_API int w2l_glu_fwd(void* stream, long long rows, int half, const float* x, float* y, float dropout_p,
                        unsigned long long seed);
W2L_API int w2l_glu_bwd(void* stream, long long rows, int half, const float* x, const float* dy, float* dx, float dropout_p,
                        unsigned long long seed);

/* fl::LayerNorm over a whole sample (R = T*C*W elements; `LN 0 1 2` / TDSBlock with lnIncludeTime)
 * with scalar gain/bias (device scalars, nullable = 1/0) and a fused residual: y = LN(a + r).
 * mean_rstd [B][2] is saved for the backward pass; scratch = W2L_LN_SCRATCH_DOUBLES(B) doubles (one partial
 * pair per CTA: no zero-fill, no atomics, deterministic).
 * Backward: d_res = ds, d_branch = ds * mask(a) where the mask undoes the fused ReLU/dropout of the
 * branch that produced `a` (branch_mode 0 none, 1 (a>0)*scale, 2 (a!=0)*scale); dgain/dbias accumulate. */
#define W2L_LN_MAX_PARTS 80
#define W2L_LN_SCRATCH_DOUBLES(B) (2 * W2L_LN_MAX_PARTS * (size_t)(B))
W2L_API int w2l_layernorm_fwd(void* stream, int B, long long R, float eps, const float* a, const float* r,
                              const float* gain, const float* bias, float* y, float* mean_rstd, double* scratch);
W2L_API int w2l_layernorm_bwd(void* stream, int B, long long R, const float* a, const float* r, const float* dy,
                              const float* gain, const float* mean_rstd, float* d_branch, float* d_res, int branch_mode,
                              float branch_scale, float* dgain, float* dbias, double* scratch);

/* out[n] += sum_m X[m][n]  (bias gradient of fl::Linear) */
W2L_API int w2l_colsum_accumulate(void* stream, int M, int N, const float* X, int ld, float* out);
/* fl::clipGradNorm + fl::SGDOptimizer::step + the loop's gradient scaling (Train.cpp:1743-1803) on a
 * flat parameter arena: out += sum g^2 ;  g' = g*grad_scale*clip ; g' += wd*p ; v = mom*v + g' ; p -= lr*v */
W2L_API int w2l_sq_norm_accumulate(void* stream, long long n, const float* g, double* out);
W2L_API int w2l_sgd_step(void* stream, long long n, float* params, const float* grads, float* velocity, float lr,
                         float momentum, float weight_decay, float grad_scale, float max_grad_norm, const double* sq_norm);
/* + Nesterov momentum (fl::SGDOptimizer useNesterov: g += momentum * v after the velocity update) and a device-side guard:
 * guard[0] != 0 -> the update is skipped.  w2l_finite_guard sets guard[0] = (any loss[i] or *sq_norm is NaN / Inf) and
 * adds 1 to guard[1] when it is: the NaN check of Train.cpp:1686-1698 and the mixed-precision overflow check of
 * :1753-1771 without a host round trip (the host reads the counter when it wants to). */
W2L_API int w2l_sgd_step_ex(void* stream, long long n, float* params, const float* grads, float* velocity, float lr, float momentum,
                            float weight_decay, float grad_scale, float max_grad_norm, const double* sq_norm, int nesterov,
                            const int* guard);
W2L_API int w2l_finite_guard(void* stream, int n_loss, const float* loss, const double* sq_norm, int* guard);
/* fl::SpecAugment masking (arch opcode SAUG, cpc/SequentialBuilder.cpp:602-613) on [B][T][C][W] activations: frequency
 * bands [f0,f1) of W and time bands [t0,t1) of T (host arrays, <= 8 each; the same bands for the whole batch) := value */
W2L_API int w2l_mask_bands(void* stream, int B, int T, int C, int W, const float* x, float* y, int n_f, const int* f0_host,
                           const int* f1_host, int n_t, const int* t0_host, const int* t1_host, float value);

/* small element-wise helpers of the host layer: network input [T,F,1,B] (ArrayFire, T fastest) -> internal
 * [B][T][1][F]; y += a*x; y = v; standalone ReLU/Dropout forward and their backward mask. */
W2L_API int w2l_transpose_input(void* stream, int B, int F, int T, const float* in, float* out);
W2L_API int w2l_axpy(void* stream, long long n, float a, const float* x, float* y);
W2L_API int w2l_fill(void* stream, long long n, float v, float* y);
W2L_API int w2l_act_fwd(void* stream, long long n, const float* x, int relu, float dropout_p, unsigned long long seed, float* y);
W2L_API int w2l_mask_mul(void* stream, long long n, const float* g, const float* ref, int mode, float scale, float* out);

/* ----------------------------------------------------------------------------------------
 * Training-step driver: the body of the reference loop (recipes/slimIPL/src/Train.cpp:1454-1803) written
 * in C++ against include/fl_compat/fl_compat.h — network forward, criterion, loss.backward(), NCCL
 * all-reduce of every gradient, division by the global batch size, clipGradNorm over net U criterion,
 * criterion + network SGD steps.  `arch_text` is a wav2letter arch file (opcodes V RO PD C2 R DO LN TDS L
 * SAUG), `criterion` "ctc" or "asg".  All pointers below are DEVICE pointers:
 * features [T,F,1,B] (ArrayFire layout, T fastest), target [L,B] int32 (-1 padded), loss_out [B].
 * Returns NULL / a status code; w2l_last_error() has the text.
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_trainer_create(void* stream, const char* arch_text, int n_feat, int n_label, const char* criterion,
                                 int scale_mode, float transdiag, float lr, float lrcrit, float momentum, float maxgradnorm);
W2L_API void w2l_trainer_destroy(void* trainer);
W2L_API int w2l_trainer_step(void* trainer, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                             float* loss_out, int train, float total_batch);
W2L_API int w2l_trainer_forward(void* trainer, void* stream, int B, int T, const float* features, float* emissions_out,
                                long long capacity, int* t_out);
/* precision of the trainer's dense contractions (W2L_PRECISION_*; default: the creating thread's w2l_set_precision) */
W2L_API int w2l_trainer_set_precision(void* trainer, int precision);
/* steps whose update was skipped on the device because the loss or a gradient was NaN / Inf (Train.cpp:1686-1698,
 * :1753-1771); synchronises `stream` */
W2L_API int w2l_trainer_status(void* trainer, void* stream, long long* skipped_steps);
W2L_API long long w2l_trainer_num_params(void* trainer, int which /*0 network, 1 criterion*/);
W2L_API int w2l_trainer_param_layout(void* trainer, int which, int max_params, long long* elements, long long* dims4);
W2L_API int w2l_trainer_get_flat(void* trainer, void* stream, int which, int what /*0 values, 1 gradients*/, float* out);
W2L_API int w2l_trainer_set_flat(void* trainer, void* stream, int which, const float* in);
W2L_API int w2l_trainer_sync_parameters(void* trainer, void* stream);   /* fl::allReduceParameters, Train.cpp:1078-1079 */
W2L_API const char* w2l_trainer_describe(void* trainer);
/* Checkpoints (SURVEY.md §8 f4; the role of Serializer::save / load in Train.cpp:747-800): own little-endian container with
 * the constructor arguments + parameter / momentum arenas of network and criterion; load rebuilds the trainer. */
W2L_API int w2l_trainer_save(void* trainer, void* stream, const char* path);
W2L_API void* w2l_trainer_load(void* stream, const char* path);
/* Export for the in-tree streaming inference stack, following the conversions of
 * recipes/streaming_convnets/tools/StreamingTDSModelConverter.cpp:46-136,203-283: every layer's arrays in the inference
 * library's layouts (acoustic_model.json + acoustic_model.bin), transitions.bin (ASG; the cereal std::vector<float> the
 * inference examples read, :310-326) and tokens.txt (tokens_text nullable).  Streaming TDS archs only (LN 1 2), like the converter. */
W2L_API int w2l_trainer_export_streaming(void* trainer, void* stream, const char* outdir, const char* tokens_text);
/* data-parallel rendezvous: rank 0 creates the 128-byte NCCL id, the launcher ships it to every rank */
W2L_API int w2l_nccl_unique_id(void* out128);
W2L_API int w2l_init_distributed(int rank, int world, const void* id128);

/* ----------------------------------------------------------------------------------------
 * Token / target pipeline either side of the criterion (SURVEY.md §8 f3; host code, no GPU work):
 *   w2l_text_create     Dictionary(tokens) + "<1>".."<replabel>" + the CTC blank appended last (Train.cpp:236-254), the
 *                       lexicon (loadWords), and the flags --criterion --surround --usewordpiece --wordseparator
 *   w2l_text_encode     the dataset's target transform (targetFeatures, Train.cpp:296-316): words -> lexicon spelling or
 *                       letter fallback -> indices -> surround -> replabel packing -> ASG dedup
 *   w2l_text_prediction2ltr / target2ltr / ltr2wrd / w2l_edit_distance   evalOutput (Train.cpp:829-872): Viterbi path ->
 *                       uniq -> drop blanks -> unpack replabels -> trim surround / silence -> letters -> words -> Levenshtein
 * Strings are UTF-8; token sequences are space-joined.  Functions returning long long give the element / byte count needed
 * (call with a zero capacity to size) or -1 on error (w2l_last_error).
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_text_create(const char* tokens_text, const char* lexicon_text, const char* criterion, int replabel,
                              const char* surround, int usewordpiece, const char* wordsep);
W2L_API void w2l_text_destroy(void* text);
W2L_API int w2l_text_num_classes(void* text);
W2L_API long long w2l_text_encode(void* text, const char* transcript, int32_t* out, long long cap);
W2L_API long long w2l_text_prediction2ltr(void* text, const int32_t* path, int n, char* out, long long cap);
W2L_API long long w2l_text_target2ltr(void* text, const int32_t* target, int len, char* out, long long cap);
W2L_API long long w2l_text_ltr2wrd(void* text, const char* letters, char* out, long long cap);
/* out4 += {reference length, deletions, insertions, substitutions} of one (hypothesis, reference) pair */
W2L_API int w2l_edit_distance(const char* hyp, const char* ref, long long* out4);

#ifdef __cplusplus
}
#endif
#endif /* W2L_B200_H_ */
