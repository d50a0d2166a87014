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
/* the process-wide seed stream that parameter initialisation, dropout and SpecAugment draw from (flashlight's
 * fl::setSeed): read it, and set it back, so that what one part of a program creates does not change the initial
 * parameters of trainers created after it */
W2L_API unsigned long long w2l_get_seed(void);
W2L_API void w2l_set_seed(unsigned long long seed);
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
 *
 * w2l_asg64_*: the same signature, layouts, scale modes, terms, target rules and error codes
 * for 1 <= N <= 64 (the 39 folded phones of the TIMIT recipe, learnable_frontend), from the
 * same kernels at twice the state width (two states per lane).  It is a separate call because
 * the N <= 32 contract above, W2L_ERR_UNSUPPORTED for N > 32 included, is published and
 * tested; callers pick the call from N (the trainer does).  N > 64: W2L_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_asg_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_asg_forward_backward(void* stream, int terms, int B, int T, int N, int L, int scale_mode,
                                     const float* emis, const int32_t* target, const float* trans,
                                     const float* dloss, float* loss, float* d_emis, float* d_trans,
                                     void* workspace, size_t workspace_bytes);
W2L_API size_t w2l_asg64_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_asg64_forward_backward(void* stream, int terms, int B, int T, int N, int L, int scale_mode,
                                       const float* emis, const int32_t* target, const float* trans,
                                       const float* dloss, float* loss, float* d_emis, float* d_trans,
                                       void* workspace, size_t workspace_bytes);

/* ----------------------------------------------------------------------------------------
 * Viterbi decoding.  w2l_fcc_viterbi replaces ASGLoss::viterbiPath (Train.cpp:838, :1375):
 * max-plus FCC + backtrace, fp32 add/compare in ascending-j order, first maximum wins —
 * bit-exact with upstream ViterbiPath.  w2l_fac_viterbi is the forced alignment
 * (upstream ForceAlignmentCriterion::viterbiPath / fl_asr_align): path = label per frame,
 * path_idx (nullable) = position in the target per frame.
 * w2l_fcc_viterbi covers N <= 32 (W2L_ERR_UNSUPPORTED beyond, as published);
 * w2l_fcc_viterbi64 is the same contract, bit-exactness included, for 1 <= N <= 64.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_fcc_viterbi_workspace_size(int B, int T, int N);
W2L_API int w2l_fcc_viterbi(void* stream, int B, int T, int N, const float* emis, const float* trans,
                            int32_t* path, void* workspace, size_t workspace_bytes);
W2L_API size_t w2l_fcc_viterbi64_workspace_size(int B, int T, int N);
W2L_API int w2l_fcc_viterbi64(void* stream, int B, int T, int N, const float* emis, const float* trans,
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

/* ----------------------------------------------------------------------------------------
 * CTC Viterbi with target: the forced alignment of a CTC model (upstream SequenceCriterion::viterbiPathWithTarget of
 * CTCLoss).  Contract, bit for bit:
 *   - inputs are raw activations emis[B][T][N], blank = N-1 as in w2l_ctc_forward_backward, and target[B][L], -1
 *     padded (L_b = index of the last non-negative entry + 1).  The extended target is z of length S = 2 L_b + 1,
 *     blanks interleaved: z_s = blank for even s, y_{(s-1)/2} for odd s.
 *   - scores are the raw activations, not the log-softmax: every path takes exactly one state per frame, so the
 *     per-frame log-partition adds the same constant to every path and the argmax is the same.
 *   - alpha_0[0] = e_0[blank], alpha_0[1] = e_0[z_1], others -inf;
 *     alpha_t[s] = fp32(max(alpha_{t-1}[s], alpha_{t-1}[s-1], alpha_{t-1}[s-2] if z_s != blank and z_s != z_{s-2})
 *                       + e_t[z_s]) — one add, no FMA, no reassociation.
 *   - ties: predecessors are taken in the order s, s-1, s-2, and a later one replaces the current one only if it is
 *     strictly greater.  The end state is S-1 unless alpha_{T-1}[S-2] > alpha_{T-1}[S-1].
 *   - path[b][t] = z of the state the path occupies at frame t (a label, or N-1 for blank); state[b][t] (nullable) = s.
 *   - every sample runs over the full padded T, like every criterion call here.  An empty target gives all blanks.
 *   - a target that needs more frames than T (L_b + adjacent repeats > T), or that holds a label outside [0, N-1),
 *     gives path = state = -1 for the whole utterance (the loss would truncate it; an alignment that drops words is
 *     worse than none).
 * Limits: those of the CTC loss, min(L, T) <= 1023 (S <= 2047), any N >= 2; W2L_ERR_UNSUPPORTED beyond.  target may be
 * NULL when L = 0.  The workspace holds the gathered scores [B][T][Sp] (Sp = 32 P >= S) and 2-bit backpointers.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_ctc_viterbi_workspace_size(int B, int T, int N, int L);
W2L_API int w2l_ctc_viterbi_target(void* stream, int B, int T, int N, int L, const float* emis, const int32_t* target,
                                   int32_t* path, int32_t* state, void* workspace, size_t workspace_bytes);

/* LinearSegmentationCriterion's target stretch (Train.cpp:589-617, --linseg): out[b][t] =
 * target[b][floor(t * L_b / T)]; LinSeg = w2l_asg_forward_backward(W2L_TERM_ASG, L = T) on it (loss FCC - FAC). */
W2L_API int w2l_linseg_target(void* stream, int B, int T, int L, const int32_t* target, int32_t* out);

/* ----------------------------------------------------------------------------------------
 * Seq2Seq criterion (--criterion=seq2seq: attention-GRU decoder, DESIGN.md §9), the kernels fl_compat's
 * Seq2SeqCriterion runs beside the GEMMs of its projections.  Rows r = b*U + u of [B*U][width] row-major, H the hidden
 * size (--encoderdim), N the dictionary size (eos and pad included), x the encoder output [B][T'][2H] (keys x[.][0:H],
 * values x[.][H:2H]), target [B][U] int32.  Limits: H a multiple of 32 and <= 1024, 3 <= N <= 65536
 * (w2l_seq2seq_check; W2L_ERR_UNSUPPORTED outside), and what fits in 220 KB of shared memory: 8 (H + T') floats for
 * the attention (T' <= 7040 - H), 16 U floats for its gradient (U <= 3520), the W_hh slice of one CTA for the recurrence.
 *   embed_fwd   tokens[b][0] = N (startEmbedding), tokens[b][u] = target[b][u-1], replaced with probability
 *               1 - pct/100 by min(floor(r2 (N-1)), N-2) (Philox block of counter b*U + u under seed: r1 = word x, r2 =
 *               word y, each (w >> 8) 2^-24; replaced iff r1 < fp32(1 - pct/100)); out[r] = E[tokens[r]] or start.
 *               Targets are checked on the device: a value outside [0, N) sets bad[b] (int32 [B], nullable, zeroed
 *               by the caller) and is read as token 0, so nothing outside E is read.
 *   embed_bwd   dE[n] += sum of din over the rows with token n, dstart likewise (row order; no atomics)
 *   gru_fwd     one GRU layer over all U steps from h0 (NULL: 0), gi = W_ih x + b_ih precomputed [B*U][3H], gate order
 *               r, z, n; stash (nullable) [5][B*U][H] = r, z, n, W_hn h + b_hn, h_{u-1}.  One cooperative launch.
 *   gru_bwd     from dout [B*U][H]: dgi = d(W_ih x + b_ih) and dgh = d(W_hh h + b_hh), both [B*U][3H]; carry [B][H]
 *               scratch.  dW_hh = dgh^T h_{u-1}, db_hh = colsum dgh are the caller's GEMM / reduction.
 *   attn_fwd    out = q + sum_t softmax_t(q.k_t / sqrt(H) + w_{u,t}) v_t, with the soft window
 *               w = -(t - u T'/window_u)^2 / (2 window_std^2) when window_std > 0; attn (nullable) [B*U][T'] the weights
 *   attn_bwd    from dout = d out: dq (the identity path included) and dx [B][T'][2H] (written), dS [B*U][T'] scratch
 *   sizes       per-utterance bounds of a padded batch (DESIGN.md §9), one launch: from durations [B] (the input frame
 *               counts; int32, or float32 holding whole numbers when durations_f32 = 1; NULL: every T'_b = T')
 *               T'_b = ceil(d_b T' / max d) in double clamped to [1, T'], into tp_sizes [B]; from target_sizes [B] int32
 *               (NULL: U) U_b into u_sizes [B].  Rejected in-band, with no host synchronisation: d_b <= 0 or not whole,
 *               no positive duration at all, a target size outside [1, U] set bad[b] (nullable); the bound stays in range.
 *   attn_fwd_sized / attn_bwd_sized   attn_fwd / attn_bwd over frames t < tp_sizes[b] of utterance b (device int32
 *               [B], nullable: T'), with the window centred at u T'_b / U_b, U_b = u_sizes[b] (nullable: window_u).
 *               Nothing at t >= T'_b is read: attn holds 0 there and dx is written as 0.  With both NULL they are
 *               attn_fwd / attn_bwd, bit for bit.
 *   loss        per row: log-softmax over N, (1-ls)(-log p_y) - (ls/N) sum_c log p_c, 0 on rows with target = pad;
 *               loss[b] = sum over u (in order), rowloss [B*U] scratch; grad != 0 also writes the logit gradient
 *               dloss[b] (NULL: 1) (p - (1-ls) e_y - ls/N) over the logits, in place, 0 on pad rows.
 *               An utterance flagged in bad (nullable: embed_fwd's flags) or with a target outside [0, N) gets loss
 *               NaN and zero gradient: rejected in-band, as the other criteria reject bad labels.
 *   scale_rows  d[b*U+u][:] *= g[b] / seed_scale
 *   decode_*    one greedy step: argmax of logits [B][N] (first maximum); eos finishes an utterance (len[b] = step, not
 *               emitted), another token is written to tokens[b][step] and in[b] = E[token]; done[B] counts finished
 *               utterances.  init: in = start, tokens = pad, len = maxlen, done = 0 ([B + 1] ints).
 *   beam_*      the beam search of DESIGN.md §9 over B utterances x K slots, decoder rows r = b*K + slot, 1 <= K <= 16
 *               (W2L_ERR_UNSUPPORTED outside).  ws: beam_workspace_size(B, K, maxlen) bytes; its first int32 counts
 *               the utterances whose search has stopped early (the host reads it between steps).
 *               init: in [B*K][H] = start, slot 0 of each utterance live with score 0.
 *               step: from logits [B*K][N] of the live rows: scores s = score + log_softmax(logits) in fp32, each row's
 *               best 2K (s desc, class asc), then per utterance the walk over the merged ranks (eos at rank < K
 *               completes the hypothesis, at rank >= K is dropped; other classes extend the beam up to K), the K-cap
 *               (stable sort of the completions, keep K) and the early stop (K-th completion > best live score).  Then
 *               state[l][r] = next[l][b*K + parent(r)] for l < layers (each [B*K][H]) and in[r] = E[token(r)].
 *               finish: tokens [B][K][maxlen] padded with pad, lengths and scores [B][K], counts [B] (<= K): the
 *               completions if there are any (sorted if the cap ever applied, else in completion order), else the
 *               live beam at length steps; slots at or beyond counts[b] hold pad, length 0 and score -inf.
 * ---------------------------------------------------------------------------------------- */
W2L_API int w2l_seq2seq_check(int H, int N);
W2L_API int w2l_seq2seq_embed_fwd(void* stream, int B, int U, int H, int N, const int32_t* target, const float* E, const float* start,
                                  float pct_teacher_forcing, unsigned long long seed, int32_t* tokens, float* out, int32_t* bad);
W2L_API int w2l_seq2seq_embed_bwd(void* stream, int B, int U, int H, int N, const int32_t* tokens, const float* din, float* dE, float* dstart);
W2L_API size_t w2l_seq2seq_gru_stash_floats(int B, int U, int H);
W2L_API int w2l_seq2seq_gru_fwd(void* stream, int B, int U, int H, const float* gi, const float* Whh, const float* bhh, const float* h0,
                                float* out, float* stash);
W2L_API int w2l_seq2seq_gru_bwd(void* stream, int B, int U, int H, const float* dout, const float* Whh, const float* stash, float* dgi, float* dgh,
                                float* carry);
W2L_API int w2l_seq2seq_attn_fwd(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, int window_u, float window_std,
                                 float* out, float* attn);
W2L_API int w2l_seq2seq_attn_bwd(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const float* attn, const float* dout,
                                 float* dq, float* dx, float* dS);
W2L_API int w2l_seq2seq_sizes(void* stream, int B, int Tp, int U, const void* durations, int durations_f32, const int32_t* target_sizes,
                              int32_t* tp_sizes, int32_t* u_sizes, int32_t* bad);
W2L_API int w2l_seq2seq_attn_fwd_sized(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const int32_t* tp_sizes,
                                       const int32_t* u_sizes, int window_u, float window_std, float* out, float* attn);
W2L_API int w2l_seq2seq_attn_bwd_sized(void* stream, int B, int U, int Tp, int H, const float* q, const float* x, const float* attn, const float* dout,
                                       const int32_t* tp_sizes, float* dq, float* dx, float* dS);
W2L_API int w2l_seq2seq_loss(void* stream, int B, int U, int N, int pad, const int32_t* target, float* logits, float label_smooth,
                             const float* dloss, int grad, float* rowloss, float* loss, const int32_t* bad);
W2L_API int w2l_seq2seq_scale_rows(void* stream, int B, int U, int N, const float* g, float seed_scale, float* d);
W2L_API int w2l_seq2seq_decode_init(void* stream, int B, int H, int maxlen, int pad, const float* start, float* in, int32_t* tokens, int32_t* len,
                                    int32_t* done);
W2L_API int w2l_seq2seq_decode_step(void* stream, int B, int N, int H, int step, int eos, const float* logits, const float* E, float* in,
                                    int32_t* tokens, int maxlen, int32_t* len, int32_t* done);
W2L_API size_t w2l_seq2seq_beam_workspace_size(int B, int K, int maxlen);
W2L_API int w2l_seq2seq_beam_init(void* stream, int B, int K, int H, int maxlen, const float* start, float* in, void* ws, size_t ws_bytes);
W2L_API int w2l_seq2seq_beam_step(void* stream, int B, int K, int N, int H, int layers, int step, int maxlen, int eos, const float* logits,
                                  const float* E, float* in, float* state, const float* next, void* ws, size_t ws_bytes);
W2L_API int w2l_seq2seq_beam_finish(void* stream, int B, int K, int maxlen, int steps, int pad, const void* ws, size_t ws_bytes, int32_t* tokens,
                                    int32_t* lengths, float* scores, int32_t* counts);

/* ----------------------------------------------------------------------------------------
 * slimIPL (recipes/slimIPL/src/Train.cpp; DESIGN.md §7).
 * w2l_soft_label_loss: student and teacher are fp32 logits [rows][N] (rows = B T'; any N, any float alignment).
 *   loss_out (one float) = -scale / rows * sum_rows sum_c p_c (z_c - lse(z)),  p = softmax(teacher row), z = student row
 *   d_student (nullable: loss only) = scale / rows * (softmax(z) - p), written, not accumulated; exactly 0 where a teacher
 *   row has the bits of its student row.  ws: device scratch of `rows` floats.  Deterministic (no atomics).
 * w2l_ema_update: ema = ema * d + params * (1 - d) over n floats, d and 1 - d each rounded once from decay, every product
 *   and the sum rounded once (no fma).
 * ---------------------------------------------------------------------------------------- */
W2L_API int w2l_soft_label_loss(void* stream, long long rows, int N, const float* student, const float* teacher, float scale, float* loss_out,
                                float* d_student, float* ws);
W2L_API int w2l_ema_update(void* stream, long long n, float* ema, const float* params, double decay);

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
 *           precision BASELINE.json configs[1] ("fp32") states; the time convolutions run their mma.sync kernels in
 *           3xTF32 the same way.
 *   BF16  : bf16 operands in HBM (activations / weights cast by their producers), fp32 accumulation — the AMP mode of
 *           the reference (recipes/slimIPL/src/Train.cpp:211-219) with bf16 instead of fp16, configs[2]/[3].
 *   FP16  : fp16 operands in HBM, fp32 accumulation — the reference's own AMP operand type
 *           (--fl_amp_use_mixed_precision casts conv and matmul inputs to fp16); same layouts, tiles and MAC rate as BF16,
 *           3 more significand bits, 3 fewer exponent bits (finite up to 65504).
 *   F32X3_SPLIT_B : F32X3 with B split ahead of the call by w2l_split_tf32: B is K-major only and points at
 *           [2][N][ldb] fp32, the tf32 hi plane then the lo plane (ldb % 4 == 0, ldb >= K).  Results are bit-identical
 *           to F32X3 on the unsplit B; the kernel loads both planes by TMA and converts nothing, which pays when B (a
 *           weight) is reused by many rows of output tiles.
 * w2l_set_precision is thread-local and selects the kind used by the fp32-operand entry points (w2l_gemm_tf32*,
 * w2l_conv_time_*) and by the fl_compat modules (which cast their GEMM operands in BF16 mode and pre-split their
 * weights in F32 mode). */
enum { W2L_GEMM_TF32 = 0, W2L_GEMM_F32X3 = 1, W2L_GEMM_BF16 = 2, W2L_GEMM_F32X3_SPLIT_B = 3, W2L_GEMM_FP16 = 4 };
/* FP16 is BF16 mode with fp16 GEMM operands: the same layers cast the same operands, everything else is unchanged */
enum { W2L_PRECISION_TF32 = 0, W2L_PRECISION_F32 = 1, W2L_PRECISION_BF16 = 2, W2L_PRECISION_FP16 = 3 };
W2L_API int w2l_set_precision(int precision);
W2L_API int w2l_get_precision(void);
/* General form: A / B are fp32 (kinds TF32, F32X3), bf16 (kind BF16) or fp16 (kind FP16) with lda / ldb in ELEMENTS (rows
 * 16-byte aligned: ld % 4 for fp32, ld % 8 for 16-bit); C is fp32 or 16-bit (c_bf16; no accumulate / split-K then); aux
 * (the backward mask source) fp32 or 16-bit (aux_bf16).  A 16-bit C or aux is fp16 for kind FP16 and bf16 for every other
 * kind.  allow_overlap: operand rows may overlap (im2col views, see w2l_gemm_tf32_view). */
W2L_API int w2l_gemm(void* stream, int kind, int a_mn_major, int b_mn_major, int M, int N, int K, const void* A, int lda,
                     const void* B, int ldb, void* C, int ldc, int c_bf16, const float* bias, int act, int accumulate,
                     const void* aux, int ld_aux, int aux_bf16, int aux_mode, float aux_scale, float dropout_p,
                     unsigned long long seed, int allow_overlap);
/* fp32 -> bf16 (round to nearest even): flat, and row-wise with zero-padded columns (rows of `cols` floats, row stride
 * ld_in, to rows of cols_padded bf16) */
W2L_API int w2l_cast_bf16(void* stream, long long n, const float* x, void* y);
W2L_API int w2l_cast_bf16_rows(void* stream, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y);
/* the same to fp16 (round to nearest even; beyond 65504 becomes +-inf) */
W2L_API int w2l_cast_fp16(void* stream, long long n, const float* x, void* y);
W2L_API int w2l_cast_fp16_rows(void* stream, long long rows, int cols, int ld_in, int cols_padded, const float* x, void* y);
/* x [rows][cols] fp32 (row stride ld) -> the B planes of W2L_GEMM_F32X3_SPLIT_B, hi = tf32(x), lo = tf32(x - hi) (round to
 * nearest, ties away, as the F32X3 kernel rounds):
 *   transpose = 0: planes [2][rows][cols_padded], plane[r][c] from x[r][c]  (B = x K-major: the forward's weight)
 *   transpose = 1: planes [2][cols][cols_padded], plane[c][r] from x[r][c]  (B = x^T K-major: the data gradient's weight)
 * the columns of a plane past the source (c >= cols, resp. r >= rows) are zero. */
W2L_API int w2l_split_tf32(void* stream, int transpose, int rows, int cols, int ld, int cols_padded, const float* x, float* planes);
/* Pin the GEMM tile width (128 / 160 / 224 / 256; 0 = choose per shape, the default).  Thread-local; for tests and tuning. */
W2L_API int w2l_gemm_set_tile(int bn);
/* 1 (default): one CTA per SM walking the tiles, so the producer stages the next tile's operands during an epilogue;
 * 0: one CTA per tile.  Thread-local; for tests (the two must agree) and tuning. */
W2L_API int w2l_gemm_set_variant(int variant);
W2L_API int w2l_gemm_tf32(void* stream, int a_mn_major, int b_mn_major, int M, int N, int K, const float* A, int lda,
                          const float* B, int ldb, float* C, int ldc, const float* bias, int act);

/* Extended epilogue: after bias/act, (a) forward dropout with keep-scale 1/(1-p) (N % 4 == 0): one murmur3-style 32-bit
 * hash of (seed, (row*N + col) >> 1) per pair of columns, 16 bits per element, kept iff bits >= floor(p * 65536)
 * (DESIGN.md, "Dropout masks"), (b) backward activation mask read back from a stored activation tensor
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
 * The shape alone selects the kernels: where W % 8 == 0, stride <= kw and kw * max(Cin, Cout) <= 512 (for a strided
 * data gradient, ceil(kw / stride) taps per phase), the mma.sync tensor-core kernels (TF32 products, 3xTF32 under
 * W2L_PRECISION_F32); otherwise the fp32 SIMT kernels.
 * The workspace size call covers all three.
 * ---------------------------------------------------------------------------------------- */
W2L_API size_t w2l_conv_time_workspace_size(int B, int Tout, int Cin, int Cout, int K);
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
/* the same with 16-bit destination operands, written directly: out_bf16 = 1 bf16 (W2L_PRECISION_BF16), 2 fp16
 * (W2L_PRECISION_FP16); 0 is fp32 */
W2L_API int w2l_conv1d_arrange_ex(void* stream, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split, const float* w,
                                  const float* bias, void* fwd, void* flip, float* bias_p, int out_bf16);
W2L_API int w2l_conv1d_unarrange_grad(void* stream, int cin, int cout, int kw, int cin_p, int cout_p, int glu_split,
                                      const float* dfwd, float* dw, long long rows, const float* dy, float* dbias);
W2L_API int w2l_glu_fwd(void* stream, long long rows, int half, const float* x, float* y, float dropout_p,
                        unsigned long long seed);
W2L_API int w2l_glu_bwd(void* stream, long long rows, int half, const float* x, const float* dy, float* dx, float dropout_p,
                        unsigned long long seed);
/* PReLU with one parameter (arch opcode `PR`, fl::PReLU): y[i] = (x[i] >= 0 ? x[i] : a[0] x[i]) * mask(i), the following
 * Dropout fused (mask = dropout_scale's Philox rule, regenerated from `seed` in the backward).  The backward writes
 * dx[i] = mask(i) dy[i] (x[i] >= 0 ? 1 : a[0]) and da[0] = sum_{x[i] < 0} x[i] mask(i) dy[i] (per-CTA partials and one
 * fixed-order sum: the same bits every run).  `a` stays on the device: no host sync. */
W2L_API int w2l_prelu_fwd(void* stream, long long n, const float* x, const float* a, float* y, float dropout_p,
                          unsigned long long seed);
W2L_API int w2l_prelu_bwd(void* stream, long long n, const float* x, const float* dy, const float* a, float* dx, float* da,
                          float dropout_p, unsigned long long seed);

/* fl::LayerNorm over a whole sample (R = T*C*W elements; `LN 0 1 2` / TDSBlock with lnIncludeTime)
 * with scalar gain/bias (device scalars, nullable = 1/0) and a fused residual: y = LN(a + r).
 * mean_rstd [B][2] is saved for the backward pass; scratch = W2L_LN_SCRATCH_DOUBLES(B) doubles (one partial
 * pair per CTA: no zero-fill, no atomics, deterministic).  Where a group's mean is far above its spread, the statistics
 * are summed about a pivot taken from the group (the mean of its first 32 values), so that costs no accuracy, and a
 * constant group comes out exactly `bias`; other groups keep plain sums.
 * Backward: d_res = ds, d_branch = ds * mask(a) where the mask undoes the fused ReLU/dropout of the
 * branch that produced `a` (branch_mode 0 none, 1 (a>0)*scale, 2 (a!=0)*scale); dgain/dbias accumulate. */
#define W2L_LN_MAX_PARTS 80
#define W2L_LN_SCRATCH_DOUBLES(B) (2 * W2L_LN_MAX_PARTS * (size_t)(B))
W2L_API int w2l_layernorm_fwd(void* stream, int B, long long R, float eps, const float* a, const float* r,
                              const float* gain, const float* bias, float* y, float* mean_rstd, double* scratch);
/* The forward of w2l_layernorm_fwd always on its one-warp-per-group kernel (G groups of R floats, no scratch).
 * w2l_layernorm_fwd picks between that kernel and a two-pass one by the group count, and their mean / rstd round
 * differently; here a group's result depends on its own R values only, whatever G is.  The streaming acoustic model
 * relies on that: its per-frame LayerNorms see batches whose row count depends on the other streams in the call. */
W2L_API int w2l_layernorm_rows_fwd(void* stream, long long G, int R, float eps, const float* a, const float* r, const float* gain,
                                   const float* bias, float* y, float* mean_rstd);
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
/* one single-thread kernel that sleeps about `us` microseconds (at most 1e6); tests use it to hold a stream back */
W2L_API int w2l_delay(void* stream, int us);
W2L_API int w2l_act_fwd(void* stream, long long n, const float* x, int relu, float dropout_p, unsigned long long seed, float* y);
W2L_API int w2l_mask_mul(void* stream, long long n, const float* g, const float* ref, int mode, float scale, float* out);

/* ----------------------------------------------------------------------------------------
 * MFSC features (`--mfsc --filterbanks=F`, fl::lib::audio::Mfsc with Train.cpp:288-290's settings, then the dataset's
 * per-utterance or local normalisation, Train.cpp:311-315): raw audio in, the trainer's input out.
 *   frame = round(sample_rate * frame_ms / 1000) samples (halves up), stride likewise; frames of an utterance of n samples:
 *   n < frame ? 0 : 1 + (n - frame) / stride (no padding) — w2l_mfsc_num_frames (-1 on bad parameters).
 *   Per frame: pre-emphasis 0.97, Hamming window, |rfft| over nfft = the next power of two >= frame, F triangular filters
 *   on the HTK mel scale between 0 and sample_rate/2, log(max(x, 1)).  The mel floor of 1 assumes samples at 16-bit
 *   integer scale.  Then mean / population standard deviation (a std <= 1e-5 counts as 1) over the whole utterance
 *   (left_ctx = 0) or, for frame t, over frames max(0, t - left_ctx) .. t (left_ctx > 0: the streaming LocalNorm(F,
 *   left_ctx, 0) of inference/module/nn/LocalNorm.cpp).
 *   audio float [B][max_samples] (device), n_samples_host int32 [B] (host, each <= max_samples);
 *   features float [B][F][T_out] = ArrayFire [T_out,F,1,B], T_out >= the longest utterance's frame count; frames
 *   t >= T_b of utterance b are 0.  Deterministic (no floating-point atomics).  The DFT is an fp32-accurate (3xTF32)
 *   GEMM whatever w2l_set_precision says.  W2L_ERR_UNSUPPORTED: a stride that is not a multiple of 4 samples (e.g.
 *   10 ms at 22.05 kHz), frames over 2048 samples, more than 256 filters.
 * ---------------------------------------------------------------------------------------- */
W2L_API int w2l_mfsc_num_frames(int n_samples, int sample_rate, int frame_ms, int stride_ms);
W2L_API size_t w2l_mfsc_workspace_size(int B, int max_samples, int sample_rate, int frame_ms, int stride_ms, int n_filters);
W2L_API int w2l_mfsc(void* stream, int B, int max_samples, const float* audio, const int32_t* n_samples_host, int sample_rate,
                     int frame_ms, int stride_ms, int n_filters, int left_ctx, float* features, int T_out, void* ws,
                     size_t ws_bytes);

/* ----------------------------------------------------------------------------------------
 * Training-step driver:the body of the reference loop (recipes/slimIPL/src/Train.cpp:1454-1803) written
 * in C++ against include/fl_compat/fl_compat.h — network forward, criterion, loss.backward(), NCCL
 * all-reduce of every gradient, division by the global batch size, clipGradNorm over net U criterion (over the
 * network alone for "linseg", whose transitions step unclipped, as Train.cpp's --linseg warm start does),
 * criterion + network SGD steps.  `arch_text` is a wav2letter arch file (opcodes V RO PD C2 R DO LN TDS L
 * SAUG), `criterion` "ctc", "asg" or "linseg".  All pointers below are DEVICE pointers:
 * features [T,F,1,B] (ArrayFire layout, T fastest), target [L,B] int32 (-1 padded), loss_out [B].
 * Returns NULL / a status code; w2l_last_error() has the text.
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_trainer_create(void* stream, const char* arch_text, int n_feat, int n_label, const char* criterion,
                                 int scale_mode, float transdiag, float lr, float lrcrit, float momentum, float maxgradnorm);
/* The seq2seq criterion (Train.cpp:411-432; DESIGN.md §9): the arch's output is the encoder, 2 * hidden features per
 * frame; n_label counts the dictionary with eos and pad.  rounds = --decoderattnround, layers = --decoderrnnlayer,
 * dropout = --decoderdropout, label_smooth = --labelsmooth, pct_teacher_forcing = --pctteacherforcing, window_std =
 * --softwstd of a SoftPretrainWindow (0: no window), train_with_window = --trainWithWindow.  Targets [U,B] hold tokens,
 * then eos, then pad; an utterance with a value outside [0, n_label) (-1 included) gets a NaN loss, so the step's
 * update is skipped and counted (w2l_trainer_status), with no host synchronisation.  Its parameters form the criterion arena: they step with lrcrit
 * and momentum 0 and are clipped with the network.  In its checkpoints (the same version 2 container) the settings and the
 * window flag follow the arch text. */
W2L_API void* w2l_trainer_create_seq2seq(void* stream, const char* arch_text, int n_feat, int n_label, int hidden, int eos, int pad,
                                         int max_decoder_output_len, int rounds, int layers, float dropout, float label_smooth,
                                         int pct_teacher_forcing, float window_std, int train_with_window, float lr, float lrcrit, float momentum,
                                         float maxgradnorm);
/* features per frame of the network output (n_label; 2 * hidden for seq2seq) */
W2L_API int w2l_trainer_output_width(void* trainer, int* width);
/* seq2seq only: {hidden, eos, pad, maxdecoderoutputlen, rounds, layers, window still set} */
W2L_API int w2l_trainer_seq2seq_config(void* trainer, int* config7);
/* seq2seq only: clearWindow() after the --pretrainWindow updates (Train.cpp:1885-1910) */
W2L_API int w2l_trainer_clear_window(void* trainer);
/* seq2seq only: the Philox seed of the last training forward (substitutions: that seed; the dropout after layer k of the
 * flattened round-major stack: seed + 1 + k) */
W2L_API int w2l_trainer_seq2seq_seed(void* trainer, unsigned long long* seed);
/* seq2seq only: eval-mode network forward, then the greedy decode of every utterance: tokens device int32
 * [B][maxdecoderoutputlen] padded with pad (capacity elements), lengths device int32 [B] (eos not counted) */
W2L_API int w2l_trainer_decode(void* trainer, void* stream, int B, int T, const float* features, int32_t* tokens, int32_t* lengths,
                               long long capacity);
/* seq2seq only: eval-mode network forward, then Seq2SeqCriterion::beamSearchBatch with beam K (1..16) and max_len steps
 * (0: maxdecoderoutputlen): tokens device int32 [B][K][max_len] (capacity elements) padded with pad, lengths int32 and
 * scores float [B][K], counts int32 [B]; slots at or beyond counts[b] hold pad, length 0 and score -inf */
W2L_API int w2l_trainer_beam_search(void* trainer, void* stream, int B, int T, const float* features, int beam, int max_len, int32_t* tokens,
                                    int32_t* lengths, float* scores, int32_t* counts, long long capacity);
W2L_API void w2l_trainer_destroy(void* trainer);
/* train != 0: backward, clip and update; total_batch (the batch summed over ranks, which divides every gradient) must
 * then be finite and > 0, else W2L_ERR_INVALID_ARGUMENT and nothing runs.  train == 0: loss only, total_batch unused. */
W2L_API int w2l_trainer_step(void* trainer, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                             float* loss_out, int train, float total_batch);
/* Padded batches of the seq2seq criterion (DESIGN.md §9): the step, decode and beam search above with the durations and
 * target sizes Train.cpp passes it.  input_sizes [B] device int32 (nullable) are the input frame counts of each
 * utterance: the attention of utterance b covers encoder frames t < T'_b = ceil(d_b T' / max d); target_sizes [B]
 * device int32 (nullable, step only) count tokens plus eos and centre the soft window at u T'_b / U_b.  Bad sizes give
 * that utterance a NaN loss (the update is skipped and counted), checked on the device.  Both NULL: the unsized call,
 * bit for bit.  A ctc, asg or linseg trainer given sizes returns W2L_ERR_INVALID_ARGUMENT: Train.cpp gives them none. */
W2L_API int w2l_trainer_step_sized(void* trainer, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                                   const int32_t* input_sizes, const int32_t* target_sizes, float* loss_out, int train, float total_batch);
W2L_API int w2l_trainer_decode_sized(void* trainer, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int32_t* tokens,
                                     int32_t* lengths, long long capacity);
W2L_API int w2l_trainer_beam_search_sized(void* trainer, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int beam,
                                          int max_len, int32_t* tokens, int32_t* lengths, float* scores, int32_t* counts, long long capacity);
/* eval-mode network output [B][T'][width] into emissions_out (capacity floats); T' through t_out.  A buffer smaller than
 * B T' width returns W2L_ERR_INVALID_ARGUMENT with nothing written to it, and t_out still set: call again with that size. */
W2L_API int w2l_trainer_forward(void* trainer, void* stream, int B, int T, const float* features, float* emissions_out,
                                long long capacity, int* t_out);
/* slimIPL (recipes/slimIPL/src/Train.cpp; DESIGN.md §7).
 * set_ema (--slimIPL_ema / --slimIPL_ema_decay): on = 1 builds the teacher, a second network from the same arch text or
 * plugin with its own value arena, copied from the network as it is now (a second call restarts it from the network);
 * on = 0 drops it.  Every training call (step, step_sized, step_soft) then runs ema = ema * decay + net * (1 - decay)
 * once after the optimizer (w2l_ema_update), also after a skipped update and once per batch under mixed-precision
 * retries; eval steps do not.  Only the network is averaged.  Without a teacher, "the teacher" below is the network.
 * w2l_trainer_ema reads the setting back.  num_params / param_layout / get_flat / set_flat take which = 2 for the
 * teacher's values (get_flat: what = 0 only).
 * forward_teacher: w2l_trainer_forward of the network (teacher = 0) or of the teacher (soft pseudo-labels, :1413-1415).
 * viterbi_path: eval-mode forward of the network or teacher, then crit->viterbiPath (:1362-1407): CTC the per-frame
 * argmax, ASG / LinSeg the FCC Viterbi path, seq2seq the greedy decode.  path device int32 [B][T'] (seq2seq
 * [B][maxdecoderoutputlen], padded with pad; capacity elements); T' (or maxdecoderoutputlen) through t_out.  input_sizes:
 * seq2seq only, as in step_sized; the CTC and ASG paths cover all T' frames of a padded batch, as Train.cpp's.
 * step_soft: a training step whose loss is the soft-label loss (w2l_soft_label_loss, :1663-1673) of the train-mode
 * output against teacher_logits, device [B][t_teacher][output width] (another shape: W2L_ERR_INVALID_ARGUMENT), scaled
 * by soft_scale (--slimIPL_soft_scale); loss_out receives one float.  Backward, all-reduce, clip, finite guard, loss
 * scaling and update are the step's; the criterion gets a zero gradient.  total_batch: the world size (the loss is one
 * scalar per rank, :1743-1747). */
W2L_API int w2l_trainer_set_ema(void* trainer, void* stream, int on, double decay);
W2L_API int w2l_trainer_ema(void* trainer, int* on, double* decay);
W2L_API int w2l_trainer_forward_teacher(void* trainer, void* stream, int B, int T, const float* features, int teacher, float* emissions_out,
                                        long long capacity, int* t_out);
W2L_API int w2l_trainer_viterbi_path(void* trainer, void* stream, int B, int T, const float* features, const int32_t* input_sizes, int teacher,
                                     int32_t* path, long long capacity, int* t_out);
W2L_API int w2l_trainer_step_soft(void* trainer, void* stream, int B, int T, const float* features, const float* teacher_logits, int t_teacher,
                                  float soft_scale, float* loss_out, float total_batch);
/* Forced alignment: the eval-mode network forward of w2l_trainer_forward, then the criterion's viterbiPathWithTarget on
 * its emissions.  path / idx: device int32 [B][T'] (capacity elements each; idx nullable), T' through t_out.  CTC:
 * w2l_ctc_viterbi_target, idx = extended-target state.  ASG / LinSeg: w2l_fac_viterbi with the criterion's transitions,
 * idx = target position.  A target that cannot be aligned gives -1 over its whole row. */
W2L_API int w2l_trainer_align(void* trainer, void* stream, int B, int T, const float* features, int L, const int32_t* target,
                              int32_t* path, int32_t* idx, long long capacity, int* t_out);
/* input frames per output frame: the product of the time strides of the network's convolutions */
W2L_API int w2l_trainer_time_stride(void* trainer);
/* 1 (default): the backward pass computes the Linear layers' weight and bias gradients on a second stream of the
 * trainer, beside the data-gradient chain; 0: everything on the caller's stream.  Results are bit-identical either way. */
W2L_API int w2l_trainer_set_grad_stream(void* trainer, int on);
/* tests: queue a w2l_delay of `us` microseconds on the gradient stream before each piece of work handed to it, so a
 * missing wait or an early free shows up as a changed result (0, the default: none) */
W2L_API int w2l_trainer_set_grad_stream_delay(void* trainer, int us);
/* precision of the trainer's dense contractions (W2L_PRECISION_*; default: the creating thread's w2l_set_precision) */
W2L_API int w2l_trainer_set_precision(void* trainer, int precision);
/* Learning-rate schedule of Train.cpp:1169-1175, 1334-1348, applied on the host at every training step (no launch, no
 * sync): with curBatch = the step's 1-based update number and curEpoch = the position's epoch,
 *   lr = lr0 * 0.5^(curEpoch < lr_decay ? 0 : 1 + (curEpoch - lr_decay) / lr_decay_step)
 *            * (lrcosine ? cos(pi/2 * curBatch / nbatches) : gamma^(curBatch / stepsize)) * min(curBatch / warmup, 1)
 * in double, rounded to float; lrcrit the same from its lr0.  lr0 / lrcrit0 are w2l_trainer_create's lr / lrcrit (or
 * w2l_trainer_set_lr's).  Every training step counts, including one whose update the finite guard skips.  Defaults
 * (flashlight's flag defaults; the factor is then exactly 1): warmup 1, gamma 1, stepsize, nbatches, lr_decay and
 * lr_decay_step INT64_MAX, lrcosine 0.  warmup = 0 means no warmup.
 * set_position: the updates already taken (curBatch before the next step) and the epoch (Train.cpp's curEpoch, which is 1
 * during the first epoch); w2l_trainer_position reads them back; w2l_trainer_lr gives the rates the next step uses. */
W2L_API int w2l_trainer_set_schedule(void* trainer, long long warmup, double gamma, long long stepsize, int lrcosine, long long nbatches,
                                     long long lr_decay, long long lr_decay_step);
W2L_API int w2l_trainer_set_position(void* trainer, long long update, long long epoch);
W2L_API int w2l_trainer_position(void* trainer, long long* update, long long* epoch);
W2L_API int w2l_trainer_set_lr(void* trainer, float lr, float lrcrit);
W2L_API int w2l_trainer_lr(void* trainer, float* lr, float* lrcrit);
/* Mixed-precision loss scaling (Train.cpp:1135-1140, 1681-1684, 1748-1790, 1806-1818; --fl_amp_use_mixed_precision).
 * With on = 1, each training step seeds the criterion's loss gradient with the scale (every backward tensor carries it)
 * and divides it out in the update (gradients / (total_batch * scale)).  A step whose loss is finite and whose gradient
 * is not, while scale >= min_scale, halves the scale and runs the same batch again on the same dropout seeds and
 * SpecAugment bands (upstream draws new ones), so a retried step equals a first attempt at the final scale; it reads one
 * flag from the device per attempt.  Otherwise a non-finite step is skipped and counted as before.  After each step the
 * scale grows, below max_scale: x2 when the attempt counter (unsigned short, incremented per attempt, wrapping to 0,
 * reset to 1 by a non-finite gradient) is a multiple of update_interval, else +2.  Reference defaults: 4096, 2000,
 * 32000, min_scale 1e-4 (flashlight's kAmpMinimumScaleFactorValue).  Loss scaling works in every precision and pays in
 * fp16.  set_amp resets the counter to 1 and the retry count to 0.  amp_state: the scale the next step starts at, the
 * counter and the number of retried attempts; host state, no sync. */
W2L_API int w2l_trainer_set_amp(void* trainer, int on, double initial_scale, int update_interval, double max_scale, double min_scale);
W2L_API int w2l_trainer_amp_state(void* trainer, void* stream, double* scale, int* counter, long long* retries);
/* steps whose update was skipped on the device because the loss or a gradient was NaN / Inf (Train.cpp:1686-1698,
 * :1753-1771); synchronises `stream` */
W2L_API int w2l_trainer_status(void* trainer, void* stream, long long* skipped_steps);
W2L_API long long w2l_trainer_num_params(void* trainer, int which /*0 network, 1 criterion, 2 teacher*/);
W2L_API int w2l_trainer_param_layout(void* trainer, int which, int max_params, long long* elements, long long* dims4);
W2L_API int w2l_trainer_get_flat(void* trainer, void* stream, int which, int what /*0 values, 1 gradients*/, float* out);
W2L_API int w2l_trainer_set_flat(void* trainer, void* stream, int which, const float* in);
W2L_API int w2l_trainer_sync_parameters(void* trainer, void* stream);   /* fl::allReduceParameters, Train.cpp:1078-1079 */
W2L_API const char* w2l_trainer_describe(void* trainer);
/* Checkpoints (SURVEY.md §8 f4; the role of Serializer::save / load in Train.cpp:747-800): own little-endian container with
 * the constructor arguments + parameter / momentum arenas of network and criterion, the position and the learning-rate
 * schedule; load rebuilds the trainer.  Files written before the schedule existed load with position 0 and the default
 * schedule.  A trainer with a teacher writes version 4 (version 2 followed by the decay and the teacher's values); one
 * without writes version 2 as before. */
W2L_API int w2l_trainer_save(void* trainer, void* stream, const char* path);
W2L_API void* w2l_trainer_load(void* stream, const char* path);
/* Export for the in-tree streaming inference stack, following the conversions of
 * recipes/streaming_convnets/tools/StreamingTDSModelConverter.cpp:46-136,203-283: every layer's arrays in the inference
 * library's layouts (acoustic_model.json + acoustic_model.bin), transitions.bin (ASG; the cereal std::vector<float> the
 * inference examples read, :310-326) and tokens.txt (tokens_text nullable).  Streaming TDS archs only (LN 1 2), like the converter. */
W2L_API int w2l_trainer_export_streaming(void* trainer, void* stream, const char* outdir, const char* tokens_text);
/* ----------------------------------------------------------------------------------------
 * Streaming acoustic model: a trained streaming TDS network run chunk by chunk over many concurrent streams, with the
 * semantics of the in-tree inference library (recipes/streaming_convnets/inference/inference/module/nn: Sequential,
 * Conv1dFbGemm start / run / finish, TDSBlock, Residual, LayerNorm, Linear, Relu).  Per stream, the emissions of all
 * run calls and the finishing one, put end to end, have the frame count of the eval-mode w2l_trainer_forward on the
 * whole utterance and its values up to the rounding of the LayerNorm statistics (the runtime always takes the
 * one-warp-per-frame kernel, w2l_layernorm_rows_fwd).  They are the same bits whatever the split into chunks and
 * whatever other streams share the calls (DESIGN.md §4).  Only the convolutions keep state, per stream slot:
 *   start  holds pad_left zero frames;
 *   run    appends the new frames; with avail frames held, nOut = (avail - kw) / stride + 1 frames come out when
 *          avail >= kw, and nOut * stride are consumed (at most kw - 1 stay);
 *   finish appends pad_right zero frames, then runs.
 * The padding of every convolution is the export's (w2l_trainer_export_streaming).  Frame counts are integer arithmetic
 * on the host: a run call neither reads from the device nor synchronises, and returns the output frame counts at once.
 * Calls on one handle must be ordered (one CUDA stream, or the caller's synchronisation).
 *
 *   w2l_stream_create   snapshots the trainer's network parameters and its criterion (kind; ASG / LinSeg transitions)
 *                       (training may go on), takes the calling thread's
 *                       w2l_set_precision, and allocates all state and per-call buffers for max_streams slots (at most
 *                       1024) and chunks of at most max_chunk frames.  Accepts exactly the archs the export accepts,
 *                       with its error text.  NULL on failure (w2l_last_error).
 *   w2l_stream_state_bytes   device bytes of carried state per slot (two planes of the held frames of every convolution,
 *                       and for ASG / LinSeg the Viterbi scores and the backpointers of the uncommitted frames)
 *   w2l_stream_max_frames_out  the most output frames one call can give a stream (sizes the emission buffer)
 *   w2l_stream_start    resets the n slots (host int slots[n]) and holds their left padding; a running slot forgets its
 *                       past, its path included
 *   w2l_stream_run      slots[n], frames_in[n] (host ints, each <= Tc <= max_chunk), features device [n][1][nFeat][Tc]
 *                       (ArrayFire [Tc,nFeat,1,n], the trainer's layout); emissions device [n][T'max][nLabel] with
 *                       T'max = max frames_out, rows t >= frames_out[i] of stream i unspecified; capacity in floats;
 *                       frames_out[n] host.  finish = 1 appends every layer's right padding after the chunk, and the
 *                       slot stays finished until the next start.  Errors (W2L_ERR_INVALID_ARGUMENT): a slot out of range
 *                       or listed twice, a slot not started or already finished, a chunk longer than Tc, Tc > max_chunk,
 *                       too small a capacity.
 *   w2l_stream_run_path   w2l_stream_run, then the criterion's viterbiPath of the call's output frames, carried per
 *                       slot (w2l_stream_run is this call without a path).  path device int32 [n][P] with
 *                       P = w2l_stream_max_path_out, path_capacity in ints (>= n * P); path_info device int32 [n][3]:
 *                       {stream frame index of the first entry committed in this call, entries committed in this call,
 *                       forced frames so far}.  emissions may be NULL (nothing is copied out; capacity is then unused).
 *                       Per stream, the entries of every call and of finish put end to end are, bit for bit, the
 *                       criterion's viterbiPath of its emissions put end to end, whatever the chunking and the other
 *                       streams: CTC w2l_argmax_path (every frame commits at once); ASG / LinSeg w2l_fcc_viterbi (N <= 32)
 *                       or w2l_fcc_viterbi64 (N <= 64), carried un-re-centred, committing each call every frame up to the
 *                       newest one at which all N states' traced-back paths agree, and on finish the rest along the
 *                       first-maximum end state.  The one exception: a slot holding more than 1024 uncommitted frames
 *                       commits its oldest along the current first-maximum state's path, and counts them as forced.
 *                       A path covers the output frames of the calls that asked for one.  Neither reads from the device
 *                       nor synchronises.  W2L_ERR_UNSUPPORTED: the criterion has no streaming path (ASG / LinSeg over
 *                       64 tokens); W2L_ERR_INVALID_ARGUMENT as w2l_stream_run, and a path_capacity below n * P.
 *   w2l_stream_max_path_out  P: the most path entries one call can commit per stream (0: no streaming path)
 *   w2l_stream_plan     host only: the frame bookkeeping of one stream over n_calls calls of frames_host[k] frames (the
 *                       last one finishing when finish_last), for every convolution c of the arch: conv_spec_host
 *                       [c][4] = {kw, stride, pad_left, pad_right}, frames_out_host[k][max_convs] and tails_host
 *                       [k][max_convs] (frames held after call k); n_convs gets the convolution count.
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_stream_create(void* trainer, void* stream, int max_streams, int max_chunk);
W2L_API void w2l_stream_destroy(void* s);
W2L_API long long w2l_stream_state_bytes(void* s);
W2L_API int w2l_stream_max_frames_out(void* s);
W2L_API int w2l_stream_start(void* s, void* stream, int n, const int* slots);
W2L_API int w2l_stream_run(void* s, void* stream, int n, const int* slots, const int* frames_in, const float* features, int Tc, int finish,
                           float* emissions, long long capacity, int* frames_out);
W2L_API int w2l_stream_run_path(void* s, void* stream, int n, const int* slots, const int* frames_in, const float* features, int Tc,
                                int finish, float* emissions, long long capacity, int* frames_out, int32_t* path, long long path_capacity,
                                int32_t* path_info);
W2L_API int w2l_stream_max_path_out(void* s);
W2L_API int w2l_stream_plan(const char* arch_text, int n_feat, int n_label, int n_calls, const int* frames_host, int finish_last,
                            int max_convs, int* n_convs, int* conv_spec_host, int* frames_out_host, int* tails_host);
/* ----------------------------------------------------------------------------------------
 * Streaming MFSC front end: raw audio chunk by chunk over many concurrent streams, with the semantics of the in-tree
 * inference library's feature module (inference/module/feature/LogMelFeature.cpp, then LocalNorm(F, left_ctx, 0) of
 * inference/module/nn/LocalNorm.cpp).  Its output is the features argument of w2l_stream_run.  Per stream, the features
 * of all run calls put end to end are the same bits whatever the split into chunks and whatever other streams share
 * the calls, and match w2l_mfsc(..., left_ctx) of the whole stream up to the order of the window sums (DESIGN.md §4).
 *   Settings: the frame and stride rounding, the mel filters, the log floor, the sample scale and the W2L_ERR_UNSUPPORTED
 *   limits of w2l_mfsc (stride a multiple of 4 samples, frames up to 2048 samples, at most 256 filters).  left_ctx >= 1:
 *   per-utterance normalisation (w2l_mfsc's left_ctx = 0) cannot be computed causally.
 *   start  holds nothing;
 *   run    appends samples_in[i] samples; with avail samples held, frames = avail < frame ? 0 : 1 + (avail - frame) /
 *          stride come out and frames * stride samples are consumed (fewer than frame stay);
 *   finish runs, then drops the remainder (no right padding); the slot refuses run until the next start.
 *   A stream's frame g (counted from start) is normalised over its frames max(0, g - left_ctx) .. g: mean and population
 *   standard deviation, a std <= 1e-5 counting as 1.
 * Frame counts are integer arithmetic on the host: a run call neither reads from the device nor synchronises.  The DFT
 * is an fp32-accurate (3xTF32) GEMM whatever w2l_set_precision says.  Calls on one handle must be ordered.
 *
 *   w2l_mfsc_stream_create   allocates state and per-call buffers for max_streams slots (at most 1024) and chunks of at
 *                            most max_chunk_samples samples (at most 65535) and builds the DFT basis and the filters.
 *                            Checks every argument before its first CUDA call.  NULL on failure (w2l_last_error).
 *   w2l_mfsc_stream_state_bytes     device bytes of carried state per slot (two planes of the held samples and of the
 *                                   held per-frame sums)
 *   w2l_mfsc_stream_max_frames_out  the most frames one call can give a stream (sizes the feature buffer)
 *   w2l_mfsc_stream_start    resets the n slots (host int slots[n]); a running slot forgets its past
 *   w2l_mfsc_stream_run      slots[n], samples_in[n] (host ints, each <= Sc <= max_chunk_samples), audio device [n][Sc];
 *                            features device [n][1][F][Tf] (ArrayFire [Tf,F,1,n], the trainer's layout) with Tf = max
 *                            frames_out, frames t >= frames_out[i] of stream i are 0; capacity in floats; frames_out[n]
 *                            host.  Errors (W2L_ERR_INVALID_ARGUMENT): a slot out of range or listed twice, a slot not
 *                            started or already finished, samples_in[i] > Sc, Sc > max_chunk_samples, too small a capacity.
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_mfsc_stream_create(void* stream, int max_streams, int max_chunk_samples, int sample_rate, int frame_ms, int stride_ms,
                                     int n_filters, int left_ctx);
W2L_API void w2l_mfsc_stream_destroy(void* h);
W2L_API long long w2l_mfsc_stream_state_bytes(void* h);
W2L_API int w2l_mfsc_stream_max_frames_out(void* h);
W2L_API int w2l_mfsc_stream_start(void* h, void* stream, int n, const int* slots);
W2L_API int w2l_mfsc_stream_run(void* h, void* stream, int n, const int* slots, const int* samples_in, const float* audio, int Sc, int finish,
                                float* features, long long capacity, int* frames_out);
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
/* Word timings of one aligned utterance (host pointers): target[len] (-1 padded) and idx[n_frames] from
 * w2l_trainer_align (CTC: extended-target state, ASG: target position).  Writes one `.align` line without its newline,
 * NUL-terminated (returns the bytes needed, terminator included; -1 on error):
 *   utt_id TAB seg \n seg \n ... (segments joined by the two characters backslash, n)
 * with seg = "utt_id 1 <begin s> <duration s> <word>", a silence segment having the word "$".  A target position
 * belongs to a word or to silence: the word separator and --surround tokens are silence and end the word, a token that
 * starts with the word separator (word pieces) starts a word, a replabel belongs to the token before it.  A word runs
 * from the first to the last frame whose state maps into it (CTC blanks inside it included); the frames before, between
 * and after words are "$" segments, and the line always starts with one (of zero duration when the first word starts
 * at frame 0).  Time = frame * ms_per_frame / 1000.  An idx of -1 (no alignment) is an error. */
W2L_API long long w2l_text_align_words(void* text, const int32_t* target, int len, const int32_t* idx, int n_frames,
                                       double ms_per_frame, const char* utt_id, char* out, long long cap);
/* out4 += {reference length, deletions, insertions, substitutions} of one (hypothesis, reference) pair */
W2L_API int w2l_edit_distance(const char* hyp, const char* ref, long long* out4);

/* ----------------------------------------------------------------------------------------
 * The same scoring on the device, for a whole batch (csrc/text_eval.cu; DESIGN.md §10).
 *   w2l_text_device_create  device tables of a w2l_text_create handle, built once with its own Dictionary and splitWrd:
 *                           each token's role (replabel <k>, or unspellable), its letters (CSR of letter ids: the
 *                           splitWrd code points with --usewordpiece, else the whole token), each letter's bytes, the
 *                           blank / eos / pad / <SIL> / surround indices and the separator's letter id.  Synchronises
 *                           `stream` once.  NULL on error.  The text handle may be destroyed afterwards.
 *   w2l_text_edit_counts    counts[B][8] = {reference letters, deletions, insertions, substitutions, reference words,
 *                           deletions, insertions, substitutions} of hypothesis row b of paths[B][n_path] (its first
 *                           path_lengths[b] entries when path_lengths is non-NULL) against target row b of targets[B][L],
 *                           exactly as w2l_text_prediction2ltr / target2ltr / ltr2wrd / w2l_edit_distance give them.
 *                           Where the host pipeline throws (a token outside the dictionary reaches the letters, a path
 *                           length outside [0, n_path]) that utterance's eight counts are -1.  Two kernels, no host sync.
 *                           Limit: n_path and L each times (1 + replabel) times the longest token's letter count
 *                           <= 1 048 576, else W2L_ERR_UNSUPPORTED and nothing is launched.
 *   w2l_text_edit_workspace_size   its workspace in bytes (0 outside the limit, with the error text set).
 * ---------------------------------------------------------------------------------------- */
W2L_API void* w2l_text_device_create(void* text, void* stream);
W2L_API void w2l_text_device_destroy(void* dev_text);
W2L_API size_t w2l_text_edit_workspace_size(void* dev_text, int B, int n_path, int L);
W2L_API int w2l_text_edit_counts(void* dev_text, void* stream, int B, int n_path, const int32_t* paths, const int32_t* path_lengths, int L,
                                 const int32_t* targets, int32_t* counts, void* ws, size_t ws_bytes);
/* Train.cpp's test() for one batch (:965-980 with evalOutput :829-872): the eval-mode forward, the criterion's eval loss
 * into loss[B] (the bits of w2l_trainer_step with train = 0), the criterion's viterbiPath (CTC argmax, ASG / LinSeg FCC
 * Viterbi, seq2seq greedy decode with input_sizes) and w2l_text_edit_counts of it against target into counts[B][8].
 * input_sizes / target_sizes as in w2l_trainer_step_sized (seq2seq only).  The only host read is the greedy decode's. */
W2L_API int w2l_trainer_evaluate(void* trainer, void* stream, void* dev_text, int B, int T, const float* features, int L, const int32_t* target,
                                 const int32_t* input_sizes, const int32_t* target_sizes, float* loss, int32_t* counts);

#ifdef __cplusplus
}
#endif
#endif /* W2L_B200_H_ */
