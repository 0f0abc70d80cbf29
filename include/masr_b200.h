/* masr_b200 — C ABI of the H100-native MASR inference hot path.
 *
 * The reference (yeyupiaoling/MASR) is pure Python and has NO FFI of its own: its hot path is
 * `MASRPredictor.predict / predict_stream` (masr/predict.py:167,237) -> `AudioFeaturizer.featurize`
 * (masr/data_utils/featurizer/audio_featurizer.py:37) -> `InferencePredictor.predict[_chunk_*]`
 * (masr/infer_utils/inference_predictor.py:52,80) -> TorchScript `get_encoder_out[_chunk]`
 * (masr/model_utils/conformer/model.py:152,169) -> `greedy_decoder` (masr/decoders/ctc_greedy_decoder.py:6).
 * Every library call on that path (torchaudio kaldi.fbank, ATen linear/conv/layer_norm/softmax, numpy
 * argmax) is replaced by one of the entry points below; the Python host code in `masr_b200/` binds them
 * with ctypes and keeps the reference's class/method interface.  INTEGRATION.md shows the stub a MASR
 * maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer (caller-owned, allocated e.g. with torch.empty(device='cuda'))
 *     unless its name ends in `_host`; nothing is allocated, freed or retained by the library;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued asynchronously on it;
 *   - float32 everywhere ("f32" suffix), row-major, leading dimensions (`ld*`) in elements;
 *   - returns MASR_OK (0) or an error code; `masr_last_error()` has the message (thread-local);
 *   - there is no CPU fallback: without an sm_90 device the calls fail.
 */
#ifndef MASR_B200_H_
#define MASR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MASR_ABI_VERSION 1

enum {
    MASR_OK = 0,
    MASR_ERR_INVALID_ARGUMENT = 10001,
    MASR_ERR_UNSUPPORTED_DEVICE = 10002,
    MASR_ERR_INTERNAL = 10003,
};

/* per-utterance status flags written by masr_wave_gain_f32 */
enum { MASR_STATUS_GAIN_EXCEEDED = 1 };

/* GEMM epilogues */
enum {
    MASR_EPI_BIAS = 0,      /* C = A.W^T + bias                                              */
    MASR_EPI_BIAS_SILU = 1, /* C = silu(A.W^T + bias)                  positionwise.py:37    */
    MASR_EPI_BIAS_RELU = 2, /* C = relu(A.W^T + bias)                  subsampling.py:82,84  */
    MASR_EPI_BIAS_GLU = 3,  /* C[:, j] = v[2j] * sigmoid(v[2j+1])      convolution.py:118    */
    MASR_EPI_BIAS_SCALE = 4,/* C = (A.W^T + bias) * alpha              embedding.py:98       */
    MASR_EPI_RESIDUAL = 5,  /* C = residual + alpha * (A.W^T + bias)   encoder.py:117,131,145,155 */
};

const char* masr_last_error(void);
int masr_abi_version(void);
int masr_check_device(void);

/* ---- audio front-end -------------------------------------------------------------------------- */

/* Host-side staging of a batch: copy B separate float32 host arrays (what MASRPredictor.predict receives one at a
 * time, masr/predict.py:147-164; waves[b] has lengths[b] samples) back to back into the page-locked buffer `pinned`
 * and from there to `dev` (both sum(lengths) floats), packing on up to `nthreads` host threads and issuing each part's
 * cudaMemcpyAsync on `stream` as soon as it is packed.  Returns once the last copy has been issued. */
int masr_stage_waves_f32(const void* const* waves, const int64_t* lengths, int B, float* pinned, float* dev, int nthreads,
                         void* stream);

/* resampy.resample(x, src_rates[b], dst_rate, filter='kaiser_best') per utterance of a packed ragged batch
 * (masr/data_utils/audio.py:306-317, called by AudioFeaturizer.featurize, audio_featurizer.py:45-47), bit-identical to
 * the restatement in oracle/resample.py.  x: packed float32 input, x_offsets int64[B+1]; src_rates int32[B] (device);
 * table: float64[table_len], the right wing of the kaiser_best filter (512 entries per zero crossing);
 * y: packed float32 output, y_offsets int64[B+1] with y_len[b] = int(x_len[b] * dst_rate / src_rates[b]).
 * Rows with src_rates[b] == dst_rate are copied verbatim (y_len[b] == x_len[b]).  Host-side launch bounds:
 * max_out >= every y_len[b]; max_src_rate >= every src_rates[b] (it sizes the shared input window; rows above it
 * are left untouched).  Fails for max_src_rate > 512 * dst_rate. */
int masr_resample_f32(const float* x, const int64_t* x_offsets, const int* src_rates, int dst_rate, int B,
                      const double* table, int table_len, float* y, const int64_t* y_offsets, int64_t max_out,
                      int max_src_rate, void* stream);

/* Bytes of scratch masr_wave_gain_f32 needs for B utterances of at most max_samples samples. */
int masr_fbank_workspace_bytes(int B, int64_t max_samples, int64_t* bytes_host);

/* dB normalisation factor per utterance: AudioSegment.normalize / rms_db / gain_db
 * (masr/data_utils/audio.py:287-304,519-529,256-264).  wave: packed float32 samples in [-1,1);
 * offsets: int64[B+1] sample offsets.  gain[b] = 10^((target_db - 10*log10(mean(x^2)))/20);
 * status[b] = MASR_STATUS_GAIN_EXCEEDED where the reference raises ValueError (gain > max_gain_db). */
int masr_wave_gain_f32(const float* wave, const int64_t* offsets, int B, int64_t max_samples, float target_db,
                       float max_gain_db, float* gain, int* status, void* workspace, void* stream);

/* AudioSegment.to('int16') + torchaudio.compliance.kaldi.fbank(num_mel_bins=80, frame_length=25,
 * frame_shift=10, dither=0, sample_frequency=16000) (audio.py:244-254,549-574;
 * audio_featurizer.py:120-138; torchaudio kaldi.py:514-645).  gain may be NULL (no dB normalisation).
 * feats: [B, Fmax, 80] raw log-mel, rows >= the utterance's frame count are zero (an utterance with more than Fmax
 * frames gets its first Fmax); num_frames[b] = 1 + (n_b - 400) / 160 (0 if n_b < 400), written for every b whatever
 * Fmax (also 0), may be NULL.  With Fmax == 0 no sample is read and no feature written: wave and feats may be NULL. */
int masr_fbank_f32(const float* wave, const int64_t* offsets, const float* gain, int B, int Fmax, float* feats,
                   int* num_frames, void* stream);

/* ---- encoder building blocks ------------------------------------------------------------------ */

/* GlobalCMVN (masr/model_utils/utils/cmvn.py:29-31) + Conv2d(1,C,3,2) + ReLU
 * (masr/model_utils/conformer/subsampling.py:81-82).  feats [B,Fmax,idim] -> out [B,F1max,W1,C]
 * channels-last; w1 [C,1,3,3] as stored by the reference; mean/istd may both be NULL. */
int masr_conv1_cmvn_relu_f32(const float* feats, const float* mean, const float* istd, const float* w1,
                             const float* b1, float* out, int B, int Fmax, int idim, int F1max, int W1, int C,
                             void* stream);

/* Conv2d(C,C,3,2) + ReLU (subsampling.py:83-84) as an implicit GEMM over the channels-last conv-1
 * activation.  w2p [C, 3, 3, C] = reference weight [co,ci,kh,kw] permuted to [co,kh,kw,ci].
 * out [B, T2max, W2, C] (== the [B*T2max, W2*C] input of the `out` linear, subsampling.py:110).
 * C % 16 == 0; c1, w2p and out 16-byte aligned (128-bit loads and stores). */
int masr_conv2_s2_relu_f32(const float* c1, const float* w2p, const float* b2, float* out, int B, int F1max,
                           int W1, int T2max, int W2, int C, void* stream);

/* torch.nn.functional.linear / Conv1d(k=1) with a fused epilogue: C[M,N] = epi(A[M,K] . W[N,K]^T).
 * K % 16 == 0, lda % 4 == 0; A, W and C 16-byte aligned (C is written with 128-bit stores when ldc % 4 == 0);
 * bias may be NULL (no bias).  For MASR_EPI_BIAS_GLU the weight/bias rows are interleaved
 * (row 2j = value j, row 2j+1 = gate j) and C has N/2 columns. */
int masr_gemm_f32(const float* A, int64_t lda, const float* W, const float* bias, const float* residual,
                  int64_t ldr, float* C, int64_t ldc, int M, int N, int K, int epilogue, float alpha,
                  void* stream);

/* Tensor-core (wgmma/TMA) variant of masr_gemm_f32 with fp32-grade results: operands are fp16
 * (h, l) pairs, h = fp16(x), l = fp16((x - h) * 2^11) (masr_split_f16); C ~= Ah.Wh^T + 2^-11 (Ah.Wl^T + Al.Wh^T)
 * accumulated in fp32.  Output: fp32 C and/or the (Ch, Cl) pair the next GEMM consumes (either may be NULL,
 * not both).  Accuracy (the masr_split_f16 operand range): |C - A.W^T| <= c * (u (sqrt(K) |a_i o w_j| + |C|) +
 * 2^-36 sqrt(K) (|a_i| + |w_j|)), u = 2^-24, the second term being the pairs' absolute floor; c < 8 is asserted with operand
 * scales 2^-16 .. 2^12, and without the floor term where both scales are >= 2^-8 (DESIGN.md, precision policy).  An operand pair at +-inf (|x| >= 65520) makes its output row / column
 * NaN in every epilogue (ReLU keeps NaN) and leaves every other output unchanged.  K % 64 == 0, lda % 8 == 0, ldc % 8 == 0 (ldc % 4 when only fp32 is written); W is [N, K] dense. */
int masr_gemm_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* Wh, const void* Wl,
                       const float* bias, const float* residual, int64_t ldr, float* C, void* Ch, void* Cl,
                       int64_t ldc, int M, int N, int K, int epilogue, float alpha, void* stream);

/* Conformer feed-forward module in ONE tensor-core kernel (positionwise.py:37):
 *   x <- x + alpha * (SiLU(A.W1^T + b1) . W2^T + b2)
 * A: the LayerNorm-ed [M, D] (h, l) pair (row pitch lda), W1: [F, D] and W2: [D, F] dense pairs, x: the fp32 residual stream
 * (row pitch ldx), updated in place.  The [M, F] hidden activation stays in shared memory.  D == 256, F % 256 == 0,
 * lda % 8 == 0, ldx even.  Bit-identical to masr_gemm_tc_f16x2(MASR_EPI_BIAS_SILU -> pair) followed by
 * masr_gemm_tc_f16x2(MASR_EPI_RESIDUAL, alpha) with residual = C = x. */
int masr_ffn_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* W1h, const void* W1l, const float* b1,
                      const void* W2h, const void* W2l, const float* b2, float* x, int64_t ldx, int M, int D, int F,
                      float alpha, void* stream);

/* CTC head without the [M, V] logits: ctc_lo Linear (loss/ctc.py:70) with a GEMM epilogue that keeps, per frame and per
 * 32-column group, (max logit, first argmax, sum exp(x - max)), then a combine kernel -> per-frame argmax id (first
 * maximum, ctc_greedy_decoder.py:21) and max-probability 1 / sum_j exp(x_j - max) (the softmax value of the argmax).
 * A frame whose softmax is undefined (a NaN or +inf logit, e.g. from an operand pair at +-inf) gets maxp = NaN and id 0,
 * which is what np.argmax returns on the reference's all-NaN probability row.  Id 0 is the CTC blank, so such a frame
 * decodes as silence: a caller that must detect poisoned input checks maxp for NaN.
 * workspace: 3 * ceil(V/32) * M * 4 bytes.  Same outputs as masr_gemm_tc_f16x2 + masr_ctc_frame_argmax_f32. */
int masr_ctc_head_argmax_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* Wh, const void* Wl,
                                  const float* bias, int M, int V, int K, void* workspace, int64_t workspace_bytes,
                                  int* ids, float* maxp, void* stream);

/* Conv2dSubsampling4's first conv (as masr_conv1_cmvn_relu_f32) written as fp16 (h,l) pairs in four
 * (t,f)-parity planes [4][B][(F1max+1)/2][20][C], and its second conv + ReLU (subsampling.py:83-84) as a
 * tensor-core implicit GEMM over those planes: the stride-2 window of tap (kh,kw) is a dense TMA box of plane
 * (kh&1, kw&1).  Wh/Wl: split of the [C, 3,3,C]-permuted weight.  Output rows ((b*T2 + t)*19 + f) x C.
 * masr_conv2_tc_f16x2: C = 256 or 512 (C / 32 K-blocks per tap; the main product is summed in 256-K chunks, so a tap at
 * C = 512 is two chunks); masr_conv1_cmvn_relu_planes_f16: any C that is a multiple of 8. */
int masr_conv1_cmvn_relu_planes_f16(const float* feats, const float* mean, const float* istd, const float* w1,
                                    const float* b1, void* planes_h, void* planes_l, int B, int Fmax, int idim,
                                    int F1max, int W1, int C, void* stream);
int masr_conv2_tc_f16x2(const void* c1h, const void* c1l, const void* Wh, const void* Wl, const float* bias,
                        float* out, void* outh, void* outl, int B, int F1, int T2, int C, void* stream);

/* fp32 -> fp16 (h, l) pair, elementwise over n contiguous values: h = fp16_rn(x), l = fp16_rn((x - h) * 2^11), the form every
 * pair producer of this header writes.  Operand range (derived from the fp16 format):
 *   2^-14 <= |x| < 65520   h + 2^-11 l = x within 2^-22 |x|;
 *   |x| < 2^-14            l is an fp16 subnormal: an absolute floor of 2^-36 (|error| <= 2^-22 |x| + 2^-36 everywhere);
 *   |x| >= 65520           h = +-inf, l = -+inf (never a saturated finite value); a contraction that multiplies such a pair
 *                          by anything yields NaN (inf - inf), so every output the operand enters is non-finite. */
int masr_split_f16(const float* x, void* h, void* l, int64_t n, void* stream);

/* torch.nn.LayerNorm(D, eps) over the last dimension (encoder.py:64-72; convolution.py:66).  D = 256, 512, 1024, 2048 or 4096
 * (4096: the bidirectional DeepSpeech2 at rnn_size 2048, deepspeech2/encoder.py:34). */
int masr_layernorm_f32(const float* x, int64_t ldx, const float* gamma, const float* beta, float* y, int64_t ldy,
                       int M, int D, float eps, void* stream);

/* LayerNorm writing the fp16 (h, l) operand pair of masr_gemm_tc_f16x2 instead of fp32.  D = 256, 1024, 2048 or 4096 (a 512-wide
 * row goes through masr_layernorm_f32 + masr_split_f16, which write the same pair). */
int masr_layernorm_split_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, void* yh, void* yl,
                             int64_t ldy, int M, int D, float eps, void* stream);

/* Two LayerNorms back to back in one pass: y1 = LN(x; gamma1, beta1) as fp32 (row pitch ldx; may alias x), then
 * LN(y1; gamma2, beta2) as fp32 y2 (optional) and as the fp16 pair (row pitch ldy) — `norm_final` of one encoder block
 * followed by the next block's `norm_ff_macaron`, or by `after_norm` after the last block (conformer/encoder.py:161,106,342).
 * Bit-identical to masr_layernorm_f32 followed by masr_layernorm_split_f16.  D = 256 or 512. */
int masr_layernorm2_split_f16(const float* x, int64_t ldx, const float* gamma1, const float* beta1, float* y1,
                              const float* gamma2, const float* beta2, float* y2, void* yh, void* yl, int64_t ldy, int M,
                              int D, float eps, void* stream);

/* Squeezeformer helpers.
 *  masr_layernorm_ada_split_f16: y = LayerNorm(x) (optional fp32 copy) and the fp16 pair of ada_scale*y+ada_bias — the
 *    post-norm + adaptive scale of the next sub-module input (squeezeformer/encoder.py:412-463, positionwise.py:57-58);
 *  masr_affine_split_f16: pair of scale*x+bias (scale/bias optional), elementwise;
 *  masr_dwconv_bn_silu_f32: conv-module middle with BatchNorm1d(eval) folded to bn_scale/bn_shift (convolution.py:136-142);
 *  masr_time_reduce_dw_split_f16 / masr_upsample2_add_f32: time reduction depthwise conv (stride 2, kernel 1 or 5) and
 *    recovery `saved[t] + z[t/2]` (time_reduction.py:53-76,174-197; encoder.py:198-204). */
int masr_layernorm_ada_split_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, float* y,
                                 const float* ada_scale, const float* ada_bias, void* yh, void* yl, int64_t ldy, int M, int D,
                                 float eps, void* stream);
int masr_affine_split_f16(const float* x, const float* scale, const float* bias, void* yh, void* yl, int64_t M, int D,
                          void* stream);
int masr_dwconv_bn_silu_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w, const float* bias,
                            const float* bn_scale, const float* bn_shift, const float* pad_vec, float* y, void* yh, void* yl,
                            int64_t ldy, int64_t y_bstride, const int* in_lens, int B, int C, int kernel_size, int lpad,
                            int out_rows, void* stream);
int masr_time_reduce_dw_split_f16(const float* x, int64_t in_bstride, const float* w, const float* bias, void* yh, void* yl,
                                  int64_t out_bstride, const int* lens, int B, int out_rows, int k, int pad, int D,
                                  void* stream);
int masr_upsample2_add_f32(const float* saved, const float* z, float* out, int64_t full_bstride, int64_t half_bstride, int B,
                           int rows, int D, void* stream);

/* RelPositionMultiHeadedAttention core (masr/model_utils/conformer/attention.py:230-251,107-118):
 * Q rows (b*q_bstride + i), K/V rows (b*k_bstride + j), head h at column h*d_k; P [>=max klen, ldp] =
 * linear_pos(pos_emb) rows aligned with key index j; pos_u/pos_v [H,d_k]; O like Q.
 * q_lens/k_lens int32[B]: valid queries / keys per utterance (rows beyond q_lens are written as 0).
 * Output: fp32 O and/or the fp16 (Oh, Ol) operand pair of masr_gemm_tc_f16x2 (same ldo; either may be NULL). */
int masr_relpos_attention_f32(const float* Q, int64_t ldq, int64_t q_bstride, const float* K, const float* V,
                              int64_t ldk, int64_t k_bstride, const float* P, int64_t ldp, const float* pos_u,
                              const float* pos_v, float* O, void* Oh, void* Ol, int64_t ldo, int64_t o_bstride,
                              const int* q_lens, const int* k_lens, int B, int H, int d_k, int max_q, void* stream);

/* Same result as masr_relpos_attention_f32, computed on the tensor cores (mma.sync m16n8k16) with the FP16x2 operand
 * split (fp32-grade); used by the batched path.  Q is fp32 (the positional biases are added before the split); K, V
 * (row stride ldk halves, head h at column h*d_k) and P = linear_pos(pe) (ldp) arrive as fp16 (h,l) pairs — the qkv
 * GEMM epilogue and the weight loader produce them — so key tiles are 16-byte cp.async copies. */
int masr_relpos_attention_tc(const float* Q, int64_t ldq, int64_t q_bstride, const void* Kh, const void* Kl, const void* Vh,
                             const void* Vl, int64_t ldk, int64_t k_bstride, const void* Ph, const void* Pl, int64_t ldp,
                             const float* pos_u, const float* pos_v, float* O, void* Oh, void* Ol, int64_t ldo,
                             int64_t o_bstride, const int* q_lens, const int* k_lens, int B, int H, int d_k, int max_q,
                             void* stream);

/* masr_relpos_attention_tc on the Hopper tensor cores (wgmma, S and O accumulators in registers, K / linear_pos(pe) / V
 * tiles by TMA, V consumed as an MN-major operand, softmax between the two products inside the kernel): one CTA per
 * (utterance, head), for utterances of up to 256 frames — max_q <= 256 and every k_lens[b] <= 256 (the batched whole-utterance
 * path of 10 s audio: T = 248).  Same arguments plus `table_rows` (rows of the P table), same results (fp32-grade).
 * Supported K / V layout: the K and V matrices hold B * k_bstride rows and every k_lens[b] <= k_bstride — one [B*T, 3d] qkv
 * buffer with k_bstride = T, or a cache of B slots of k_bstride rows, where any slot (the last included) may hold more keys
 * than max_q.  The K / V tensor maps end at row B * k_bstride. */
int masr_relpos_attention_tc5(const float* Q, int64_t ldq, int64_t q_bstride, const void* Kh, const void* Kl, const void* Vh,
                              const void* Vl, int64_t ldk, int64_t k_bstride, const void* Ph, const void* Pl, int64_t ldp,
                              int64_t table_rows, const float* pos_u, const float* pos_v, float* O, void* Oh, void* Ol,
                              int64_t ldo, int64_t o_bstride, const int* q_lens, const int* k_lens, int B, int H, int d_k,
                              int max_q, void* stream);

/* ConvolutionModule middle (masr/model_utils/conformer/convolution.py:121-126): depthwise Conv1d(k)
 * -> LayerNorm(C) -> SiLU.  y[b,t,:] for t < out_rows from g[b, t - lpad + k, :], k < kernel_size;
 * g rows < 0 read pad_vec (NULL = 0), rows >= in_lens[b] read 0.  w [C,k] (reference [C,1,k]).
 * Output: fp32 y and/or the fp16 (yh, yl) pair (either may be NULL).  C = 256 or 512, kernel_size 7 / 15 / 31. */
int masr_dwconv_ln_silu_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w, const float* bias,
                            const float* ln_gamma, const float* ln_beta, const float* pad_vec, float* y, void* yh,
                            void* yl, int64_t ldy, int64_t y_bstride, const int* in_lens, int B, int C,
                            int kernel_size, int lpad, int out_rows, float eps, void* stream);

/* masr_dwconv_ln_silu_f32 with a time stride (1 or 2): y[t] reads g[t*stride - lpad + k] — the strided depthwise conv of
 * the EfficientConformer's block 3 (masr/model_utils/efficient_conformer/convolution.py:40-48, encoder.py:160-175).
 * Stride 2: C = 256 and kernel_size 15 only. */
int masr_dwconv_ln_silu_strided_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w, const float* bias,
                                    const float* ln_gamma, const float* ln_beta, const float* pad_vec, float* y, void* yh,
                                    void* yl, int64_t ldy, int64_t y_bstride, const int* in_lens, int B, int C,
                                    int kernel_size, int lpad, int stride, int out_rows, float eps, void* stream);

/* GroupedRelPositionMultiHeadedAttention core (masr/model_utils/efficient_conformer/attention.py:35-69,120-182): q/k/v
 * [B*bstride, ld] and p [>=max_t, H*d_k] row-major; `group` consecutive frames are viewed as H heads of width group*d_k;
 * frames >= lens[b] read as the reference's zero padding; pos_u/pos_v [H, group*d_k]; outputs for frames < lens[b]. */
int masr_grouped_attention_f32(const float* Q, const float* K, const float* V, const float* P, int64_t ld, int64_t bstride,
                               const float* pos_u, const float* pos_v, float* O, void* Oh, void* Ol, const int* lens,
                               int B, int H, int d_k, int group, int max_t, void* stream);

/* The same with a K|V cache (``forward`` with ``cache``, attention.py:151-158): q_lens[b] query frames at Q rows
 * b*q_bstride.. (pitch ldq), k_lens[b] key/value frames = [cache ++ chunk] at K/V rows b*k_bstride.. (pitch ldk); P row j
 * belongs to key j; queries are grouped from the first chunk frame, keys from key 0.  Outputs in Q's layout. */
int masr_grouped_attention_cache_f32(const float* Q, int64_t ldq, int64_t q_bstride, const float* K, const float* V,
                                     int64_t ldk, int64_t k_bstride, const float* P, const float* pos_u, const float* pos_v,
                                     float* O, void* Oh, void* Ol, const int* q_lens, const int* k_lens, int B, int H,
                                     int d_k, int group, int max_q, void* stream);

/* AvgPool1d(2, 2, ceil_mode=True, count_include_pad=False) over time per utterance (efficient_conformer/encoder.py:
 * 173-175): y[b,t] = mean(x[b,2t], x[b,2t+1]) (single element at an odd tail), rows >= ceil(len/2) are 0. */
int masr_avgpool2_time_f32(const float* x, int64_t in_bstride, float* y, int64_t out_bstride, const int* lens, int B,
                           int out_rows, int D, void* stream);

/* One time step of torch.nn.LSTM as DeepSpeech2 uses it (masr/model_utils/deepspeech2/encoder.py:36-45, packed ragged
 * batches): gates_x [B*bstride, 4H] = W_ih x + b_ih + b_hh (gate order i,f,g,o); Whh [4H, H]; states transposed and
 * batch-chunked h_*_T [ceil(B/32)][H][32] (ping-pong: in != out), c_state [B][H]; utterance b is active while
 * step < lens[b] and uses time index step (forward) or lens[b]-1-step (reverse); h_t is written to
 * out[(b*bstride + t), col_off + u] as fp32 and/or fp16 pair. */
int masr_lstm_step_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h_in_T,
                       float* h_out_T, float* c_state, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                       const int* lens, int B, int H, int step, int reverse, void* stream);

/* All T steps of one LSTM layer / direction in ONE persistent launch: every CTA keeps its slice of W_hh (the four gate rows
 * of 8 hidden units) resident in shared memory, h_{t-1} is streamed through a shared-memory window and the steps are
 * separated by a grid-wide barrier.  Same results as T calls of masr_lstm_step_f32 up to the order of the K summation.
 * h0_T / hN_T: initial / final hidden state, transposed [ceil(B/32)][H][32]; c_state [B][H] updated in place; workspace
 * from masr_lstm_seq_workspace_bytes.  H % 128 == 0, H <= 1024 (the shipped configs: 1024). */
int masr_lstm_seq_workspace_bytes(int B, int H, int64_t* bytes);
int masr_lstm_seq_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h0_T, float* hN_T,
                      float* c_state, float* out, void* outh, void* outl, int64_t ld_out, int col_off, const int* lens, int B,
                      int H, int T, int reverse, void* workspace, int64_t workspace_bytes, void* stream);

/* The GRU forms of the two entry points above, for DeepSpeech2 with use_gru: True (masr/model_utils/deepspeech2/encoder.py:
 * 24-33 -> gru.py:6-22, torch.nn.GRU, gate order r, z, n).  Same arguments as their LSTM counterparts except that there is
 * no c_state (a GRU carries h only) and b_hn [H] takes its place: gates_x [., 3H] = W_ih x + b_ih + [b_hr, b_hz, 0];
 * Whh [3H, H];
 *     r = sigmoid(gx_r + W_hr h) ; z = sigmoid(gx_z + W_hz h) ; n = tanh(gx_n + r * (W_hn h + b_hn)) ; h' = n + z (h - n)
 * (b_hn stays inside the product with r, so it cannot be folded into gates_x).  The persistent form keeps the three gate rows
 * of 8 hidden units resident (96 KB at H = 1024) and uses the same workspace layout as masr_lstm_seq_f32, so
 * masr_lstm_seq_workspace_bytes sizes it too.  masr_gru_step_f32: H % 4 == 0, in != out; masr_gru_seq_f32: H % 128 == 0,
 * H <= 1024, H / 8 CTAs co-resident (h0_T == hN_T allowed). */
int masr_gru_step_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h_in_T,
                      float* h_out_T, const float* bhn, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                      const int* lens, int B, int H, int step, int reverse, void* stream);
int masr_gru_seq_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h0_T, float* hN_T,
                     const float* bhn, float* out, void* outh, void* outl, int64_t ld_out, int col_off, const int* lens, int B,
                     int H, int T, int reverse, void* workspace, int64_t workspace_bytes, void* stream);

/* The persistent recurrences of masr_lstm_seq_f32 / masr_gru_seq_f32 at H = 2048 (encoder_conf.rnn_size: 2048, the large-
 * data size of configs/deepspeech2.yml; encoder.py:36-45, gru.py:6-22), on the tensor cores: W_hh . h_{t-1} by mma.sync
 * m16n8k16 in the FP16x2 split of masr_gemm_tc_f16x2 (fp32 accumulators), the cell in fp32.  One CTA per 16 hidden units
 * (H / 16 = 128 CTAs, all co-resident, a grid barrier per step); part of each CTA's weight slice stays in shared memory, the
 * rest is streamed from L2 on every step.  Same arguments and semantics as the fp32 forms (ragged lengths, both directions,
 * h0_T == hN_T allowed, c_state in place, fp32 and/or pair output at col_off) except:
 *   Whh_packed: W_hh [G*H, H] packed once by masr_rnn_tc_pack_f16x2 (G = 4 for the LSTM, 3 for the GRU; G*H*H*4 bytes);
 *   workspace:  masr_rnn_seq_tc_workspace_bytes(B, H).
 * H = 2048 only.  Fails with MASR_ERR_INVALID_ARGUMENT, launching nothing, when the grid cannot be resident at once. */
int masr_rnn_seq_tc_workspace_bytes(int B, int H, int64_t* bytes);
int masr_rnn_tc_pack_f16x2(const float* Whh, void* packed, int G, int H, void* stream);
int masr_lstm_seq_tc_f16x2(const float* gates_x, int64_t ldg, int64_t bstride, const void* Whh_packed, const float* h0_T,
                           float* hN_T, float* c_state, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                           const int* lens, int B, int H, int T, int reverse, void* workspace, int64_t workspace_bytes,
                           void* stream);
int masr_gru_seq_tc_f16x2(const float* gates_x, int64_t ldg, int64_t bstride, const void* Whh_packed, const float* h0_T,
                          float* hN_T, const float* bhn, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                          const int* lens, int B, int H, int T, int reverse, void* workspace, int64_t workspace_bytes,
                          void* stream);

/* ---- batched chunk (streaming) state ------------------------------------------------------------ */

/* Append the chunk's new rows to every slot's cache (the `torch.cat` on time of the attention K|V cache, conformer/
 * attention.py:218-225), on the device: for slot s and t < cnt[s]
 *   dst{0,1}[(s*cap + base[s] + t) * dst_pitch + c] = src{0,1}[(s*rows_per_slot + t) * src_pitch + col0 + c],  c < row_bytes
 * (all sizes in BYTES, multiples of 16; src1/dst1 may both be NULL; the pair form moves the fp16 (h,l) operand halves). */
int masr_stream_append_rows(const void* src0, const void* src1, int64_t src_pitch_bytes, int64_t col0_bytes, int row_bytes,
                            void* dst0, void* dst1, int64_t dst_pitch_bytes, int64_t cap, const int* base, const int* cnt,
                            int rows_per_slot, int S, void* stream);

/* Slide every slot's conv-module left context (convolution.py:105-109, `new_cache = x[:, :, -lorder:]`): for slot s with
 * n = cnt[s] > 0, rows [0, lorder) <- rows [n, n + lorder) of its [rows_per_slot, row_bytes] block of x0 (and x1). */
int masr_stream_shift_cache(void* x0, void* x1, int64_t rows_per_slot, int lorder, int row_bytes, const int* cnt, int S,
                            void* stream);

/* ---- CTC head / greedy decode ------------------------------------------------------------------- */

/* softmax statistics of CTCLoss.softmax (masr/model_utils/loss/ctc.py:70) fused with the argmax of
 * greedy_decoder (masr/decoders/ctc_greedy_decoder.py:21-22): ids[m] = first argmax_v, maxp[m] =
 * softmax(logits[m])[ids[m]] (a frame with a NaN or +inf logit: maxp = NaN, id 0, as masr_ctc_head_argmax_tc_f16x2).
 * probs (optional, may be NULL): full posterior [M, ldp]. */
int masr_ctc_frame_argmax_f32(const float* logits, int64_t ldl, int M, int V, int* ids, float* maxp, float* probs,
                              int64_t ldp, void* stream);

/* greedy_decoder's collapse (ctc_greedy_decoder.py:23-30): per utterance b over frames t < lens[b]
 * (rows b*bstride + t): tokens = ids with consecutive repeats merged and `blank` dropped;
 * psum/pcount = float32 left-to-right sum / count of maxp over non-blank frames (score = 100*psum/pcount). */
int masr_ctc_greedy_collapse(const int* ids, const float* maxp, int64_t bstride, const int* lens, int B, int blank,
                             int* tokens, int64_t tok_stride, int* ntok, float* psum, int* pcount, void* stream);

/* ---- CTC prefix beam search (no LM) --------------------------------------------------------------------
 * Replaces the external paddlespeech_ctcdecoders call behind masr/decoders/swig_wrapper.py:35-64
 * (`ctc_beam_search_decoding(probs, vocab, beam_size, cutoff_prob, cutoff_top_n, scorer, blank_id)`), scorer = None.
 * PARITY UNPINNED (library absent): semantics per SURVEY.md Appendix D, checked against oracle/beam.py.
 *  masr_ctc_topk_f32:     per frame the <= top_n (<= 40) most probable tokens, cut where the cumulative probability
 *                         reaches cutoff_prob: cand_id / cand_logp [M, 40] (best first), cand_cnt [M];
 *  masr_ctc_prefix_beam:  per utterance (rows b*bstride + t, t < lens[b]) the best prefix: out_tok [B, tok_stride],
 *                         out_n [B], out_score [B] = log P(prefix); beam_size <= 512.  Scratch sizes from
 *                         masr_ctc_prefix_beam_workspace (pool floats total, trie ints per utterance for each of
 *                         trie_parent / trie_tok). */
int masr_ctc_topk_f32(const float* logits, int64_t ldl, int M, int V, int top_n, float cutoff_prob, int* cand_id,
                      float* cand_logp, int* cand_cnt, void* stream);
int masr_ctc_prefix_beam_workspace(int B, int Tmax, int64_t* pool_floats_host, int64_t* trie_ints_per_utt_host);
int masr_ctc_prefix_beam(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride, const int* lens,
                         int B, int beam_size, int blank, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                         int* out_tok, int64_t tok_stride, int* out_n, float* out_score, void* stream);

/* Streaming form of masr_ctc_prefix_beam (beam_search_decoder.py:75-96: CTCBeamSearchDecoder.next() + decode(),
 * reset_state()): the same search fed chunk by chunk.  lens[b] = frames of THIS chunk; resume = 0 starts a new utterance
 * (reset_decoder), != 0 continues from state_i / state_f (sizes per utterance from masr_ctc_prefix_beam_state_size);
 * trie_parent / trie_tok are sized for the whole stream (masr_ctc_prefix_beam_workspace with Tmax = its frame count) and
 * persist between calls.  Outputs: the best prefix and its score after all frames seen so far — identical to one
 * masr_ctc_prefix_beam call over the concatenated chunks. */
int masr_ctc_prefix_beam_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume, int* out_tok,
                                int64_t tok_stride, int* out_n, float* out_score, void* stream);

/* ---- character n-gram LM fusion (ARPA) ------------------------------------------------------------------
 * Replaces the external `Scorer(alpha, beta, model_path, vocabulary)` (masr/decoders/swig_wrapper.py:4-18) that
 * BeamSearchDecoder builds and queries (beam_search_decoder.py:29-32: is_character_based / get_max_order /
 * get_dict_size; :47 reset_params(alpha, beta) before every decode) for a CHARACTER-based plain-text ARPA LM.
 * PARITY UNPINNED (library absent): semantics per oracle/lm.py (DESIGN.md §2).
 *
 * The loader is the one part of the library that owns memory: a host handle from masr_lm_load_arpa, released with
 * masr_lm_free.  Its tables are copied out with masr_lm_export into caller buffers (host), which the caller uploads to
 * device buffers and points a masr_lm_tables at; the device entry points below take that struct (a host pointer to it). */
typedef struct masr_lm_tables {
    const uint32_t* keys;     /* device: 4 words per slot (n word ids, 16 bits each, in words 0..2)            */
    const float* vals;        /* device: 2 floats per slot: ln p, ln backoff                                    */
    const int* tok2lm;        /* device [V]: model token id -> LM word id, -1 = not an LM word (or <unk>)       */
    int order;                /* N, 1..6                                                                        */
    int bos, eos;             /* LM word ids of <s>, </s>                                                       */
    int vocab;                /* V                                                                              */
    int64_t off[8];           /* off[n]: first slot of the order-n table (n = 1..order)                         */
    int64_t mask[8];          /* mask[n]: slots of the order-n table - 1 (a power of two - 1)                   */
} masr_lm_tables;

/* info_host[32] layout written by masr_lm_info */
enum {
    MASR_LM_INFO_ORDER = 0, MASR_LM_INFO_CHAR_BASED = 1, MASR_LM_INFO_DICT_SIZE = 2, MASR_LM_INFO_VOCAB = 3,
    MASR_LM_INFO_KEY_WORDS = 4, MASR_LM_INFO_VAL_FLOATS = 5, MASR_LM_INFO_BOS = 6, MASR_LM_INFO_EOS = 7,
    MASR_LM_INFO_READ = 8,    /* + n - 1: n-grams of order n in the file          */
    MASR_LM_INFO_KEPT = 14,   /* + n - 1: n-grams of order n kept in the tables   */
    MASR_LM_INFO_SLOTS = 20,  /* + n - 1: slots of the order-n table              */
    MASR_LM_INFO_TABLE_BYTES = 26,
};

/* Parse a plain-text ARPA file (path_host, UTF-8) against the model vocabulary vocab_host (V UTF-8 tokens joined by
 * '\n'): n-grams containing a word that is neither a model token nor <s> / </s> are dropped (no query reaches them),
 * `<unk>` counts as out of vocabulary.  Rejects a KenLM binary, a missing \data\ section, count or section mismatches,
 * a missing <s> or </s>, an order above 6 and malformed lines.  *handle_host receives the handle. */
int masr_lm_load_arpa(const char* path_host, const char* vocab_host, int V, void** handle_host);
int masr_lm_info(const void* handle_host, int64_t* info_host);
/* copy the packed tables (sizes from masr_lm_info) into keys_host / vals_host / tok2lm_host and fill layout_host
 * (everything but the three pointers, which the caller sets to its device copies) */
int masr_lm_export(const void* handle_host, uint32_t* keys_host, float* vals_host, int* tok2lm_host,
                   masr_lm_tables* layout_host);
int masr_lm_free(void* handle_host);

/* Q queries of lnP(word | window): ctx [Q, order-1] and word [Q] are model token ids, or -1 = <s>, -2 = </s>
 * (the window oldest first); out [Q].  The lookup the beam search uses, exposed for testing the tables. */
int masr_lm_score_f32(const masr_lm_tables* lm_host, const int* ctx, const int* word, int Q, float* out, void* stream);

/* masr_ctc_topk_f32 that also writes blank_logp[m] = ln softmax(logits[m])[blank] (whether or not blank is a
 * candidate): the `std::log(prob[blank_id])` term of the LM search's min_cutoff. */
int masr_ctc_topk_blank_f32(const float* logits, int64_t ldl, int M, int V, int top_n, float cutoff_prob, int blank,
                            int* cand_id, float* cand_logp, int* cand_cnt, float* blank_logp, void* stream);

/* masr_ctc_prefix_beam with shallow fusion of the LM (alpha, beta as in the config's ctc_beam_search_decoder_conf):
 * every extension l -> l+c adds alpha * lnP(c | l) + beta, pairs below min_cutoff are skipped, the beam is ranked by the
 * fused score (out_score) and out_approx = fused score - len * beta - alpha * lnP(<s>.. tokens </s>) (the reference's
 * approx_ctc).  Same workspace as masr_ctc_prefix_beam. */
int masr_ctc_prefix_beam_lm(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                            int64_t bstride, const int* lens, int B, int beam_size, int blank, const masr_lm_tables* lm_host,
                            float alpha, float beta, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                            int* out_tok, int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream);
/* streaming form: as masr_ctc_prefix_beam_stream; the state also carries each beam entry's LM window, so its size
 * comes from masr_ctc_prefix_beam_lm_state_size */
int masr_ctc_prefix_beam_lm_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_lm_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                   int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                   const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                   int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume, int* out_tok,
                                   int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream);

/* Pool forms of the two streaming searches, for the slots of a stream pool that start and end utterances independently:
 * as masr_ctc_prefix_beam_stream / masr_ctc_prefix_beam_lm_stream with a device flag per slot, fresh[B], in place of
 * `resume`.  fresh[b] != 0 starts slot b at the root (the kernel clears the flag once the slot is initialised), else the
 * slot resumes from its state.  The kernel never clears a slot's hash: whoever marks slot b fresh also sets
 * trie_parent[b*trie_cap + trie_cap/5, (b+1)*trie_cap) to -1 (the hash is also -1 before the first launch).  A slot with
 * lens[b] == 0 is not touched at all (state, trie and outputs unchanged).  trie_cap per slot = 5 * (frames * beam_size + 1)
 * suffices for `frames` frames of that slot (at most beam_size new prefixes per frame). */
int masr_ctc_prefix_beam_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                              const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                              int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                              int64_t tok_stride, int* out_n, float* out_score, void* stream);
int masr_ctc_prefix_beam_lm_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                 int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                 const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                 int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                                 int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream);

/* Token onsets of the prefix beam search (every form above and the word-LM forms below).
 * Trie layout per slot (trie_cap ints each of trie_parent and trie_tok, nc = trie_cap / 5):
 *   trie_parent [0, nc)       parent node of node id (root 0: -1)
 *   trie_parent [nc, 5 nc)    the persistent (parent, token) -> node hash (-1 = empty)
 *   trie_tok    [0, nc)       last token of node id (root: -1)
 *   trie_tok    [nc, 2 nc)    word-LM forms: 1 = the node's lexicon state was reset after <space>
 *   trie_tok    [2 nc, 3 nc)  the onset of node id: the frame at which the search allocated it, i.e. the first frame after
 *                             whose selection its prefix was in the beam (nodes are allocated for survivors only, and a
 *                             prefix that leaves the beam and comes back keeps its node, so onsets strictly increase
 *                             along a prefix)
 *   trie_tok    [4 nc]        frames searched since the slot started fresh (one-shot, resume = 0, or fresh[b]); frames
 *                             count from there, so a stream fed in any chunking records the one-shot search's onsets.
 * masr_ctc_prefix_beam_frames: after a search, for each slot b < B the onset frame of every token of the prefix it
 * reported: out_frame[b * tok_stride_f + p] for p < out_n[b], found by walking the hash from the root along
 * out_tok[b * tok_stride + p] (so it serves the word-LM forms, which may report an entry other than rank 0); -1 where
 * the prefix has no node (the trie ran out of nodes, or the slot was reset since).  One CTA per slot; the search's own
 * trie_parent / trie_tok / trie_cap / out_tok / out_n. */
int masr_ctc_prefix_beam_frames(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* out_tok,
                                int64_t tok_stride, const int* out_n, int B, int* out_frame, int64_t tok_stride_f, void* stream);

/* ---- word n-gram LM fusion (ARPA) with the lexicon constraint -------------------------------------------
 * The external Scorer for a WORD-based LM (English models: configs/english_example.yml): the LM scores a word once, when
 * the <space> after it is emitted, and every hypothesis is limited to words of a lexicon built from the LM's unigrams
 * (the library's OpenFST dictionary).  PARITY UNPINNED (library absent): semantics per oracle/word_lm.py (DESIGN.md §2).
 *
 * Word ids are 24 bits (lexicon words 0 .. dict_size-1 in unigram file order, <s> = dict_size, </s> = dict_size + 1),
 * packed 24 bits each into the 4-word key, so orders 1..5 and at most 2^24 - 1 declared unigrams are accepted.
 * The lexicon: every unigram except <s>, </s>, <unk> whose code points are each a model token, as a trie over token ids
 * (node 0 = root, nodes in insertion order); its arcs in CSR form, ascending token within a node. */
typedef struct masr_word_lm_tables {
    const uint32_t* keys;     /* device: 4 words per slot (n word ids, 24 bits each from bit 0)                 */
    const float* vals;        /* device: 2 floats per slot: ln p, ln backoff                                    */
    const int* lex_off;       /* device [nodes + 1]: first arc of each lexicon node                             */
    const int* lex_tok;       /* device [arcs]: token of each arc                                               */
    const int* lex_next;      /* device [arcs]: node each arc leads to                                          */
    const int* lex_word;      /* device [nodes]: word id ending at the node, -1 if none                         */
    int order;                /* N, 1..5                                                                        */
    int bos, eos;             /* word ids of <s>, </s>                                                          */
    int vocab;                /* V                                                                              */
    int space;                /* token id of <space>                                                            */
    int root;                 /* lexicon root node (0)                                                          */
    int nodes;                /* lexicon nodes                                                                  */
    int dict_size;            /* lexicon words                                                                  */
    int64_t off[8];           /* off[n]: first slot of the order-n table (n = 1..order)                         */
    int64_t mask[8];          /* mask[n]: slots of the order-n table - 1 (a power of two - 1)                   */
} masr_word_lm_tables;

/* info_host[32] written by masr_word_lm_info: the masr_lm_info layout (KEY_WORDS, READ, KEPT, ... of the word tables;
 * CHAR_BASED = 0, DICT_SIZE = lexicon words) plus these */
enum { MASR_WORD_LM_INFO_NODES = 27, MASR_WORD_LM_INFO_ARCS = 28, MASR_WORD_LM_INFO_SPACE = 29 };

/* Parse a word-based plain-text ARPA file against the vocabulary (as masr_lm_load_arpa).  Rejects, besides every case
 * masr_lm_load_arpa rejects: a character-based file, a vocabulary without "<space>", an order above 5 and more than
 * 2^24 - 1 declared unigrams.  n-grams with a word outside the lexicon (other than <s>, </s>) are dropped. */
int masr_word_lm_load_arpa(const char* path_host, const char* vocab_host, int V, void** handle_host);
int masr_word_lm_info(const void* handle_host, int64_t* info_host);
/* copy the tables and the lexicon (sizes from masr_word_lm_info) into host buffers and fill layout_host (all but the
 * six pointers); the handle is released with masr_lm_free */
int masr_word_lm_export(const void* handle_host, uint32_t* keys_host, float* vals_host, int* lex_off_host, int* lex_tok_host,
                        int* lex_next_host, int* lex_word_host, masr_word_lm_tables* layout_host);
/* Q queries of lnP(word | window) over word ids: ctx [Q, order-1] (oldest first) and word [Q]; -1 = out of vocabulary */
int masr_word_lm_score_f32(const masr_word_lm_tables* lm_host, const int* ctx, const int* word, int Q, float* out, void* stream);

/* masr_ctc_prefix_beam_lm with a word LM: an extension by <space> adds alpha * lnP(word just completed | the N-1 words
 * before it) + beta, any other extension adds nothing; extensions the lexicon rejects contribute nothing (after <space>,
 * a prefix's first attempt in candidate order is rejected and resets it to the lexicon root, once).  After the last frame
 * every non-empty prefix not ending in <space> gets alpha * lnP(its last word | h) + beta (-1000 for lnP of a partial
 * word) on the side; the best of those adjusted scores is reported (out_score) with its approx_ctc (out_approx).
 * The word-LM forms also keep one flag per trie node in trie_tok[trie_cap/5, 2*trie_cap/5) of each utterance.
 * Same workspace as masr_ctc_prefix_beam; the streaming and pool forms size their state with
 * masr_ctc_prefix_beam_wordlm_state_size and are otherwise as masr_ctc_prefix_beam_lm_stream / _lm_pool. */
int masr_ctc_prefix_beam_wordlm(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                float* out_approx, void* stream);
int masr_ctc_prefix_beam_wordlm_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_wordlm_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                       int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                       const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool,
                                       int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                       int resume, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                       float* out_approx, void* stream);
int masr_ctc_prefix_beam_wordlm_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                     int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                     const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                     int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                                     int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream);

/* ---- hotword biasing ------------------------------------------------------------------------------------------------
 * Boosts user hotwords inside the prefix beam search (semantics: oracle/hotwords.py, masr_b200/hotwords.py).  The
 * hotwords' token sequences form an Aho-Corasick automaton; one buffer may hold several graphs (one per stream-pool
 * slot), each a contiguous node range whose first node is its root.  Node ids, arc targets, fail and tail are indices of
 * the whole buffer.  Per node n: acc = float32(w) * depth, leaf = no hotword extends str(n), fail = the longest proper
 * suffix of str(n) that is a node, tail = -1 if no prefix of str(n) (itself included) is a whole hotword, else the state
 * reached from the root by what follows the deepest such prefix ta(n), whose credit is ta_acc; fin = the credit banked
 * when a token that extends nothing follows n.  Arcs in CSR form, ascending token within a node. */
typedef struct masr_hotword_graph {
    const int* arc_off;       /* device [nodes + 1]: first arc of each node                                     */
    const int* arc_tok;       /* device [arcs]: token of each arc                                               */
    const int* arc_next;      /* device [arcs]: node each arc leads to                                          */
    const int* fail;          /* device [nodes]                                                                 */
    const int* tail;          /* device [nodes]: -1 = no whole hotword in the match                             */
    const int* leaf;          /* device [nodes]: 1 = no hotword extends the match                               */
    const float* acc;         /* device [nodes]                                                                 */
    const float* ta_acc;      /* device [nodes]: acc of the deepest whole hotword in the match                  */
    const float* fin;         /* device [nodes]                                                                 */
    int nodes;                /* nodes of the buffer                                                            */
} masr_hotword_graph;

/* The nine prefix beam searches above with hotword biasing: the same arguments, then hot_host (the graph) and slot_root
 * [B] (device: slot b's root node, -1 = no hotwords for that slot, which searches exactly as without).  Every extension
 * by a non-blank token with a finite base adds the automaton's credit delta after the LM terms; the reported entry is the
 * best after adding each entry's read-out fin(s) - acc(s), and out_score (and out_approx) exclude every credit: they
 * are the reported entry's selection score minus the float32 sum of its tokens' deltas and read-out.  The streaming and
 * pool forms size their state with the *_hot_state_size answers (BEAM_CAP ints more than without). */
int masr_ctc_prefix_beam_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_lm_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_wordlm_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt);
int masr_ctc_prefix_beam_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride, const int* lens,
                             int B, int beam_size, int blank, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                             int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                             const masr_hotword_graph* hot_host, const int* slot_root, void* stream);
int masr_ctc_prefix_beam_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                    const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                    int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume, int* out_tok,
                                    int64_t tok_stride, int* out_n, float* out_score, const masr_hotword_graph* hot_host,
                                    const int* slot_root, void* stream);
int masr_ctc_prefix_beam_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                  const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                  int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                                  int64_t tok_stride, int* out_n, float* out_score, const masr_hotword_graph* hot_host,
                                  const int* slot_root, void* stream);
int masr_ctc_prefix_beam_lm_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                int64_t bstride, const int* lens, int B, int beam_size, int blank, const masr_lm_tables* lm_host,
                                float alpha, float beta, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                                int* out_tok, int64_t tok_stride, int* out_n, float* out_score, float* out_approx,
                                const masr_hotword_graph* hot_host, const int* slot_root, void* stream);
int masr_ctc_prefix_beam_lm_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                       int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                       const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                       int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume, int* out_tok,
                                       int64_t tok_stride, int* out_n, float* out_score, float* out_approx,
                                       const masr_hotword_graph* hot_host, const int* slot_root, void* stream);
int masr_ctc_prefix_beam_lm_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                     int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                     const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                     int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                                     int64_t tok_stride, int* out_n, float* out_score, float* out_approx,
                                     const masr_hotword_graph* hot_host, const int* slot_root, void* stream);
int masr_ctc_prefix_beam_wordlm_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                    int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                    const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                    int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride, int* out_n,
                                    float* out_score, float* out_approx, const masr_hotword_graph* hot_host,
                                    const int* slot_root, void* stream);
int masr_ctc_prefix_beam_wordlm_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                           const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                           int blank, const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool,
                                           int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                           int resume, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                           float* out_approx, const masr_hotword_graph* hot_host, const int* slot_root,
                                           void* stream);
int masr_ctc_prefix_beam_wordlm_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                         const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                         int blank, const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool,
                                         int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                         int* fresh, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                         float* out_approx, const masr_hotword_graph* hot_host, const int* slot_root,
                                         void* stream);

/* ---- N-best read-out ------------------------------------------------------------------------------------------------
 * The reference decoder returns "a list of (log probability, sentence) tuples, sorted by probability, descending"
 * (masr/decoders/swig_wrapper.py:58,61-64; MASR's wrapper keeps the first, beam_search_decoder.py:56,72,89-91).  These
 * read the n best hypotheses of slots 0..B-1 out of the beam a streaming or pool search of the matching kind left in
 * state_i / state_f (the same trie_parent / trie_tok / trie_cap, and with an LM the same tables, alpha and beta; with
 * hotwords the same graph and slot_root).  The search's state is only read, so the read-out may follow any launch.
 * Order: the search's own selection score after the read-out terms (the word LM's alpha lnP(last word | h) + beta, the
 * hotwords' fin(s) - acc(s)), descending, ties to the lower beam rank, so hypothesis 0 is the prefix the search reported.
 * Per slot b and hypothesis h < out_count[b] = min(n, live beam entries): tokens out_tok[(b*n + h) * tok_stride + p] for
 * p < out_len[b*n + h], out_score[b*n + h] as the search's out_score (log P without an LM, the fused score with one;
 * hotword credit taken out) and with an LM out_approx[b*n + h] as its out_approx (approx_ctc).  With an LM the list is
 * ordered by the fused score, so the approx_ctc values need not decrease down it.  fresh (may be NULL): the pool form's
 * flags; a slot whose flag is set has no beam yet and reports out_count[b] = 0, nothing else.  n in 1..512; a refused
 * call writes nothing.  One CTA per slot. */
int masr_ctc_prefix_beam_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                               const float* state_f, const int* fresh, int B, int n, int* out_tok, int64_t tok_stride,
                               int* out_len, float* out_score, int* out_count, void* stream);
int masr_ctc_prefix_beam_lm_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                  const float* state_f, const int* fresh, int B, int n, const masr_lm_tables* lm_host,
                                  float alpha, float beta, int* out_tok, int64_t tok_stride, int* out_len, float* out_score,
                                  float* out_approx, int* out_count, void* stream);
int masr_ctc_prefix_beam_wordlm_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                      const float* state_f, const int* fresh, int B, int n, const masr_word_lm_tables* lm_host,
                                      float alpha, float beta, int* out_tok, int64_t tok_stride, int* out_len,
                                      float* out_score, float* out_approx, int* out_count, void* stream);
int masr_ctc_prefix_beam_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                   const float* state_f, const int* fresh, int B, int n, int* out_tok, int64_t tok_stride,
                                   int* out_len, float* out_score, int* out_count, const masr_hotword_graph* hot_host,
                                   const int* slot_root, void* stream);
int masr_ctc_prefix_beam_lm_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                      const float* state_f, const int* fresh, int B, int n, const masr_lm_tables* lm_host,
                                      float alpha, float beta, int* out_tok, int64_t tok_stride, int* out_len,
                                      float* out_score, float* out_approx, int* out_count, const masr_hotword_graph* hot_host,
                                      const int* slot_root, void* stream);
int masr_ctc_prefix_beam_wordlm_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                          const float* state_f, const int* fresh, int B, int n,
                                          const masr_word_lm_tables* lm_host, float alpha, float beta, int* out_tok,
                                          int64_t tok_stride, int* out_len, float* out_score, float* out_approx,
                                          int* out_count, const masr_hotword_graph* hot_host, const int* slot_root,
                                          void* stream);

/* The silero VAD network (16 kHz branch of silero_vad.onnx, weights packed by masr_b200/silero.py) over one recording
 * of n_samples 16 kHz samples in windows of `window` samples (512, 1024 or 1536; the last window zero-padded),
 * T = window / 512 recurrent steps per window, N = ceil(n_samples / window) windows.
 * masr_silero_vad_layout: floats[0..3] = float32 counts of the STFT basis, the packed encoder and recurrence buffers,
 * and the gate-input row (256) per step.
 * masr_silero_vad_encode_f32: every window in parallel, reflect pad -> STFT -> magnitude / log -> adaptive
 * normalisation -> first_layer -> encoder -> gates_x[N*T][256] = W_ih1 x + (Wb1 + Rb1) (gate rows i, f, g, o).
 * masr_silero_vad_recur_f32: one CTA runs both LSTM layers (state zero at the start) over all N*T steps, then the
 * decoder: logits[N*T] (workspace), probs[N] = mean over each window's steps of sigmoid(logit).
 * masr_silero_vad_recur_slots_f32: one CTA per slot; slot s runs windows [win_off[s], win_off[s+1]) of gates_x
 * (win_off: device int32 [n_slots + 1], non-decreasing from 0) from its carried state[s] = (h1, c1, h2, c2), each [64],
 * writes probs[w] for each of those windows (logits as above, same rows) and the final state back to state[s].  A
 * slot without windows is not touched; with every state zero and one slot it computes masr_silero_vad_recur_f32. */
int masr_silero_vad_layout(int64_t* floats);
int masr_silero_vad_encode_f32(const float* audio, int64_t n_samples, int window, const float* basis, const float* enc,
                               float* gates_x, void* stream);
int masr_silero_vad_recur_f32(const float* gates_x, int64_t n_windows, int window, const float* rec, float* logits,
                              float* probs, void* stream);
int masr_silero_vad_recur_slots_f32(const float* gates_x, const int32_t* win_off, int n_slots, int window, const float* rec,
                                    float* state, float* logits, float* probs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MASR_B200_H_ */
