/* b200vc — C ABI of the GPU-native (H100, sm_90a) RVC / MDX hot path.
 *
 * The reference (SociallyIneptWeeb/AICoverGen) is pure Python; its "operator
 * boundary" for this path is the set of library calls it makes into
 * torch/cuDNN/cuBLAS/cuFFT/onnxruntime/faiss.  Every entry point below names
 * the reference call site(s) it replaces (paths relative to the reference
 * repo).  A maintainer binds them with ctypes (see INTEGRATION.md and
 * aicovergen_b200/_ffi.py): plain pointers and sizes only, no torch types.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; the message is
 *     retrievable with b200vc_last_error() (thread local).
 *   - all device pointers are caller-owned CUDA allocations (torch tensors
 *     passed by data_ptr()); fp32 unless stated; the library never frees or
 *     keeps them beyond the stream work it enqueues.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream);
 *     calls are asynchronous unless documented otherwise.
 *   - activations are channels-last: 1-D signals [T, C], images [H, W, C].
 */
#ifndef B200VC_H_
#define B200VC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200VC_MAX_TAPS 128

/* activation codes */
enum {
  B200VC_ACT_NONE = 0,
  B200VC_ACT_RELU = 1,
  B200VC_ACT_LRELU = 2,
  B200VC_ACT_GELU = 3,
  B200VC_ACT_TANH = 4,
  B200VC_ACT_SIGMOID = 5,
  B200VC_ACT_EXP = 6
};

/* which kernel family executes a tap-GEMM */
enum {
  B200VC_BACKEND_SIMT_FP32 = 0, /* exact fp32 FMA kernel                      */
  B200VC_BACKEND_TC_TF32 = 1,   /* wgmma (TF32, or fp16 per `dtype`), TMA-fed, fp32 register accumulators. Picks the
                                   weight-stationary + halo kernel (tapgemm_ws.cu) for small-channel regular
                                   convolutions, else the persistent kernel (tapgemm_tc.cu)                         */
  B200VC_BACKEND_TC_TF32_PERSISTENT = 2, /* persistent launch of tapgemm_tc.cu (one CTA per SM walks the tiles)        */
  B200VC_BACKEND_TC_TF32_TILE = 3,       /* one tile per CTA launch of tapgemm_tc.cu                                  */
  B200VC_BACKEND_TC_TF32_WS = 4          /* force tapgemm_ws.cu (error if the descriptor does not qualify)            */
};

typedef struct b200vc_tap {
  int32_t c_off; /* channel offset inside A dim 0                     */
  int16_t dw;    /* offset along A dim 1                              */
  int16_t dh;    /* offset along A dim 2                              */
  int16_t dp;    /* coordinate along A dim 4                          */
  int16_t widx;  /* weight slice multiplied with this tap             */
} b200vc_tap;

/* Tap-GEMM problem descriptor:
 *   D[pixel, n] = sum_tap sum_{k<Kc} A[pixel + tap, tap.c_off + k] * W[tap.widx + b*w_batch_step, n, k]
 * Replaces F.conv1d / F.conv2d / F.conv_transpose1d/2d / F.linear / torch.matmul
 * calls at: infer_pack/modules.py:196,206,304,308 ; infer_pack/models.py:97,105,497-514 ;
 * infer_pack/attentions.py:217-223,233,263,392-398 ; rmvpe.py:27-49,147-155,241,245 ;
 * fairseq HubertModel (vc_infer_pipeline.py:405) ; the ONNX session at mdx.py:77 ;
 * the STFT/iSTFT DFTs at mdx.py:39,53 and rmvpe.py:305. */
typedef struct b200vc_tapgemm_params {
  const float* A;
  int32_t a_dim[5];     /* extents (c, w, h, b, p)                            */
  int64_t a_stride[5];  /* element strides, a_stride[0] == 1                  */
  const float* Wt;
  int64_t ldw, wstride; /* weight strides: (k, n, widx) = (1, ldw, wstride)   */
  int32_t w_batch_step;
  int32_t Kc, N, ntaps;
  int32_t OW, OH, OB;   /* output pixel space                                 */
  int32_t BW, BH;       /* tile box, BW*BH == 128                             */
  int32_t osh, osw, ooh, oow; /* out pixel = (h*osh+ooh, w*osw+oow)           */
  int32_t o_fh, o_fw;   /* full output extents: mapped pixel must lie in [0,o_fh) x [0,o_fw) */
  int64_t o_sb, o_sh, o_sw;   /* output element strides                       */
  int64_t r_sb, r_sh, r_sw;   /* residual #1 element strides (pixel b,h,w)    */
  int64_t o_sn, r_sn;   /* element stride of the n (channel) index in out/res2 and in res: 1 = channels-last; any
                           other value writes/reads a transposed layout (MDX-Net TDF: NHCW <-> NHWC)            */
  int64_t o2_sb, o2_sh, o2_sw, o2_sn; /* out2 strides when out2_own != 0 (addressed by the mapped output pixel) */
  int32_t out2_own;     /* 0: out2 shares out's addressing; 1: out2 uses the o2_* strides                       */
  const float* row_scale_pre; /* optional: acc *= row_scale_pre[h*OW + w] BEFORE the bias                        */
  const float* bias;
  int32_t bias_per_row;
  int32_t act_pre;
  float act_pre_p;
  const float* row_scale; /* optional: v *= row_scale[h*OW + w] after act_pre (per-output-row scale)   */
  /* epilogue: v = acc * row_scale_pre + bias; v = act_pre(v); v *= row_scale; v (+|*)= res; v *= scale; v += res2;
   *           v = act_post(v); out = v; out2 = act2(v)                                                         */
  const float* res;
  int32_t res_op;       /* bit0: v *= res instead of v += res (MDX-Net multiplicative skip); bit1: address res by the
                           mapped output pixel (h*osh+ooh, w*osw+oow) instead of the GEMM pixel */
  float scale;
  const float* res2;
  int32_t act_post;
  float act_post_p;
  float* out;
  float* out2;
  int32_t act2;
  float act2_p;
  int32_t vec4;         /* vectorisation licences (a bit is also set when its tensor is absent): 1 = k-vectorised operand
                           loads; 2 = out/res2 (and a layout-sharing out2) channels-last + 16-byte aligned; 4 = per-column
                           bias float4-loadable; 8 = own-layout out2 channels-last + aligned; 16 = res likewise        */
  int32_t round_tf32;   /* bit0: round `out` to TF32 (RN), bit1: round `out2` — for tensors only consumed by TF32 GEMMs */
  int32_t dtype;        /* element types (0 = everything fp32): bit0 A and W are IEEE fp16 (wgmma f16, fp32
                           accumulate; same 10-bit mantissa as TF32 at half the operand bytes) — tensor-core backends
                           only; bit1 out, bit2 out2, bit3 res, bit4 res2 are fp16.  Pointers stay typed `float*` in
                           this struct; offsets and strides are in ELEMENTS of the tensor's own type. */
  int32_t split;        /* 3xTF32 split-operand storage (fp32 accuracy on the TF32 tensor core: x = hi + lo with hi = RN_tf32(x),
                           lo = RN_tf32(x - hi); a consumer GEMM reads the K-concatenation [hi | lo | hi] against weights
                           [W_hi | W_hi | W_lo], i.e. hi.W_hi + lo.W_hi + hi.W_lo, dropping only lo.W_lo ~ 2^-22):
                           bit0: `out` is written as three planes hi | lo | hi, plane p at element offset p * o_split;
                           bit1: `res` is such a split tensor: the residual value is res[..] + res[.. + r_split].       */
  int64_t o_split, r_split;
  const float* acc_in;  /* optional fp32 partial sums (channels-last, element (b,h,w,n) at b*ai_sb + h*ai_sh + w*ai_sw + n) added to
                           the accumulator BEFORE the epilogue: a long reduction is split over several launches (subsets of the
                           taps) so that no tensor-core accumulation chain is longer than a few hundred K=8 steps — the tensor
                           core rounds its fp32 accumulator toward zero, CUDA-core adds between launches round to nearest.     */
  int64_t ai_sb, ai_sh, ai_sw;
  b200vc_tap taps[B200VC_MAX_TAPS];
} b200vc_tapgemm_params;

/* ---- library ---- */
const char* b200vc_version(void);
const char* b200vc_last_error(void);
/* number of kernels this library has launched in this process (bench.py: gpu_launches) */
int64_t b200vc_launch_count(void);
/* adds n to that counter: a host that replays a captured CUDA graph of this library's launches accounts for them here */
void b200vc_count_launches(int64_t n);
/* sizeof(b200vc_tapgemm_params) as compiled: bindings verify their struct mirror against it */
int64_t b200vc_sizeof_tapgemm_params(void);

/* ---- launch plans: the per-shape model handle below Python -----------------------------------------------------------
 * A forward pass of any model on the path (HuBERT / rmvpe / synthesizer / MDX-Net for ONE input shape) is a fixed sequence of
 * the launches declared in this header over buffers the caller owns.  b200vc_plan_begin starts RECORDING on the calling
 * thread: until b200vc_plan_end, every tap-GEMM / row-kernel entry point below (all whose pointers are device pointers; not
 * the VC.pipeline glue group) is appended to the plan with a copy of its arguments instead of being launched.
 * b200vc_plan_run(plan, stream) then enqueues the whole forward pass natively — one call per inference, from any host
 * language, and capturable in a CUDA graph.  Replaces the Python-side loops over torch modules at
 * infer_pack/models.py:745-751, rmvpe.py:254-258, fairseq HubertModel.extract_features, and the ort.run call at mdx.py:77. */
typedef struct b200vc_plan b200vc_plan;
int b200vc_plan_begin(b200vc_plan** out);
int b200vc_plan_end(void);
int b200vc_plan_size(const b200vc_plan* plan);                 /* number of recorded launches, -1 for NULL */
int b200vc_plan_run(const b200vc_plan* plan, void* stream);
int b200vc_plan_destroy(b200vc_plan* plan);

/* ---- tap-GEMM ---- */
int b200vc_tapgemm(const b200vc_tapgemm_params* p, int backend, void* stream);
/* experimental: let the persistent tensor-core kernel use 256-row tiles (one weight tile feeds two 128-row blocks); off by default */
int b200vc_tapgemm_set_rows256(int on);
/* 1 when the descriptor satisfies the TMA alignment rules of the tensor-core path */
int b200vc_tapgemm_tc_supported(const b200vc_tapgemm_params* p);
/* 1 when the descriptor is a small-channel regular convolution the weight-stationary kernel handles */
int b200vc_tapgemm_ws_applicable(const b200vc_tapgemm_params* p);

/* ---- row / elementwise kernels (fp32, HBM-bound) ---- */

/* out[r,:] = LayerNorm(x[r,:] + res[r,:]) * gamma + beta over C channels (res may be NULL).
 * Replaces F.layer_norm at infer_pack/modules.py:29-32 and fairseq's LayerNorm calls. */
int b200vc_layernorm(const float* x, const float* res, const float* gamma, const float* beta, float* out,
                     int64_t rows, int C, int64_t ldx, int64_t ldr, int64_t ldo, float eps, int round_out,
                     void* stream);

/* In-place softmax over the last dim of S[heads][rows_per_head][T] (row pitch ld, head pitch head_stride).
 * With emb_rel_k != NULL adds the VITS banded relative-key bias q_i . emb_rel_k[j-i+W] first
 * (infer_pack/attentions.py:238-243,261); q rows are [ldq] wide with head h at column h*dk.
 * S may hold a BLOCK of query rows: local row i is query row0 + i (q is always the full [T, .] matrix). */
int b200vc_softmax_rows(float* S, int heads, int rows_per_head, int T, int64_t ld, int64_t head_stride,
                        const float* q, int ldq, const float* emb_rel_k, int window, int dk,
                        int round_out, int row0, void* stream);

/* out[row0+i, h*dk+d] += sum_r P[h,i,row0+i+r-W] * emb_rel_v[r,d] for the `rows` query rows of the block P
 * (infer_pack/attentions.py:264-271); out is the full [T, .] matrix. */
int b200vc_relpos_value_add(float* out, int ldo, const float* P, int rows, int T, int64_t ld, int64_t head_stride,
                            const float* emb_rel_v, int window, int dk, int heads, int row0, void* stream);

/* out[r,:] = table[idx[r],:]  (nn.Embedding at infer_pack/models.py:97,746) */
int b200vc_gather_rows(const float* table, const int64_t* idx, float* out, int64_t rows, int C, void* stream);

/* out[t,c] = tanh(a[t,c]) * sigmoid(a[t,C+c])  (infer_pack/commons.py:105-112) */
int b200vc_gate_tanh_sigmoid(const float* a, float* out, int64_t rows, int C, int round_out, void* stream);

/* z[t,c] = stats[t,c] + exp(stats[t,C+c]) * noise[c*P+t] * scale  (infer_pack/models.py:748; noise is the
 * caller-supplied randn_like(m_p) draw in the reference's [C,P] layout) */
int b200vc_zp_sample(const float* stats, const float* noise, float* z, int64_t P, int C, float scale, void* stream);

/* out = alpha*a + beta*b (b may be NULL) */
int b200vc_axpby(const float* a, const float* b, float* out, int64_t n, float alpha, float beta, void* stream);

/* out = act(x) elementwise */
int b200vc_act(const float* x, float* out, int64_t n, int act, float p, int round_out, void* stream);

/* NSF harmonic source: har[T*upp] = tanh(lin_w * SineGen(f0, upp, sr; noise) + lin_b)
 * (infer_pack/models.py:320-370 with harmonic_num=0, :414-419). noise[T*upp] is the caller-supplied
 * randn_like(sine_waves) draw; scratch_cum holds T doubles. */
int b200vc_nsf_source(const float* f0, const float* noise, float* har, double* scratch_cum, int T, int upp,
                      float sr, float lin_w, float lin_b, void* stream);

/* Strided Conv1d from ONE input channel as a write-bound row kernel:
 *   out[t,c] = res[t,c] + bias[c] + sum_j w[c,j] * src[src_off + t*stride + j]   (zero outside [0,n_src)); out2 = act2(out)
 * res, bias, out2 may be NULL; res may alias out.  round_out2: bit0 = round out2 to TF32, bit1 = out2 holds IEEE fp16.  Replaces Conv1d(1, C, k, stride) at infer_pack/models.py:477-486,505-506
 * (NSF noise_convs) and HuBERT's first feature-extractor convolution. */
int b200vc_conv1d_from1(const float* src, int64_t n_src, const float* w, const float* bias, const float* res, float* out,
                        float* out2, int64_t T, int C, int K, int stride, int64_t src_off, int act2, float act2_p,
                        int round_out2, void* stream);

/* out[t] = act(sum_k sum_c w[k,c] x[t+k-pad,c]) : Conv1d C->1 (conv_post + tanh, infer_pack/models.py:514-515) */
int b200vc_conv1d_to1(const float* x, const float* w, float* out, int64_t T, int C, int K, int pad, int act,
                      void* stream);

/* ---- RMVPE F0 estimator pieces (rmvpe.py) ---- */

/* out[i] = in[reflect(i - pad)] for i in [0, N+2*pad): torch.stft(center=True) framing (rmvpe.py:305-313, mdx.py:39) */
int b200vc_reflect_pad_1d(const float* in, float* out, int64_t N, int64_t pad, void* stream);

/* mag[t,k] = |spec[t,k] + i spec[t,nb+k]| with zero-filled row tail up to ldm (rmvpe.py:314) */
int b200vc_magnitude(const float* spec, float* mag, int64_t rows, int nb, int64_t lds, int64_t ldm, void* stream);

/* out[t,c] = a*log(max(x[t,c],clampv))+b (clampv < 0: a*x[t,c]+b, x already log-mel) for t<rows, reflect-padded to rows_total rows
 * (rmvpe.py:324 ; the scalar BatchNorm2d(1) of Encoder.bn, rmvpe.py:74,92 ; F.pad reflect, rmvpe.py:353-355) */
int b200vc_logmel_affine_reflect(const float* x, float* out, int rows, int rows_total, int C, float clampv,
                                 float a, float b, void* stream);

/* NHWC 2x2 average pooling; input pixel pitch ldi (nn.AvgPool2d, rmvpe.py:111,117) */
int b200vc_avgpool2x2(const float* in, float* out, int B, int H, int W, int C, int64_t ldi, void* stream);
/* the same on 3xTF32 split tensors (see b200vc_tapgemm_params.split): x = in[..] + in[.. + in_split] is pooled in fp32 and
 * written as planes hi | lo | hi at out + {0,1,2} * out_split; pixel pitches ldi / ldo */
int b200vc_avgpool2x2_split(const float* in, float* out, int B, int H, int W, int C, int64_t ldi, int64_t in_split,
                            int64_t ldo, int64_t out_split, void* stream);

/* Bidirectional GRU recurrence (nn.GRU(384,256,bidirectional), rmvpe.py:8-20) as a 2x8-CTA cluster kernel.
 * xp [T, 2*3H] = x W_ih^T + b_ih (dir d at column d*3H); whh [2,3H,H]; bhh [2,3H]; out [T,2H]. */
int b200vc_bigru(const float* xp, const float* whh, const float* bhh, float* out, int T, int hidden, void* stream);

/* salience [T,n_bins] -> cents[T] and f0[T] = 10*2^(cents/1200) (float64) with numpy's summation order, as
 * RMVPE.to_local_average_cents / decode (rmvpe.py:359-409). cents may be NULL. */
int b200vc_rmvpe_decode(const float* salience, double* f0, double* cents, int T, int n_bins, int64_t ld, float thred,
                        void* stream);

/* Per-channel normalisation over the time axis of x[rows,C] (nn.GroupNorm(C, C) on [1,C,T]) followed by `act`:
 * fairseq ConvFeatureExtractionModel layer 0 (called through vc_infer_pipeline.py:405). stats: 2*C doubles scratch. */
int b200vc_groupnorm_time(const float* x, const float* gamma, const float* beta, float* out, double* stats,
                          int64_t rows, int C, float eps, int act, int round_out, void* stream);

/* ---- crepe F0 estimator pieces (f0_method "mangio-crepe": vc_infer_pipeline.py:96-137 -> torchcrepe.predict) ---- */

/* torchcrepe.preprocess: frame f (f = first_frame .. first_frame+nframes-1) = zero-padded audio[f*hop - win/2 .. + win), minus its
 * mean, divided by max(1e-10, unbiased std); written at out[(f-first_frame)*ldo + off .. + win). */
int b200vc_crepe_frames(const float* audio, int64_t n_audio, int64_t first_frame, int hop, int win, float* out, int64_t ldo,
                        int off, int nframes, int round_out, void* stream);

/* out[r, c] = max(s[c]*x[2r, c] + t[c], s[c]*x[2r+1, c] + t[c]): eval BatchNorm applied AFTER the ReLU + MaxPool2d((2,1)) of
 * every torchcrepe layer (conv -> relu -> BN -> pool), rows = positions, channels-last. */
int b200vc_maxpool2_affine(const float* x, const float* scale, const float* shift, float* out, int64_t rows_out, int C,
                           int round_out, void* stream);

/* torchcrepe.postprocess + the head of librosa.sequence.viterbi: bins outside [lo, hi) -> -inf, softmax over bins (fp32),
 * logp = log(prob + FLT_MIN) (fp32). act, logp: [n, n_bins]. */
int b200vc_crepe_logprob(const float* act, float* logp, int n, int n_bins, int lo, int hi, void* stream);

/* librosa.sequence.viterbi for a banded transition matrix, float64: log_band[from][d] = log T[from -> from + d - (band-1)] for
 * |to - from| < band, every other transition = log_out; uniform start (log_init).  ptr: [n, n_states] scratch; states: [n] out.
 * One thread block; n_states <= 512. */
int b200vc_viterbi_band(const float* logp, const double* log_band, double log_out, double log_init, uint16_t* ptr, int* states,
                        int n, int n_states, int band, void* stream);

/* ---- VC.pipeline glue (vc_infer_pipeline.py) ---- */

/* out[r] = index of the first minimum of S[r, 0..n) */
int b200vc_argmin_rows(const float* S, int* out, int rows, int n, int64_t ld, void* stream);

/* faiss IndexIVFFlat(nprobe=1) search(k=8) + the weighting/blend of vc_infer_pipeline.py:421-431 in one kernel:
 * for query t scan inverted list assign[t] (vectors vecs[offsets[l]..offsets[l+1]), list order), take the 8 smallest
 * squared-L2, w=(1/d)^2 normalised, out = rate * sum w_k v_k + (1-rate) * q.  out_score/out_ids ([T,8]) optional. */
int b200vc_ivf_scan_blend(const float* q, int64_t ldq, const int* assign, const int* offsets, const int64_t* ids,
                          const float* vecs, float* out, int64_t ldo, int T, int d, float rate, float* out_score,
                          int64_t* out_ids, void* stream);

/* F.interpolate(scale_factor=2) (nearest) of feats/feats0 [T,C] -> [P,C] fused with the `protect` blend
 * (vc_infer_pipeline.py:433-452); do_protect=0 only upsamples. */
int b200vc_upsample2_protect(const float* feats, const float* feats0, const float* pitchf, float* out, int64_t P,
                             int C, float protect, int do_protect, void* stream);

/* out[i] = sum_{j<window} x[i+j] in fp64, accumulated in index order exactly like the 160-pass numpy loop at
 * vc_infer_pipeline.py:517-519 (x has n+window-1 valid elements). */
int b200vc_boxsum_f64(const double* x, double* out, int64_t n, int window, void* stream);

/* ---- MDX-Net pass (src/mdx.py) ---- */

/* Build the reflect-padded STFT input of B chunks straight from the song: out[b,ch,j], j in [0, chunk+2*half),
 * = sign * wave[ch, src_start[b] + reflect(j-half)] when that song index is inside [lo[b],hi[b]) else 0
 * (MDX.pad_wave zero regions, mdx.py:156-171, + torch.stft(center=True) reflect padding, mdx.py:39). */
int b200vc_mdx_gather_chunks(const float* wave, int64_t n_song, const int64_t* src_start, const int64_t* lo,
                             const int64_t* hi, float* out, int B, int chunk, int half, float sign, int round_out,
                             void* stream);

/* First / final 1x1 convolutions of the TFC-TDF U-Net (the ONNX graph run at mdx.py:77), as HBM-bound pointwise kernels.
 * first: spec[B][2][T][F][2] (ch, ri) -> out[B][T][F][g] = relu(W4[g][4] . (ch0re, ch0im, ch1re, ch1im) + bias)  (BN folded)
 * final: x[B][T][F][c] -> spec[B][2][T][F][2] = W[4][c] . x + bias                                                  */
int b200vc_mdx_first_conv(const float* spec, const float* w4, const float* bias, float* out, int B, int T, int F, int g,
                          int round_out, int out_half /* out holds fp16 */, void* stream);
int b200vc_mdx_final_conv(const float* x, const float* w, const float* bias, float* spec, int B, int T, int F, int c,
                          int round_out, int x_half /* x holds fp16 */, void* stream);

/* x [R,W,C] -> out [R,C,W] * scale[c] and back with a fused residual add: the layout change around the
 * frequency-axis Linear layers (TDF) of the MDX-Net graph executed at mdx.py:77. */
int b200vc_nhwc_to_nhcw(const float* x, const float* scale, float* out, int64_t R, int W, int C, int round_out,
                        void* stream);
int b200vc_nhcw_to_nhwc_add(const float* t, const float* x, float* out, int64_t R, int W, int C, int round_out,
                            void* stream);

/* torch.istft tail (mdx.py:53) fused with the trim / concat / [:-pad] / margin logic of mdx.py:195-197,107-117:
 * frames [B,2,T,n_fft] = irfft(X)*window; overlap-add, divide by the window envelope env[chunk+n_fft], keep
 * s in [trim, chunk-trim) and write song[ch, dst_start[b]+s-trim] (if inside [keep_lo[b],keep_hi[b])) with
 * song = (accumulate ? song : 0) + coef*y. */
int b200vc_mdx_ola_store(const float* frames, const float* env, const int64_t* dst_start, const int64_t* keep_lo,
                         const int64_t* keep_hi, float* song, int64_t n_song, int B, int T, int n_fft, int hop,
                         int chunk, int trim, float coef, int accumulate, void* stream);

/* proc *= peak; inverse = -proc*compensation + wave_norm   (mdx.py:267, 280) */
int b200vc_mdx_finalize(float* proc, const float* wave_norm, float* inverse, int64_t n, float peak,
                        float compensation, void* stream);

/* ---- ingest / mix stand-ins (SURVEY.md 8(f) "next" rows; not parity-claimed against ffmpeg/pydub) ---- */

/* out[m] = band-limited (Hann-windowed sinc) resample of the channel mean of x[channels, n_in]; ratio = rate_in/rate_out.
 * Stands where my_utils.load_audio's ffmpeg "-ac 1 -ar 16000" stands (my_utils.py:13-17). */
int b200vc_resample_sinc_mono(const float* x, int64_t n_in, int channels, float* out, int64_t n_out, double ratio,
                              int zero_crossings, void* stream);

/* ---- vocal effects + final mix (main.add_audio_effects main.py:206-226, main.combine_audio main.py:229-233) ---- */

/* pedalboard HighpassFilter (JUCE dsp::IIR first-order high-pass, TDF-II: y = b0 x + s; s = b1 x - a1 y) followed by
 * pedalboard Compressor (JUCE dsp::Compressor: peak BallisticsFilter env += cte (env - |y|) with cte = cte_at when rising else
 * cte_rl; gain = env < thr ? 1 : (env * thr_inv) ^ expo).  x: the int16 WAV samples (mono), read as x * 2^-15; y: float out.
 * The signal is processed in chunks of `chunk` samples, each recomputed from `warm` samples earlier with zero state (chunk, warm:
 * multiples of 8; x, y, env_scratch [n]: 16-byte aligned); env_scratch receives the envelope. */
int b200vc_fx_hpf_comp(const int16_t* x, float* y, float* env_scratch, int64_t n, int chunk, int warm, float b0, float b1, float a1,
                       float cte_at, float cte_rl, float thr, float thr_inv, float expo, void* stream);

/* juce::Reverb, mono: the eight parallel comb filters (delays8: HOST array; input x * gain, damping low-pass `damp`, feedback)
 * written as their delay-line contents Y [8, n] (scratch) and summed into comb_sum [n].  terms = Horner terms of the damping
 * low-pass (damp^terms below float resolution). */
int b200vc_fx_reverb_combs(const float* x, float* Y, float* comb_sum, int64_t n, const int* delays8, float gain, float damp,
                           float feedback, int terms, void* stream);

/* juce::Reverb AllPassFilter (gain 0.5): out[t] = w[t - delay] - in[t], w[t] = in[t] + 0.5 w[t - delay]; in != out. */
int b200vc_fx_allpass(const float* in, float* out, int64_t n, int delay, int terms, void* stream);

/* samples = reverb * wet1 + x * dry, then JUCE's float -> 16-bit WAV conversion (int32 full scale, round-half-even, >> 16).
 * out_f (optional): the float samples before the conversion. */
int b200vc_fx_finish(const float* reverb, const float* x, int16_t* out16, float* out_f, int64_t n, float wet1, float dry,
                     void* stream);

/* x [channels, n] float (a stem in HBM) -> out [n, channels] int16 as soundfile writes a float array to a PCM_16 WAV
 * (mdx.py:273,280; libsndfile with clipping on: lrintf(x * 2^31) >> 16, saturated). */
int b200vc_pcm16_from_planar(const float* x, int64_t n, int channels, int16_t* out, void* stream);

/* One operand of the pydub mix: interleaved int16 frames as read from the WAV file. */
typedef struct b200vc_mix_source {
  const int16_t* x; /* DEVICE [n, channels] */
  int64_t n;        /* frames */
  int64_t used;     /* frames of the (rate-converted) segment that take part in the overlay */
  int32_t channels; /* 1 or 2; mono is copied to both channels (audioop.tostereo) */
  int32_t in_rate;  /* frame rate of the file */
  int32_t out_rate; /* frame rate of the mix (AudioSegment._sync: the maximum); != in_rate -> audioop.ratecv */
  int32_t pad_;
  double gain1;     /* AudioSegment - x   -> audioop.mul(data, 2, 10 ** (-x / 20)) */
  double gain2;     /* AudioSegment + g   -> a second audioop.mul */
} b200vc_mix_source;

/* main.combine_audio up to the encoder: out[j, c] = clip(clip(s0 + s1) + s2), s_i = ratecv(mul(mul(x_i, g1), g2)), bit-exact
 * against CPython's audioop (what pydub 0.25.1 calls).  src3: HOST array of 3; out: DEVICE int16 [n_out, channels]. */
int b200vc_pydub_mix(const b200vc_mix_source* src3, int16_t* out, int64_t n_out, int channels, void* stream);

/* change_rms (vc_infer_pipeline.py:41-60) on the device: half-second RMS envelopes of data1 (fp64, rate sr1) and data2
 * (fp32, rate sr2; librosa.feature.rms center/reflect), linear interpolation to n2 samples, data2 *= rms1^(1-rate) *
 * max(rms2,1e-6)^(rate-1) in place. scratch: (2 + n1/(sr1/2) + n2/(sr2/2)) doubles. */
int b200vc_change_rms(const double* data1, int64_t n1, int sr1, float* data2, int64_t n2, int sr2, double rate,
                      double* scratch, void* stream);

/* Peak guard + int16 conversion of vc_infer_pipeline.py:645-649: scale by 32768 (or 32768/(max|x|/0.99) when that
 * exceeds 1) and truncate toward zero. scratch_absmax: one float. */
int b200vc_to_int16_peak_guard(const float* x, int64_t n, float* scratch_absmax, int16_t* out, void* stream);

/* Zero-phase IIR as a cascade of `nsec` second-order sections, fp64, block-parallel: scipy.signal.sosfiltfilt semantics
 * (odd extension by padlen, sosfilt_zi initial conditions). Replaces signal.filtfilt(bh, ah, audio) at
 * vc_infer_pipeline.py:22,513 (the two scipy forms of this filter agree to ~7e-7; this matches sosfiltfilt to ~4e-13).
 * sos_host: HOST [nsec,6]; zi_dev [nsec,2], H_dev [nsec,L,2] (zero-input responses), ML_dev [nsec,4] (L-step state
 * transition): DEVICE tables prepared by the caller; work: 2*(n+2*padlen) + 2 + 4*ceil((n+2*padlen)/L) doubles. */
int b200vc_sosfiltfilt_f64(const float* x, int64_t n, const double* sos_host, int nsec, const double* zi_dev,
                           const double* H_dev, const double* ML_dev, int L, int padlen, double* work, double* out,
                           void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200VC_H_ */
