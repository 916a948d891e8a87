// Row kernels of the crepe F0 path (`f0_method="mangio-crepe"`, vc_infer_pipeline.py:96-137 -> torchcrepe.predict).
// The six convolutions and the classifier of torchcrepe's Crepe('full') run as tap-GEMMs on the tensor cores; what is left is
// framing + per-frame normalisation, the (ReLU ->) BatchNorm -> MaxPool tail of every layer, the masked softmax / log of
// the decoder input and the Viterbi recursion itself (librosa.sequence.viterbi with torchcrepe's banded transition).
#include "common.cuh"
#include "../../include/b200vc.h"
#include <cfloat>

namespace b200vc {
namespace {

static inline unsigned blocks_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// torchcrepe.preprocess: frame f = audio_pad[f*hop : f*hop + win] (audio_pad = zero-padded by win/2 on both sides, handled
// here by index range), minus its mean, divided by max(1e-10, unbiased std); written at out[f*ldo + off .. + win).
__global__ void crepe_frames_kernel(const float* __restrict__ audio, long long n_audio, long long f0, int hop, int win,
                                    float* __restrict__ out, long long ldo, int off, int nframes, int round_out) {
  const int f = blockIdx.x;
  if (f >= nframes) return;
  const long long start = (f0 + f) * (long long)hop - win / 2;
  float s = 0.f;
  for (int i = threadIdx.x; i < win; i += blockDim.x) {
    const long long j = start + i;
    s += (j >= 0 && j < n_audio) ? audio[j] : 0.f;
  }
  __shared__ float red[32];
  __shared__ float stat[2];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) stat[0] = v / win;
  }
  __syncthreads();
  const float mean = stat[0];
  float q = 0.f;
  for (int i = threadIdx.x; i < win; i += blockDim.x) {
    const long long j = start + i;
    const float d = ((j >= 0 && j < n_audio) ? audio[j] : 0.f) - mean;
    q += d * d;
  }
  q = warp_sum(q);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) stat[1] = fmaxf(1e-10f, sqrtf(v / (win - 1)));
  }
  __syncthreads();
  const float inv = 1.f / stat[1];
  for (int i = threadIdx.x; i < win; i += blockDim.x) {
    const long long j = start + i;
    const float v = (((j >= 0 && j < n_audio) ? audio[j] : 0.f) - mean) * inv;
    out[(long long)f * ldo + off + i] = round_out ? round_tf32(v) : v;
  }
}

// BatchNorm (eval, applied AFTER the ReLU in torchcrepe: conv -> relu -> BN -> max_pool (2,1)) fused with the pooling:
// out[b, p, c] = max(s_c * x[b, 2p, c] + t_c, s_c * x[b, 2p+1, c] + t_c)
__global__ void maxpool2_affine_kernel(const float* __restrict__ x, const float* __restrict__ s, const float* __restrict__ t,
                                       float* __restrict__ out, long long rows_out, int C, int round_out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows_out * (C / 4)) return;
  const long long r = e / (C / 4);
  const int c = (int)(e % (C / 4)) * 4;
  const float4 a = *reinterpret_cast<const float4*>(x + (2 * r) * C + c);
  const float4 b = *reinterpret_cast<const float4*>(x + (2 * r + 1) * C + c);
  const float4 sc = __ldg(reinterpret_cast<const float4*>(s + c)), sh = __ldg(reinterpret_cast<const float4*>(t + c));
  float4 o;
  o.x = fmaxf(a.x * sc.x + sh.x, b.x * sc.x + sh.x);
  o.y = fmaxf(a.y * sc.y + sh.y, b.y * sc.y + sh.y);
  o.z = fmaxf(a.z * sc.z + sh.z, b.z * sc.z + sh.z);
  o.w = fmaxf(a.w * sc.w + sh.w, b.w * sc.w + sh.w);
  if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
  *reinterpret_cast<float4*>(out + r * C + c) = o;
}

// torchcrepe.postprocess + the head of decode.viterbi / librosa.sequence.viterbi: bins outside [lo, hi) -> -inf, softmax
// over bins (fp32), log(prob + tiny_f32) in fp32.  One warp per frame.
__global__ void crepe_logprob_kernel(const float* __restrict__ act, float* __restrict__ logp, int n, int nb, int lo, int hi) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n) return;
  const float* a = act + (long long)w * nb;
  float m = -INFINITY;
  for (int k = lo + lane; k < hi; k += 32) m = fmaxf(m, a[k]);
  m = warp_max(m);
  float s = 0.f;
  for (int k = lo + lane; k < hi; k += 32) s += expf(a[k] - m);
  s = warp_sum(s);
  for (int k = lane; k < nb; k += 32) {
    const float p = (k >= lo && k < hi) ? expf(a[k] - m) / s : 0.f;
    logp[(long long)w * nb + k] = logf(p + FLT_MIN);
  }
}

// Viterbi recursion over n steps and NS <= 512 states with a banded transition (|from - to| < W carries log_band[from][d],
// everything else the constant log_out): value_t[j] = logp_t[j] + max_k (value_{t-1}[k] + logT[k -> j]); ptr_t[j] = argmax.
// One block, one thread per state; the out-of-band term needs only the global maximum of value_{t-1}.  float64 like librosa.
constexpr int VIT_MAX = 512;
__global__ void __launch_bounds__(VIT_MAX)
viterbi_band_kernel(const float* __restrict__ logp, const double* __restrict__ log_band /*[NS][2W-1]*/, double log_out,
                    double log_init, unsigned short* __restrict__ ptr, int* __restrict__ states, int n, int NS, int W) {
  __shared__ double val[2][VIT_MAX];
  __shared__ double wmax[VIT_MAX / 32];
  __shared__ int warg[VIT_MAX / 32];
  __shared__ double gmax_s;
  __shared__ int garg_s;
  const int j = threadIdx.x;
  const int nw = (blockDim.x + 31) >> 5;
  if (j < NS) val[0][j] = (double)logp[j] + log_init;
  __syncthreads();
  for (int t = 1; t < n; ++t) {
    const int cur = (t - 1) & 1, nxt = t & 1;
    // global (max, first argmax) of val[cur]
    double v = j < NS ? val[cur][j] : -INFINITY;
    int a = j < NS ? j : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oa = __shfl_xor_sync(0xffffffffu, a, o);
      if (ov > v || (ov == v && oa < a)) { v = ov; a = oa; }
    }
    if ((j & 31) == 0) { wmax[j >> 5] = v; warg[j >> 5] = a; }
    __syncthreads();
    if (j < 32) {
      v = j < nw ? wmax[j] : -INFINITY;
      a = j < nw ? warg[j] : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oa = __shfl_xor_sync(0xffffffffu, a, o);
        if (ov > v || (ov == v && oa < a)) { v = ov; a = oa; }
      }
      if (j == 0) { gmax_s = v; garg_s = a; }
    }
    __syncthreads();
    if (j < NS) {
      double best = -INFINITY;
      int bk = 0;
      const int k0 = max(0, j - (W - 1)), k1 = min(NS - 1, j + (W - 1));
      // numpy.argmax over k = 0..NS-1 returns the FIRST maximum: out-of-band candidates below the band come first
      const int ga = garg_s;
      const double go = gmax_s + log_out;
      if (ga < k0) { best = go; bk = ga; }
      for (int k = k0; k <= k1; ++k) {
        const double c = val[cur][k] + log_band[k * (2 * W - 1) + (j - k + W - 1)];
        if (c > best) { best = c; bk = k; }
      }
      if (ga > k1 && go > best) { best = go; bk = ga; }
      val[nxt][j] = (double)logp[(long long)t * NS + j] + best;
      ptr[(long long)t * NS + j] = (unsigned short)bk;
    }
    __syncthreads();
  }
  // backtrack (single thread; ptr reads are dependent)
  if (j == 0) {
    const int last = (n - 1) & 1;
    double best = -INFINITY;
    int bs = 0;
    for (int k = 0; k < NS; ++k)
      if (val[last][k] > best) { best = val[last][k]; bs = k; }
    states[n - 1] = bs;
    for (int t = n - 2; t >= 0; --t) {
      bs = ptr[(long long)(t + 1) * NS + bs];
      states[t] = bs;
    }
  }
}

}  // namespace
}  // namespace b200vc

using namespace b200vc;

extern "C" {

int b200vc_crepe_frames(const float* audio, int64_t n_audio, int64_t first_frame, int hop, int win, float* out, int64_t ldo,
                        int off, int nframes, int round_out, void* stream) {
  B200VC_RECORD(b200vc_crepe_frames(audio, n_audio, first_frame, hop, win, out, ldo, off, nframes, round_out, stream));
  B200VC_REQUIRE(audio && out && n_audio > 0 && hop > 0 && win > 1 && nframes > 0 && ldo >= off + win, "crepe_frames: bad args");
  crepe_frames_kernel<<<(unsigned)nframes, 256, 0, (cudaStream_t)stream>>>(audio, n_audio, first_frame, hop, win, out, ldo, off, nframes,
                                                                        round_out);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_maxpool2_affine(const float* x, const float* scale, const float* shift, float* out, int64_t rows_out, int C,
                           int round_out, void* stream) {
  B200VC_RECORD(b200vc_maxpool2_affine(x, scale, shift, out, rows_out, C, round_out, stream));
  B200VC_REQUIRE(x && scale && shift && out && rows_out > 0 && C > 0 && C % 4 == 0, "maxpool2_affine: bad args (C=%d)", C);
  maxpool2_affine_kernel<<<blocks_for(rows_out * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(x, scale, shift, out, rows_out, C, round_out);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_crepe_logprob(const float* act, float* logp, int n, int n_bins, int lo, int hi, void* stream) {
  B200VC_RECORD(b200vc_crepe_logprob(act, logp, n, n_bins, lo, hi, stream));
  B200VC_REQUIRE(act && logp && n > 0 && n_bins > 0 && 0 <= lo && lo < hi && hi <= n_bins, "crepe_logprob: bad args");
  crepe_logprob_kernel<<<blocks_for((long long)n * 32, 256), 256, 0, (cudaStream_t)stream>>>(act, logp, n, n_bins, lo, hi);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_viterbi_band(const float* logp, const double* log_band, double log_out, double log_init, uint16_t* ptr, int* states,
                        int n, int n_states, int band, void* stream) {
  B200VC_RECORD(b200vc_viterbi_band(logp, log_band, log_out, log_init, ptr, states, n, n_states, band, stream));
  B200VC_REQUIRE(logp && log_band && ptr && states && n > 0 && n_states > 0 && n_states <= VIT_MAX && band >= 1, "viterbi_band: bad args");
  const int threads = ((n_states + 31) / 32) * 32;
  viterbi_band_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(logp, log_band, log_out, log_init, ptr, states, n, n_states, band);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

}  // extern "C"
