// "Tap-GEMM": the one implicit-GEMM formulation every conv / linear / batched
// matmul on the hot path is lowered to.
//
//   D[pixel, n] = sum_{tap} sum_{k < Kc}  A[pixel + tap.offset, tap.c_off + k] * W[tap.widx (+batch), n, k]
//
// * A is a rank-5 strided view (c, w, h, b, p) of a channels-last fp32 tensor;
//   out-of-range coordinates read as zero (this is the conv zero padding).
// * Output pixels are tiled BW x BH (BW*BH == 128 GEMM rows per tile).
// * The epilogue (bias / activation / residuals / scale / second output) is
//   shared verbatim by the SIMT fp32 kernel and the wgmma tensor-core kernels so
//   all produce the same graph semantics.
//
// Reference call sites this replaces (all cuDNN/cuBLAS library calls there):
//   infer_pack/modules.py:299-312 (ResBlock1 convs), models.py:494-516
//   (GeneratorNSF), modules.py:188-213 (WN), attentions.py:216-275 (1x1 convs,
//   QK^T / PV matmuls), rmvpe.py:23-58 (Conv2d 3x3), fairseq HuBERT convs and
//   linears, mdx.py:77 (the ONNX TFC-TDF net).
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>
#include "../../include/b200vc.h"

namespace b200vc {

constexpr int TG_MAX_TAPS = B200VC_MAX_TAPS;
constexpr int TG_TILE_M = 128;

// The descriptor is the public C struct (include/b200vc.h); see there for field docs.
//   epilogue: v = acc + bias; v = act_pre(v); v += res; v *= scale; v += res2;
//             v = act_post(v); out = v; out2 = act2(v)
using TgTap = b200vc_tap;
using TgParams = b200vc_tapgemm_params;

// dtype bits (b200vc.h): which tensors hold IEEE fp16 instead of fp32
constexpr int TG_DT_AB = 1, TG_DT_OUT = 2, TG_DT_OUT2 = 4, TG_DT_RES = 8, TG_DT_RES2 = 16;
constexpr int TG_DT_EPI = TG_DT_OUT | TG_DT_OUT2 | TG_DT_RES | TG_DT_RES2;

__device__ __forceinline__ float tg_ld(const float* base, long long idx, bool half) {
  return half ? __half2float(reinterpret_cast<const __half*>(base)[idx]) : base[idx];
}
__device__ __forceinline__ void tg_st(float* base, long long idx, float v, bool half) {
  if (half) reinterpret_cast<__half*>(base)[idx] = __float2half_rn(v);
  else base[idx] = v;
}

// One GEMM row's addressing state.
struct TgRow {
  long long o_off;   // offset into out/res2 (n * o_sn added later)
  long long r_off;   // offset into res (n * r_sn added later)
  long long o2_off;  // offset into out2 (n * its n-stride added later)
  long long a_off;   // offset into acc_in (n added later)
  int brow;          // index for per-row bias / row scales
  bool valid;
};

__device__ __forceinline__ TgRow tg_row(const TgParams& p, int b, int h, int w) {
  TgRow r;
  const int mh = h * p.osh + p.ooh, mw = w * p.osw + p.oow;
  r.valid = (h < p.OH) && (w < p.OW) && (b < p.OB) && (mh >= 0) && (mh < p.o_fh) && (mw >= 0) &&
            (mw < p.o_fw);
  r.o_off = (long long)b * p.o_sb + (long long)mh * p.o_sh + (long long)mw * p.o_sw;
  // residual #1 is addressed by the GEMM pixel, or by the mapped output pixel when res_op bit1 is set
  if (p.res_op & 2) r.r_off = (long long)b * p.r_sb + (long long)mh * p.r_sh + (long long)mw * p.r_sw;
  else r.r_off = (long long)b * p.r_sb + (long long)h * p.r_sh + (long long)w * p.r_sw;
  r.o2_off = p.out2_own ? (long long)b * p.o2_sb + (long long)mh * p.o2_sh + (long long)mw * p.o2_sw : r.o_off;
  r.brow = h * p.OW + w;
  r.a_off = (long long)b * p.ai_sb + (long long)h * p.ai_sh + (long long)w * p.ai_sw;
  return r;
}

__device__ __forceinline__ float tg_epi1(const TgParams& p, const TgRow& r, int n, float acc) {
  float v = acc;
  if (p.acc_in) v += p.acc_in[r.a_off + n];
  if (p.row_scale_pre) v *= __ldg(p.row_scale_pre + r.brow);
  if (p.bias) v += p.bias_per_row ? __ldg(p.bias + r.brow) : __ldg(p.bias + n);
  v = apply_act(v, p.act_pre, p.act_pre_p);
  if (p.row_scale) v *= __ldg(p.row_scale + r.brow);
  if (p.res) {
    float rr = tg_ld(p.res, r.r_off + n * p.r_sn, p.dtype & TG_DT_RES);
    if (p.split & 2) rr += p.res[r.r_off + n * p.r_sn + p.r_split];      // split residual: hi + lo
    v = (p.res_op & 1) ? v * rr : v + rr;
  }
  v *= p.scale;
  if (p.res2) v += tg_ld(p.res2, r.o_off + n * p.o_sn, p.dtype & TG_DT_RES2);
  v = apply_act(v, p.act_post, p.act_post_p);
  return v;
}

// Scalar store of one element (any layout).
__device__ __forceinline__ void tg_store1(const TgParams& p, const TgRow& r, int n, float acc) {
  if (!r.valid || n >= p.N) return;
  float v = tg_epi1(p, r, n, acc);
  if (p.split & 1) {          // 3xTF32 planes hi | lo | hi
    const float hi = round_tf32(v);
    float* o = p.out + r.o_off + n * p.o_sn;
    o[0] = hi; o[p.o_split] = round_tf32(v - hi); o[2 * p.o_split] = hi;
    return;
  }
  tg_st(p.out, r.o_off + n * p.o_sn, (p.round_tf32 & 1) ? round_tf32(v) : v, p.dtype & TG_DT_OUT);
  if (p.out2) {
    float v2 = apply_act(v, p.act2, p.act2_p);
    tg_st(p.out2, r.o2_off + n * (p.out2_own ? p.o2_sn : p.o_sn), (p.round_tf32 & 2) ? round_tf32(v2) : v2, p.dtype & TG_DT_OUT2);
  }
}

// vec4 bits (set by the host binding; a bit is also set when the tensor it talks about is absent)
constexpr int TG_VEC_K = 1;      // k-vectorised operand loads (SIMT kernel)
constexpr int TG_VEC_OUT = 2;    // out / res2 (and out2 when it shares out's layout): channels-last, 16-byte aligned
constexpr int TG_VEC_BIAS = 4;   // per-column bias float4-loadable
constexpr int TG_VEC_OUT2 = 8;   // own-layout out2 channels-last + aligned
constexpr int TG_VEC_RES = 16;   // res channels-last + aligned
constexpr int TG_VEC_ALL = TG_VEC_OUT | TG_VEC_BIAS | TG_VEC_OUT2 | TG_VEC_RES;

// Store 4 consecutive n (n % 4 == 0). Uses float4 when every epilogue tensor is channels-last + aligned and in range.
__device__ __forceinline__ void tg_store4(const TgParams& p, const TgRow& r, int n, float4 acc) {
  if (!r.valid || n >= p.N) return;
  if ((p.vec4 & TG_VEC_ALL) == TG_VEC_ALL && n + 3 < p.N && !(p.dtype & TG_DT_EPI) && !p.split && !p.acc_in) {
    float v[4] = {acc.x, acc.y, acc.z, acc.w};
    if (p.row_scale_pre) {
      const float rs = __ldg(p.row_scale_pre + r.brow);
      v[0] *= rs; v[1] *= rs; v[2] *= rs; v[3] *= rs;
    }
    if (p.bias) {
      if (p.bias_per_row) {
        float bb = __ldg(p.bias + r.brow);
        v[0] += bb; v[1] += bb; v[2] += bb; v[3] += bb;
      } else {
        float4 bb = __ldg(reinterpret_cast<const float4*>(p.bias + n));
        v[0] += bb.x; v[1] += bb.y; v[2] += bb.z; v[3] += bb.w;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = apply_act(v[i], p.act_pre, p.act_pre_p);
    if (p.row_scale) {
      const float rs = __ldg(p.row_scale + r.brow);
      v[0] *= rs; v[1] *= rs; v[2] *= rs; v[3] *= rs;
    }
    if (p.res) {
      float4 rr = *reinterpret_cast<const float4*>(p.res + r.r_off + n);
      if (p.res_op & 1) { v[0] *= rr.x; v[1] *= rr.y; v[2] *= rr.z; v[3] *= rr.w; }
      else { v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w; }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] *= p.scale;
    if (p.res2) {
      float4 rr = *reinterpret_cast<const float4*>(p.res2 + r.o_off + n);
      v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = apply_act(v[i], p.act_post, p.act_post_p);
    if (p.round_tf32 & 1)
      *reinterpret_cast<float4*>(p.out + r.o_off + n) =
          make_float4(round_tf32(v[0]), round_tf32(v[1]), round_tf32(v[2]), round_tf32(v[3]));
    else
      *reinterpret_cast<float4*>(p.out + r.o_off + n) = make_float4(v[0], v[1], v[2], v[3]);
    if (p.out2) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[i] = apply_act(v[i], p.act2, p.act2_p);
        if (p.round_tf32 & 2) v[i] = round_tf32(v[i]);
      }
      *reinterpret_cast<float4*>(p.out2 + r.o2_off + n) = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
    tg_store1(p, r, n + 0, acc.x);
    tg_store1(p, r, n + 1, acc.y);
    tg_store1(p, r, n + 2, acc.z);
    tg_store1(p, r, n + 3, acc.w);
  }
}

// Activation over a register array; the switch is warp-uniform so it costs one branch per group, not per element.
template <int NV>
__device__ __forceinline__ void tg_act_vec(float (&v)[NV], int act, float prm) {
  switch (act) {
    case ACT_NONE: break;
    case ACT_RELU:
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = fmaxf(v[j], 0.f);
      break;
    case ACT_LRELU:
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * prm;
      break;
    default:
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = apply_act(v[j], act, prm);
      break;
  }
}

// 16 values <- 16 consecutive n at `ptr` with element stride `sn` (vector loads when the caller knows sn == 1 and the
// address is 16-byte aligned).
__device__ __forceinline__ void tg_load16(float (&d)[16], const float* ptr, long long sn, bool vec) {
  if (vec) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 t = reinterpret_cast<const float4*>(ptr)[j];
      d[4 * j] = t.x; d[4 * j + 1] = t.y; d[4 * j + 2] = t.z; d[4 * j + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) d[j] = ptr[j * sn];
  }
}
// fp16 tensors: 16 consecutive halfs are one 32-byte sector (two 16-byte vector accesses)
__device__ __forceinline__ void tg_load16h(float (&d)[16], const __half* ptr, long long sn, bool vec) {
  if (vec) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint4 t = reinterpret_cast<const uint4*>(ptr)[j];
      const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        d[8 * j + 2 * i] = f.x;
        d[8 * j + 2 * i + 1] = f.y;
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) d[j] = __half2float(ptr[j * sn]);
  }
}
__device__ __forceinline__ void tg_put16(float* ptr, long long sn, bool vec, bool rnd, const float (&v)[16]) {
  if (vec) {
    float w[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) w[j] = rnd ? round_tf32(v[j]) : v[j];
    float4* op = reinterpret_cast<float4*>(ptr);
#pragma unroll
    for (int j = 0; j < 4; ++j) op[j] = make_float4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
  } else {
    // transposed layouts: consecutive lanes own consecutive pixels, so each of these scalar stores is lane-coalesced
    if (rnd) {
#pragma unroll
      for (int j = 0; j < 16; ++j) ptr[j * sn] = round_tf32(v[j]);
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) ptr[j * sn] = v[j];
    }
  }
}
__device__ __forceinline__ void tg_put16h(__half* ptr, long long sn, bool vec, const float (&v)[16]) {
  if (vec) {
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    reinterpret_cast<uint4*>(ptr)[0] = make_uint4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<uint4*>(ptr)[1] = make_uint4(w[4], w[5], w[6], w[7]);
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) ptr[j * sn] = __float2half_rn(v[j]);
  }
}

// Store 16 consecutive n (n % 16 == 0) of one GEMM row from registers: the epilogue the wgmma kernels use after
// regrouping their accumulator fragments so that one thread owns one row (hopper.cuh, wg_epilogue).  Every stage is a
// pass over the register array behind a warp-uniform test, so a plain bias+activation epilogue is ~5 instructions per
// element.  Same arithmetic, in the same order, as tg_epi1.
__device__ __forceinline__ void tg_store16(const TgParams& p, const TgRow& r, int n, const uint32_t* acc) {
  if (!r.valid || n >= p.N) return;
  if (n + 15 >= p.N) {      // ragged tail of N: element-wise path with bounds checks
#pragma unroll
    for (int j = 0; j < 16; j += 4)
      tg_store4(p, r, n + j, make_float4(__uint_as_float(acc[j]), __uint_as_float(acc[j + 1]), __uint_as_float(acc[j + 2]),
                                         __uint_as_float(acc[j + 3])));
    return;
  }
  const bool vec = (p.vec4 & TG_VEC_OUT) != 0;
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(acc[j]);
  if (p.acc_in) {            // partial sums of earlier launches (split reduction), added in fp32 round-to-nearest
    float pa[16];
    tg_load16(pa, p.acc_in + r.a_off + n, 1, true);
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] += pa[j];
  }
  if (p.row_scale_pre) {
    const float rs = __ldg(p.row_scale_pre + r.brow);
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] *= rs;
  }
  if (p.bias) {
    if (p.bias_per_row) {
      const float bb = __ldg(p.bias + r.brow);
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] += bb;
    } else if (p.vec4 & TG_VEC_BIAS) {
#pragma unroll
      for (int j = 0; j < 16; j += 4) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(p.bias + n + j));
        v[j] += bb.x; v[j + 1] += bb.y; v[j + 2] += bb.z; v[j + 3] += bb.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] += __ldg(p.bias + n + j);
    }
  }
  tg_act_vec(v, p.act_pre, p.act_pre_p);
  if (p.row_scale) {
    const float rs = __ldg(p.row_scale + r.brow);
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] *= rs;
  }
  if (p.res) {
    float rr[16];
    if (p.dtype & TG_DT_RES) tg_load16h(rr, reinterpret_cast<const __half*>(p.res) + r.r_off + n * p.r_sn, p.r_sn, (p.vec4 & TG_VEC_RES) != 0);
    else tg_load16(rr, p.res + r.r_off + n * p.r_sn, p.r_sn, (p.vec4 & TG_VEC_RES) != 0);
    if (p.split & 2) {        // split residual: hi + lo
      float r2[16];
      tg_load16(r2, p.res + r.r_off + n * p.r_sn + p.r_split, p.r_sn, (p.vec4 & TG_VEC_RES) != 0);
#pragma unroll
      for (int j = 0; j < 16; ++j) rr[j] += r2[j];
    }
    if (p.res_op & 1) {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] *= rr[j];
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] += rr[j];
    }
  }
  if (p.scale != 1.f) {
    const float sc = p.scale;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] *= sc;
  }
  if (p.res2) {
    float rr[16];
    if (p.dtype & TG_DT_RES2) tg_load16h(rr, reinterpret_cast<const __half*>(p.res2) + r.o_off + n * p.o_sn, p.o_sn, vec);
    else tg_load16(rr, p.res2 + r.o_off + n * p.o_sn, p.o_sn, vec);
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] += rr[j];
  }
  tg_act_vec(v, p.act_post, p.act_post_p);
  if (p.split & 1) {          // 3xTF32 planes hi | lo | hi (fp32, channels-last)
    float hi[16], lo[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { hi[j] = round_tf32(v[j]); lo[j] = round_tf32(v[j] - hi[j]); }
    float* o = p.out + r.o_off + n * p.o_sn;
    tg_put16(o, p.o_sn, vec, false, hi);
    tg_put16(o + p.o_split, p.o_sn, vec, false, lo);
    tg_put16(o + 2 * p.o_split, p.o_sn, vec, false, hi);
    return;
  }
  if (p.dtype & TG_DT_OUT) tg_put16h(reinterpret_cast<__half*>(p.out) + r.o_off + n * p.o_sn, p.o_sn, vec, v);
  else tg_put16(p.out + r.o_off + n * p.o_sn, p.o_sn, vec, (p.round_tf32 & 1) != 0, v);
  if (p.out2) {
    tg_act_vec(v, p.act2, p.act2_p);
    const long long sn2 = p.out2_own ? p.o2_sn : p.o_sn;
    const bool vec2 = p.out2_own ? (p.vec4 & TG_VEC_OUT2) != 0 : vec;
    if (p.dtype & TG_DT_OUT2) tg_put16h(reinterpret_cast<__half*>(p.out2) + r.o2_off + n * sn2, sn2, vec2, v);
    else tg_put16(p.out2 + r.o2_off + n * sn2, sn2, vec2, (p.round_tf32 & 2) != 0, v);
  }
}

// Host-side launchers (tapgemm_simt.cu / tapgemm_tc.cu / tapgemm_ws.cu).
int tapgemm_simt_launch(const TgParams& p, cudaStream_t stream);
int tapgemm_tc_launch(const TgParams& p, cudaStream_t stream);    // v1: one tile per CTA
int tapgemm_tc2_launch(const TgParams& p, cudaStream_t stream);   // v2: persistent (one CTA per SM walks the tiles)
bool tapgemm_tc_supported(const TgParams& p);
void tapgemm_tc2_set_rows256(int on);                            // experimental 256-row tiles of the persistent kernel
int tapgemm_ws_launch(const TgParams& p, cudaStream_t stream);    // v3: weight-stationary + halo (small-channel convs)
bool tapgemm_ws_applicable(const TgParams& p);

}  // namespace b200vc
