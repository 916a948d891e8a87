// fp32 SIMT tap-GEMM: exact-fp32 path (rmvpe, IVF coarse quantiser, small-K
// layers) and the on-device cross-check for the wgmma kernels.
// 128 x BN output tile, BK = 16, 256 threads, 8 x (BN/16) register tile,
// register-prefetch double buffering.
#include "tapgemm.cuh"

namespace b200vc {

namespace {

constexpr int BK = 16;
constexpr int NT = 256;

template <int BN>
__global__ void __launch_bounds__(NT, BN >= 128 ? 2 : (BN >= 64 ? 3 : 4))
tapgemm_simt_kernel(const __grid_constant__ TgParams p) {
  constexpr int CPT = BN / 16;               // columns per thread
  constexpr int VW = (CPT >= 4) ? 4 : CPT;   // vector width of a column group
  constexpr int NG = CPT / VW;               // column groups per thread
  constexpr int WPT = BN * BK / NT;          // weight elements loaded per thread per chunk
  constexpr int WTPR = BK / WPT;             // threads per weight row
  constexpr int APAD = 4, BPAD = 4;

  __shared__ __align__(16) float As[2][BK][TG_TILE_M + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN + BPAD];

  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;

  // ---- tile coordinates
  const int ntw = (p.OW + p.BW - 1) / p.BW;
  const int nth = (p.OH + p.BH - 1) / p.BH;
  int tile = blockIdx.x;
  const int tw = tile % ntw; tile /= ntw;
  const int th = tile % nth; tile /= nth;
  const int tb = tile;
  const int w0 = tw * p.BW, h0 = th * p.BH;
  const int n0 = blockIdx.y * BN;

  // ---- A loader mapping: row = tid / 2, k half = tid % 2 (8 consecutive k)
  const int a_row = tid >> 1;
  const int a_k0 = (tid & 1) * 8;
  const int a_h = h0 + a_row / p.BW;
  const int a_w = w0 + a_row % p.BW;
  const bool a_vec = p.vec4 & 1;   // host guarantees A/W alignment when set

  // ---- W loader mapping
  const int w_n = tid / WTPR;
  const int w_k0 = (tid % WTPR) * WPT;

  const int kchunks = (p.Kc + BK - 1) / BK;
  const int nchunks = p.ntaps * kchunks;

  float a_reg[8];
  float w_reg[WPT];

  auto prefetch = [&](int chunk) {
    const int tap_i = chunk / kchunks;
    const int kc0 = (chunk - tap_i * kchunks) * BK;
    const TgTap tap = p.taps[tap_i];
    // A
    {
      const int iw = a_w + tap.dw, ih = a_h + tap.dh;
      const bool pix_ok = (iw >= 0) && (iw < p.a_dim[1]) && (ih >= 0) && (ih < p.a_dim[2]) &&
                          (tb < p.a_dim[3]);
      const float* src = p.A + (long long)iw * p.a_stride[1] + (long long)ih * p.a_stride[2] +
                         (long long)tb * p.a_stride[3] + (long long)tap.dp * p.a_stride[4];
      const int kk = kc0 + a_k0;
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        const int k = kk + v * 4;
        const int c = tap.c_off + k;
        if (pix_ok && a_vec && (k + 3 < p.Kc) && (c + 3 < p.a_dim[0])) {
          float4 t = __ldg(reinterpret_cast<const float4*>(src + c));
          a_reg[v * 4 + 0] = t.x; a_reg[v * 4 + 1] = t.y; a_reg[v * 4 + 2] = t.z; a_reg[v * 4 + 3] = t.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const bool ok = pix_ok && (k + j < p.Kc) && (c + j < p.a_dim[0]);
            a_reg[v * 4 + j] = ok ? __ldg(src + c + j) : 0.f;
          }
        }
      }
    }
    // W
    {
      const int n = n0 + w_n;
      const int widx = tap.widx + tb * p.w_batch_step;
      const float* src = p.Wt + (long long)widx * p.wstride + (long long)n * p.ldw;
      const int k = kc0 + w_k0;
      if constexpr (WPT >= 4) {
#pragma unroll
        for (int v = 0; v < WPT / 4; ++v) {
          const int kv = k + v * 4;
          if (n < p.N && a_vec && kv + 3 < p.Kc) {
            float4 t = __ldg(reinterpret_cast<const float4*>(src + kv));
            w_reg[v * 4 + 0] = t.x; w_reg[v * 4 + 1] = t.y; w_reg[v * 4 + 2] = t.z; w_reg[v * 4 + 3] = t.w;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              w_reg[v * 4 + j] = (n < p.N && kv + j < p.Kc) ? __ldg(src + kv + j) : 0.f;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < WPT; ++j)
          w_reg[j] = (n < p.N && k + j < p.Kc) ? __ldg(src + k + j) : 0.f;
      }
    }
  };

  auto stage = [&](int buf) {
#pragma unroll
    for (int j = 0; j < 8; ++j) As[buf][a_k0 + j][a_row] = a_reg[j];
#pragma unroll
    for (int j = 0; j < WPT; ++j) Bs[buf][w_k0 + j][w_n] = w_reg[j];
  };

  float acc[8][CPT];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < CPT; ++j) acc[i][j] = 0.f;

  prefetch(0);
  stage(0);
  __syncthreads();

  for (int chunk = 0; chunk < nchunks; ++chunk) {
    const int buf = chunk & 1;
    if (chunk + 1 < nchunks) prefetch(chunk + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[CPT];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        if constexpr (VW == 4) {
          const float4 t = *reinterpret_cast<const float4*>(&Bs[buf][k][g * 64 + tx * 4]);
          b[g * 4 + 0] = t.x; b[g * 4 + 1] = t.y; b[g * 4 + 2] = t.z; b[g * 4 + 3] = t.w;
        } else {
          const float2 t = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
          b[0] = t.x; b[1] = t.y;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < CPT; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (chunk + 1 < nchunks) {
      stage(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = ty * 8 + i;
    const int h = h0 + m / p.BW, w = w0 + m % p.BW;
    const TgRow r = tg_row(p, tb, h, w);
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      if constexpr (VW == 4) {
        const int n = n0 + g * 64 + tx * 4;
        tg_store4(p, r, n, make_float4(acc[i][g * 4 + 0], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]));
      } else {
        const int n = n0 + tx * 2;
        tg_store1(p, r, n, acc[i][0]);
        tg_store1(p, r, n + 1, acc[i][1]);
      }
    }
  }
}

}  // namespace

int tapgemm_simt_launch(const TgParams& p, cudaStream_t stream) {
  B200VC_REQUIRE(p.dtype == 0, "tapgemm_simt: the exact-fp32 kernel takes fp32 tensors only (dtype flags 0x%x)", p.dtype);
  const int ntw = ceil_div(p.OW, p.BW), nth = ceil_div(p.OH, p.BH);
  const long long tiles = (long long)ntw * nth * p.OB;
  B200VC_REQUIRE(tiles > 0 && tiles < (1ll << 31), "tapgemm: bad tile count %lld", tiles);
  dim3 block(NT);
  if (p.N > 64) {
    dim3 grid((unsigned)tiles, ceil_div(p.N, 128));
    tapgemm_simt_kernel<128><<<grid, block, 0, stream>>>(p);
  } else if (p.N > 32) {
    dim3 grid((unsigned)tiles, 1);
    tapgemm_simt_kernel<64><<<grid, block, 0, stream>>>(p);
  } else {
    dim3 grid((unsigned)tiles, 1);
    tapgemm_simt_kernel<32><<<grid, block, 0, stream>>>(p);
  }
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

}  // namespace b200vc
