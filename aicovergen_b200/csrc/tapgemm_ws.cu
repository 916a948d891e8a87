// wgmma tap-GEMM v3: WEIGHT-STATIONARY + INPUT-HALO kernel for small-channel convolutions (Cout <= 64).
//
// The one-tile-per-CTA kernel re-reads the input tile once per tap and the whole weight slab once per tile from L2.  Here:
//   * every CTA is persistent and first parks ALL weights of the layer in shared memory (ntaps x kchunks tiles of
//     [Nr x 128 B]) — they are never fetched again;
//   * per output tile (1 x 128 pixel strip) and 128-byte K chunk ONE TMA box brings the strip WITH ITS HALO
//     ([KH rows] x [128 + (KW-1)*dil] pixels); the taps are just row offsets of the wgmma A descriptor inside that box
//     (the 128-byte swizzle is a function of absolute shared-memory address bits, so shifting the start address by whole
//     128-byte rows keeps TMA's layout and the descriptor's view consistent);
//   * warpgroup 0 is the TMA producer, warpgroups 1-2 each own 64 rows of the strip and accumulate all taps of a chunk
//     with m64 x Nr wgmma; the producer keeps fetching the next strips' halo boxes while they run the epilogue.
// L2->SM traffic per tile drops to the halo box only (for MDX-Net's c=48 3x3 layers ~100 KB instead of ~430 KB).
#include "hopper.cuh"

namespace b200vc {

using namespace hop;

namespace {

constexpr int NUM_THREADS = 3 * WG_THREADS;
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int MAX_STAGES = 4;

struct WsGeom {
  int KH, KW, dil_w, dil_h, pad_w, pad_h;
  int BWh;            // halo box width in pixels = 128 + (KW-1)*dil_w
  int a_stage_bytes;  // KH * BWh * 128 rounded up to 1024
  int b_tile_bytes;   // Nr * 128
  int Nr;             // wgmma N: N rounded up to 16, at least 32
  int stages;
  int total_tiles;
};

// Tile walker: tile = first + i * stride decomposed into (strip, row, batch) and advanced with carries.
struct TileWalk {
  int tw, h, b;        // current coordinates
  int dw, dh, db;      // stride decomposition
  int left;            // tiles still to process
  __device__ __forceinline__ void init(int first, int stride, int total, int ntw, int OH) {
    tw = first % ntw; int t = first / ntw; h = t % OH; b = t / OH;
    dw = stride % ntw; t = stride / ntw; dh = t % OH; db = t / OH;
    left = first < total ? (total - first + stride - 1) / stride : 0;
  }
  __device__ __forceinline__ void next(int ntw, int OH) {
    tw += dw; if (tw >= ntw) { tw -= ntw; ++h; }
    h += dh; if (h >= OH) { h -= OH; ++b; }
    b += db;
    --left;
  }
};

template <int NR, bool F16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapgemm_ws_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                  const __grid_constant__ TgParams p, const WsGeom g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  constexpr int KE = F16 ? 2 * KCHUNK : KCHUNK;       // K elements per 128-byte chunk row
  constexpr int ES = F16 ? 2 : 4;
  const int kchunks = (p.Kc + KE - 1) / KE;
  const int w_bytes = p.ntaps * kchunks * g.b_tile_bytes;
  const uint32_t w_base = smem_base;                              // resident weights
  const uint32_t a_base = smem_base + w_bytes;                    // A halo ring (w_bytes is a multiple of 1024)
  const uint32_t stg_off = w_bytes + g.stages * g.a_stage_bytes;  // two epilogue staging blocks
  const uint32_t bar_base = smem_base + stg_off + 2 * STG_BYTES;
  auto a_stage = [&](int s) { return a_base + s * g.a_stage_bytes; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (MAX_STAGES + s); };
  const uint32_t w_bar = bar_base + 8u * 2 * MAX_STAGES;

  const int wg = threadIdx.x / WG_THREADS;
  const int ntw = (p.OW + 127) / 128;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmA);
    prefetch_tensormap(&tmW);
    for (int s = 0; s < g.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);              // one arrival per consumer warp
    }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x != 0) return;
    // park the whole weight slab: [tap][kchunk] tiles of Nr x 128 B
    mbar_expect_tx(w_bar, (uint32_t)w_bytes);
    for (int j = 0; j < p.ntaps; ++j)
      for (int kc = 0; kc < kchunks; ++kc)
        tma_load_3d(w_base + (uint32_t)((j * kchunks + kc) * g.b_tile_bytes), &tmW, w_bar, kc * KE, 0, j);
    const uint32_t a_tx = (uint32_t)(g.KH * g.BWh * 128);
    int s = 0;
    uint32_t ph = 0;
    TileWalk tk;
    for (tk.init(blockIdx.x, gridDim.x, g.total_tiles, ntw, p.OH); tk.left > 0; tk.next(ntw, p.OH)) {
      for (int kc = 0; kc < kchunks; ++kc) {
        mbar_wait(empty_bar(s), ph ^ 1u);
        mbar_expect_tx(full_bar(s), a_tx);
        tma_load_5d(a_stage(s), &tmA, full_bar(s), kc * KE, tk.tw * 128 - g.pad_w, tk.h - g.pad_h, tk.b, 0);
        if (++s == g.stages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 1, 2) =====================
  setmaxnreg_inc<232>();
  const int gi = wg - 1;
  const int t = threadIdx.x & (WG_THREADS - 1);
  float* stg = reinterpret_cast<float*>(smem_gen + stg_off + gi * STG_BYTES);
  // descriptors differ only in their 14-bit start-address field: walk it with adds
  const uint64_t b_step = (uint64_t)((kchunks * g.b_tile_bytes) >> 4);
  const uint64_t a_kw_step = (uint64_t)(g.dil_w * 8), a_kh_step = (uint64_t)(g.BWh * 8);   // rows x 128 B >> 4
  float acc[NR / 2];
#pragma unroll
  for (int i = 0; i < NR / 2; ++i) acc[i] = 0.f;
  mbar_wait(w_bar, 0);
  int s = 0;
  uint32_t ph = 0;
  TileWalk tk;
  for (tk.init(blockIdx.x, gridDim.x, g.total_tiles, ntw, p.OH); tk.left > 0; tk.next(ntw, p.OH)) {
    int prev = -1;
    for (int kc = 0; kc < kchunks; ++kc) {
      mbar_wait(full_bar(s), ph);
      // short last k-chunk (Kc = 48 -> 32 + 16): only the 32-byte K steps that hold data
      const int nk = (kc == kchunks - 1) ? (((p.Kc - kc * KE) * ES + 31) >> 5) : 4;
      uint64_t adesc_row = make_desc(a_stage(s) + gi * WG_ROWS * 128);
      uint64_t bdesc = make_desc(w_base + (uint32_t)(kc * g.b_tile_bytes));
      uint32_t accum = kc > 0 ? 1u : 0u;
      fence_operands(acc);
      wgmma_fence();
      for (int kh = 0; kh < g.KH; ++kh, adesc_row += a_kh_step) {
        uint64_t adesc = adesc_row;
        for (int kw = 0; kw < g.KW; ++kw, adesc += a_kw_step, bdesc += b_step) {
          if (nk == 4) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              wgmma<F16, NR>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accum);
              accum = 1u;
            }
          } else {
            for (int k = 0; k < nk; ++k) {
              wgmma<F16, NR>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accum);
              accum = 1u;
            }
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                          // the previous chunk's wgmma have retired: its stage can be refilled
      fence_operands(acc);
      if (prev >= 0) {
        __syncwarp();
        if ((t & 31) == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
      if (++s == g.stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_operands(acc);
    __syncwarp();
    if ((t & 31) == 0) mbar_arrive(empty_bar(prev));
    const TgRow r = tg_row(p, tk.b, tk.h, tk.tw * 128 + gi * WG_ROWS + (t & (WG_ROWS - 1)));
    wg_epilogue<NR>(p, r, 0, acc, stg, 1 + gi);
  }
}

// Does the descriptor describe a dense stride-1 convolution over a regular tap grid, small enough for the weights to
// stay in shared memory?  Fills the geometry when it does.
bool ws_geometry(const TgParams& p, WsGeom& g) {
  if (!tapgemm_tc_supported(p)) return false;
  if (p.N > 64 || p.BW != 128 || p.BH != 1 || p.OW < 128 || p.w_batch_step != 0 || p.ntaps < 2) return false;
  // recover (KH, KW, dilation, padding) from the tap table
  int KW = 1;
  while (KW < p.ntaps && p.taps[KW].dh == p.taps[0].dh) ++KW;
  if (p.ntaps % KW) return false;
  const int KH = p.ntaps / KW;
  const int dil_w = KW > 1 ? p.taps[1].dw - p.taps[0].dw : 1;
  const int dil_h = KH > 1 ? p.taps[KW].dh - p.taps[0].dh : 1;
  if (dil_w < 1 || dil_h != 1) return false;          // rows of the halo box are consecutive image rows
  for (int j = 0; j < p.ntaps; ++j) {
    const b200vc_tap& t = p.taps[j];
    const int kh = j / KW, kw = j % KW;
    if (t.c_off != 0 || t.dp != 0 || t.widx != j) return false;
    if (t.dw != p.taps[0].dw + kw * dil_w || t.dh != p.taps[0].dh + kh * dil_h) return false;
  }
  g.KH = KH; g.KW = KW; g.dil_w = dil_w; g.dil_h = dil_h;
  g.pad_w = -p.taps[0].dw; g.pad_h = -p.taps[0].dh;
  g.BWh = 128 + (KW - 1) * dil_w;
  if (g.BWh > 256 || KH > 256) return false;
  g.Nr = (p.N + 15) & ~15;                 // wgmma N and weight-tile rows (16 rows x 128 B = 2 KB granules: stays 1024-aligned)
  if (g.Nr < 32) g.Nr = 32;
  g.b_tile_bytes = g.Nr * 128;
  g.a_stage_bytes = ((KH * g.BWh * 128 + 1023) / 1024) * 1024;   // 1024-aligned stages (swizzle atom = 8 rows x 128 B)
  const int ke = (p.dtype & TG_DT_AB) ? 2 * KCHUNK : KCHUNK;
  const int kchunks = (p.Kc + ke - 1) / ke;
  const int w_bytes = p.ntaps * kchunks * g.b_tile_bytes;
  const int fixed = 2 * STG_BYTES + 8 * (2 * MAX_STAGES + 1) + 1024;
  int stages = (SMEM_LIMIT - fixed - w_bytes) / g.a_stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  if (stages < 2) return false;
  g.stages = stages;
  const long long tiles = (long long)((p.OW + 127) / 128) * p.OH * p.OB;
  if (tiles <= 0 || tiles >= (1ll << 31)) return false;
  g.total_tiles = (int)tiles;
  return true;
}

template <int NR, bool F16>
int ws_launch_cfg(const CUtensorMap& tmA, const CUtensorMap& tmW, const TgParams& p, const WsGeom& g, int grid, int smem,
                  cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    B200VC_CHECK_CUDA(cudaFuncSetAttribute(tapgemm_ws_kernel<NR, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    configured = true;
  }
  tapgemm_ws_kernel<NR, F16><<<grid, NUM_THREADS, smem, stream>>>(tmA, tmW, p, g);
  return kOk;
}

template <bool F16>
int ws_dispatch_nr(const CUtensorMap& tmA, const CUtensorMap& tmW, const TgParams& p, const WsGeom& g, int grid, int smem,
                   cudaStream_t stream) {
  switch (g.Nr) {
    case 32: return ws_launch_cfg<32, F16>(tmA, tmW, p, g, grid, smem, stream);
    case 48: return ws_launch_cfg<48, F16>(tmA, tmW, p, g, grid, smem, stream);
    default: return ws_launch_cfg<64, F16>(tmA, tmW, p, g, grid, smem, stream);
  }
}

}  // namespace

bool tapgemm_ws_applicable(const TgParams& p) {
  WsGeom g;
  return ws_geometry(p, g);
}

int tapgemm_ws_launch(const TgParams& p, cudaStream_t stream) {
  WsGeom g;
  B200VC_REQUIRE(ws_geometry(p, g), "tapgemm_ws: descriptor is not a small-channel regular convolution");
  const bool f16 = (p.dtype & TG_DT_AB) != 0;
  const int ke = f16 ? 2 * KCHUNK : KCHUNK;
  const int kchunks = (p.Kc + ke - 1) / ke;
  CUtensorMap tmA, tmW;
  const cuuint32_t abox[5] = {(cuuint32_t)ke, (cuuint32_t)g.BWh, (cuuint32_t)g.KH, 1, 1};
  int rc = encode_a_map(&tmA, p, abox);
  if (rc) return rc;
  rc = encode_w_map(&tmW, p, p.ntaps, p.wstride, ke, g.Nr);
  if (rc) return rc;
  const int w_bytes = p.ntaps * kchunks * g.b_tile_bytes;
  const int smem = w_bytes + g.stages * g.a_stage_bytes + 2 * STG_BYTES + 8 * (2 * MAX_STAGES + 1) + 1024;
  const int grid = g.total_tiles < num_sms() ? g.total_tiles : num_sms();
  rc = f16 ? ws_dispatch_nr<true>(tmA, tmW, p, g, grid, smem, stream) : ws_dispatch_nr<false>(tmA, tmW, p, g, grid, smem, stream);
  if (rc) return rc;
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

}  // namespace b200vc
