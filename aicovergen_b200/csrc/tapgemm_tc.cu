// wgmma / TMA tap-GEMM for sm_90a (TF32 or fp16 operands, fp32 accumulate).
//
// One CTA = three warpgroups:
//   warpgroup 0    : TMA producer (one thread): per tap and 128-byte K chunk a 5-D box of A (the tile's pixels) and a
//                    3-D box of W into a ring of shared-memory stages, mbarrier complete_tx
//   warpgroups 1-2 : consumers: each issues m64 x BN wgmma for its 64 rows of every 128-row block of the tile straight from
//                    the ring (descriptors, no register staging of operands), releases a stage once the wgmma that read it
//                    has retired, then runs the fused epilogue (tapgemm.cuh) on its accumulator registers
//
// A pixels x 32 fp32 (64 fp16) channels land in shared memory as rows of 128 B with the hardware 128-byte swizzle, which is
// the canonical K-major SWIZZLE_128B wgmma operand layout: conv zero padding comes for free from TMA's out-of-bounds zero
// fill, so no im2col buffer ever exists in HBM.
//
// The same kernel serves both launch forms: one tile per CTA (tapgemm_tc_launch) and persistent, one CTA per SM walking
// the tiles with the n-tile fastest so neighbouring CTAs share the A box in L2 (tapgemm_tc2_launch).
#include "hopper.cuh"
#include <cstdlib>

namespace b200vc {

using namespace hop;

namespace {

constexpr int NUM_THREADS = 3 * WG_THREADS;

// MH = 128-row blocks per tile: with MH == 2 one W tile feeds the MMAs of 256 rows.
template <int BN, int STAGES, int MH, bool F16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapgemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                  const __grid_constant__ TgParams p, int ntiles_n, int total_tiles, int tbw, int tbh) {
  constexpr int KE = F16 ? 2 * KCHUNK : KCHUNK;                    // K elements per 128-byte chunk row
  constexpr int ES = F16 ? 2 : 4;
  constexpr int A_STAGE_BYTES = MH * TG_TILE_M * 128;
  constexpr int B_STAGE_BYTES = BN * 128;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES + 2 * STG_BYTES;
  auto a_stage = [&](int s) { return smem_base + s * STAGE_BYTES; };
  auto b_stage = [&](int s) { return smem_base + s * STAGE_BYTES + A_STAGE_BYTES; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int wg = threadIdx.x / WG_THREADS;
  const int ntw = (p.OW + tbw - 1) / tbw;
  const int nth = (p.OH + tbh - 1) / tbh;
  const int kchunks = (p.Kc + KE - 1) / KE;
  const int nchunks = p.ntaps * kchunks;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmA);
    prefetch_tensormap(&tmW);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);              // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  auto tile_coords = [&](int tile, int& w0, int& h0, int& tb, int& n0) {
    const int nt = tile % ntiles_n;
    int mt = tile / ntiles_n;
    const int tw = mt % ntw; mt /= ntw;
    const int th = mt % nth; mt /= nth;
    tb = mt;
    w0 = tw * tbw;
    h0 = th * tbh;
    n0 = nt * BN;
  };

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();                      // registers go to the consumers' accumulators
    if (threadIdx.x != 0) return;
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int w0, h0, tb, n0;
      tile_coords(tile, w0, h0, tb, n0);
      const int wsel = tb * p.w_batch_step;
      for (int tap_i = 0; tap_i < p.ntaps; ++tap_i) {
        const TgTap tap = p.taps[tap_i];
        const int cw = w0 + tap.dw, ch = h0 + tap.dh, cp = tap.dp, widx = tap.widx + wsel;
        int ca = tap.c_off;
        for (int kc0 = 0; kc0 < p.Kc; kc0 += KE, ca += KE) {
          mbar_wait(empty_bar(s), ph ^ 1u);
          mbar_expect_tx(full_bar(s), STAGE_BYTES);
          tma_load_5d(a_stage(s), &tmA, full_bar(s), ca, cw, ch, tb, cp);
          tma_load_3d(b_stage(s), &tmW, full_bar(s), kc0, n0, widx);
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 1, 2) =====================
  setmaxnreg_inc<232>();
  const int g = wg - 1;
  const int t = threadIdx.x & (WG_THREADS - 1);
  float* stg = reinterpret_cast<float*>(smem_gen + STAGES * STAGE_BYTES + g * STG_BYTES);
  // the last k-chunk of a tap may be short (Kc = 48 -> 32 + 16): issue only the 32-byte K steps that hold data
  const int klast = ((p.Kc - (kchunks - 1) * KE) * ES + 31) >> 5;
  float acc[MH][BN / 2];
#pragma unroll
  for (int mh = 0; mh < MH; ++mh)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[mh][i] = 0.f;
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int w0, h0, tb, n0;
    tile_coords(tile, w0, h0, tb, n0);
    int prev = -1;
    for (int chunk = 0, kc = 0; chunk < nchunks; ++chunk) {
      mbar_wait(full_bar(s), ph);
      const int nk = (kc == kchunks - 1) ? klast : 4;
      const uint64_t adesc = make_desc(a_stage(s) + g * WG_ROWS * 128);
      const uint64_t bdesc = make_desc(b_stage(s));
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) fence_operands(acc[mh]);
      wgmma_fence();
      if (nk == 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int mh = 0; mh < MH; ++mh)      // 128 rows x 128 B = 16 KB further into the A box: +1024 in the (addr >> 4) field
            wgmma<F16, BN>(acc[mh], adesc + (uint64_t)(mh * 1024 + 2 * k), bdesc + (uint64_t)(2 * k), (chunk | k) != 0);
      } else {
        for (int k = 0; k < nk; ++k)
#pragma unroll
          for (int mh = 0; mh < MH; ++mh)
            wgmma<F16, BN>(acc[mh], adesc + (uint64_t)(mh * 1024 + 2 * k), bdesc + (uint64_t)(2 * k), (chunk | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<1>();                          // the previous chunk's wgmma have retired: its stage can be refilled
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) fence_operands(acc[mh]);
      if (prev >= 0) {
        __syncwarp();
        if ((t & 31) == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1u; }
      if (++kc == kchunks) kc = 0;
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mh = 0; mh < MH; ++mh) fence_operands(acc[mh]);
    __syncwarp();
    if ((t & 31) == 0) mbar_arrive(empty_bar(prev));
#pragma unroll
    for (int mh = 0; mh < MH; ++mh) {
      const int m = mh * TG_TILE_M + g * WG_ROWS + (t & (WG_ROWS - 1));   // row inside the (tbw x tbh) box, w fastest
      const TgRow r = tg_row(p, tb, h0 + m / tbw, w0 + m % tbw);
      wg_epilogue<BN>(p, r, n0, acc[mh], stg, 1 + g);
    }
  }
}

// ---------------------------------------------------------------------------
// Host side: tensor-map encoding through the driver entry point (no -lcuda).
// ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

int encode_map(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims,
               const cuuint64_t* strides_bytes, const cuuint32_t* box, bool half = false) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable");
    return kErrDriver;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(tm, half ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base),
                  dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error(
        "cuTensorMapEncodeTiled failed (%d): rank %d base %p dims [%llu %llu %llu %llu %llu] "
        "strides [%llu %llu %llu %llu] box [%u %u %u %u %u]",
        (int)r, rank, base, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
        (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
        (unsigned long long)(rank > 4 ? dims[4] : 0), (unsigned long long)strides_bytes[0],
        (unsigned long long)(rank > 2 ? strides_bytes[1] : 0),
        (unsigned long long)(rank > 3 ? strides_bytes[2] : 0),
        (unsigned long long)(rank > 4 ? strides_bytes[3] : 0), box[0], rank > 1 ? box[1] : 0,
        rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
    return kErrDriver;
  }
  return kOk;
}

constexpr int SMEM_LIMIT = 227 * 1024;

template <int BN, int STAGES, int MH, bool F16>
int launch_cfg(const CUtensorMap& tmA, const CUtensorMap& tmW, const TgParams& p, int ntiles_n, int total_tiles,
               int grid, int tbw, int tbh, cudaStream_t stream) {
  constexpr int smem = STAGES * (MH * TG_TILE_M * 128 + BN * 128) + 2 * STG_BYTES + 8 * 2 * STAGES + 1024;
  static_assert(smem <= SMEM_LIMIT, "shared memory budget");
  static bool configured = false;
  if (!configured) {
    B200VC_CHECK_CUDA(cudaFuncSetAttribute(tapgemm_wg_kernel<BN, STAGES, MH, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  tapgemm_wg_kernel<BN, STAGES, MH, F16><<<grid, NUM_THREADS, smem, stream>>>(tmA, tmW, p, ntiles_n, total_tiles, tbw, tbh);
  return kOk;
}

template <int MH, bool F16>
int launch_bn(int BN, const CUtensorMap& tmA, const CUtensorMap& tmW, const TgParams& p, int ntiles_n, int total, int grid,
              int tbw, int tbh, cudaStream_t stream) {
  // ring depth: as many stages as fit beside the two 9 KB epilogue staging blocks (~192 KB of operands)
  if constexpr (MH == 1) {
    switch (BN) {
      case 256: return launch_cfg<256, 4, 1, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
      case 128: return launch_cfg<128, 6, 1, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
      case 64:  return launch_cfg<64, 8, 1, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
      default:  return launch_cfg<32, 8, 1, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
    }
  } else {
    switch (BN) {       // 256-row tiles: two m64 accumulators per consumer thread, so at most 128 columns
      case 128: return launch_cfg<128, 4, 2, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
      case 64:  return launch_cfg<64, 5, 2, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
      default:  return launch_cfg<32, 5, 2, F16>(tmA, tmW, p, ntiles_n, total, grid, tbw, tbh, stream);
    }
  }
}

int g_rows256 = [] { const char* e = getenv("B200VC_TC2_ROWS256"); return (e && e[0] == '1') ? 1 : 0; }();

int tc_launch(const TgParams& p, cudaStream_t stream, bool persistent) {
  B200VC_REQUIRE(tapgemm_tc_supported(p), "tapgemm_tc: operand alignment not TMA-compatible");
  const bool f16 = (p.dtype & TG_DT_AB) != 0;
  const int BN = p.N > 128 ? 256 : (p.N > 64 ? 128 : (p.N > 32 ? 64 : 32));
  const int ntiles_n = ceil_div(p.N, BN);
  // 256-row tiles (one W tile feeds the MMAs of two 128-row blocks) halve the W traffic per FLOP; experimental, off by
  // default (b200vc_tapgemm_set_rows256, initial value from env B200VC_TC2_ROWS256), persistent launches only
  int tbw = p.BW, tbh = p.BH, MH = 1;
  if (persistent && g_rows256 && !f16 && BN <= 128) {
    const int bw2 = p.BH == 1 ? 2 * p.BW : p.BW, bh2 = p.BH == 1 ? 1 : 2 * p.BH;
    if (bw2 <= 256 && bh2 <= 256) {
      const long long t1 = (long long)ceil_div(p.OW, p.BW) * ceil_div(p.OH, p.BH) * p.OB;
      const long long t2 = (long long)ceil_div(p.OW, bw2) * ceil_div(p.OH, bh2) * p.OB;
      if (t2 * ntiles_n >= num_sms() && 2 * t2 * 100 <= t1 * 105) { tbw = bw2; tbh = bh2; MH = 2; }
    }
  }
  const long long total = (long long)ceil_div(p.OW, tbw) * ceil_div(p.OH, tbh) * p.OB * ntiles_n;
  B200VC_REQUIRE(total > 0 && total < (1ll << 31), "tapgemm_tc: bad tile count %lld", total);

  const cuuint32_t ke = f16 ? 2 * KCHUNK : KCHUNK;
  CUtensorMap tmA, tmW;
  const cuuint32_t abox[5] = {ke, (cuuint32_t)tbw, (cuuint32_t)tbh, 1, 1};
  int rc = encode_a_map(&tmA, p, abox);
  if (rc) return rc;
  int max_widx = 0;
  for (int i = 0; i < p.ntaps; ++i) max_widx = p.taps[i].widx > max_widx ? p.taps[i].widx : max_widx;
  rc = encode_w_map(&tmW, p, max_widx + 1 + (p.OB - 1) * p.w_batch_step, p.wstride, (int)ke, BN);
  if (rc) return rc;
  const int grid = (int)(persistent && total > num_sms() ? num_sms() : total);
  if (MH == 2) rc = launch_bn<2, false>(BN, tmA, tmW, p, ntiles_n, (int)total, grid, tbw, tbh, stream);
  else if (f16) rc = launch_bn<1, true>(BN, tmA, tmW, p, ntiles_n, (int)total, grid, tbw, tbh, stream);
  else rc = launch_bn<1, false>(BN, tmA, tmW, p, ntiles_n, (int)total, grid, tbw, tbh, stream);
  if (rc) return rc;
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

}  // namespace

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

int encode_map_f32(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims,
                   const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  return encode_map(tm, base, rank, dims, strides_bytes, box);
}
int encode_map_f16(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims,
                   const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  return encode_map(tm, base, rank, dims, strides_bytes, box, true);
}

namespace hop {

int encode_a_map(CUtensorMap* tm, const TgParams& p, const cuuint32_t (&box)[5]) {
  const bool f16 = (p.dtype & TG_DT_AB) != 0;
  const unsigned long long es = f16 ? 2ull : 4ull;
  const int epb = f16 ? 8 : 4;                           // elements per 16 bytes (TMA stride granule)
  cuuint64_t dims[5], strides[4];
  long long span = 1;                                    // safe stride for size-1 dims
  for (int i = 0; i < 5; ++i) {
    dims[i] = (cuuint64_t)(p.a_dim[i] > 0 ? p.a_dim[i] : 1);
    if (i > 0) {
      long long st = p.a_stride[i];
      if (p.a_dim[i] <= 1) st = ((span + epb - 1) / epb) * epb;
      strides[i - 1] = (cuuint64_t)st * es;
      span = st * (long long)dims[i];
    } else {
      span = (long long)dims[0];
    }
  }
  return encode_map(tm, p.A, 5, dims, strides, box, f16);
}

int encode_w_map(CUtensorMap* tm, const TgParams& p, int nw, long long wstride, int box_k, int box_n) {
  const bool f16 = (p.dtype & TG_DT_AB) != 0;
  const unsigned long long es = f16 ? 2ull : 4ull;
  const int epb = f16 ? 8 : 4;
  cuuint64_t dims[3] = {(cuuint64_t)p.Kc, (cuuint64_t)p.N, (cuuint64_t)nw};
  if (nw <= 1) wstride = ((p.ldw * p.N + epb - 1) / epb) * epb;
  cuuint64_t strides[2] = {(cuuint64_t)p.ldw * es, (cuuint64_t)wstride * es};
  cuuint32_t box[3] = {(cuuint32_t)box_k, (cuuint32_t)box_n, 1};
  return encode_map(tm, p.Wt, 3, dims, strides, box, f16);
}

}  // namespace hop

// Whether a problem can go through the TMA/wgmma path (alignment rules of
// cuTensorMapEncodeTiled); otherwise callers use the SIMT kernel.
bool tapgemm_tc_supported(const TgParams& p) {
  const int epb = (p.dtype & TG_DT_AB) ? 8 : 4;            // elements per 16 bytes
  if ((reinterpret_cast<uintptr_t>(p.A) & 15) || (reinterpret_cast<uintptr_t>(p.Wt) & 15)) return false;
  for (int i = 1; i < 5; ++i)
    if (p.a_dim[i] > 1 && (p.a_stride[i] % epb != 0)) return false;
  if (p.a_stride[0] != 1) return false;
  if (p.ldw % epb != 0 || (p.wstride % epb != 0)) return false;
  if (p.BW > 256 || p.BH > 256 || p.BW * p.BH != TG_TILE_M) return false;
  return true;
}

int tapgemm_tc_launch(const TgParams& p, cudaStream_t stream) {
  B200VC_REQUIRE(!(p.dtype & TG_DT_AB), "tapgemm_tc: fp16 operands are handled by the persistent / weight-stationary kernels");
  return tc_launch(p, stream, false);
}

int tapgemm_tc2_launch(const TgParams& p, cudaStream_t stream) { return tc_launch(p, stream, true); }

void tapgemm_tc2_set_rows256(int on) { g_rows256 = on ? 1 : 0; }

}  // namespace b200vc
