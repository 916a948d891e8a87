// RMVPE-specific kernels: STFT framing helpers, 2x2 average pooling (NHWC), the
// bidirectional GRU recurrence as a thread-block-cluster kernel with DSMEM state
// exchange, and the salience -> cents -> Hz decode in the reference's exact numpy order.
#include "common.cuh"
#include "../../include/b200vc.h"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200vc {
namespace {

inline unsigned blocks_for(long long n, int bs) { return (unsigned)((n + bs - 1) / bs); }

// out[i] = in[reflect(i - pad)], i in [0, N + 2*pad)   (torch.stft center=True, pad_mode="reflect")
__global__ void reflect_pad_1d_kernel(const float* __restrict__ in, float* __restrict__ out, long long N,
                                      long long pad, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long j = i - pad;
  if (j < 0) j = -j;
  if (j >= N) j = 2 * (N - 1) - j;
  out[i] = (j >= 0 && j < N) ? in[j] : 0.f;
}

// mag[t,k] = sqrt(re^2 + im^2), spec rows hold [re(0..nb-1) | im(0..nb-1)], mag row pitch ldm (zero-padded tail)
__global__ void magnitude_kernel(const float* __restrict__ spec, float* __restrict__ mag, long long rows,
                                 int nb, long long lds, long long ldm) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows * ldm) return;
  const long long t = e / ldm;
  const int k = (int)(e % ldm);
  float v = 0.f;
  if (k < nb) {
    const float re = spec[t * lds + k], im = spec[t * lds + nb + k];
    v = sqrtf(re * re + im * im);
  }
  mag[e] = v;
}

// y = a * log(max(x, clamp)) + b on the first `rows` rows, then reflect-pad rows up to rows_total
// (rmvpe.py:324 log-mel; unet.encoder.bn as a scalar affine; F.pad(mode="reflect") at rmvpe.py:353-355)
__global__ void logmel_affine_reflect_kernel(const float* __restrict__ x, float* __restrict__ out,
                                             int rows, int rows_total, int C, float clampv, float a, float b) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)rows_total * C) return;
  int t = (int)(e / C);
  const int c = (int)(e % C);
  if (t >= rows) t = 2 * (rows - 1) - t;
  const float v = x[(long long)t * C + c];
  out[e] = a * (clampv < 0.f ? v : logf(fmaxf(v, clampv))) + b;     // clampv < 0: x already holds log-mel (RMVPE.mel2hidden)
}

// NHWC 2x2 average pool, input may be a channel slice (pixel pitch ldi)
__global__ void avgpool2x2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W,
                                  int C, long long ldi) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int Ho = H / 2, Wo = W / 2;
  if (e >= (long long)B * Ho * Wo * C) return;
  const int c = (int)(e % C);
  long long r = e / C;
  const int wo = (int)(r % Wo); r /= Wo;
  const int ho = (int)(r % Ho);
  const int b = (int)(r / Ho);
  const float* p = in + (((long long)b * H + 2 * ho) * W + 2 * wo) * ldi + c;
  out[e] = 0.25f * (p[0] + p[ldi] + p[(long long)W * ldi] + p[(long long)W * ldi + ldi]);
}

// the same on 3xTF32 split tensors: x = hi + lo per input pixel, pooled in fp32, written back as hi | lo | hi planes
__global__ void avgpool2x2_split_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C,
                                        long long ldi, long long in_split, long long ldo, long long out_split) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int Ho = H / 2, Wo = W / 2;
  if (e >= (long long)B * Ho * Wo * C) return;
  const int c = (int)(e % C);
  long long r = e / C;
  const int wo = (int)(r % Wo); r /= Wo;
  const int ho = (int)(r % Ho);
  const int b = (int)(r / Ho);
  const float* p = in + (((long long)b * H + 2 * ho) * W + 2 * wo) * ldi + c;
  const long long dn = (long long)W * ldi;
  const float x00 = p[0] + p[in_split], x01 = p[ldi] + p[ldi + in_split];
  const float x10 = p[dn] + p[dn + in_split], x11 = p[dn + ldi] + p[dn + ldi + in_split];
  const float v = 0.25f * (x00 + x01 + x10 + x11);
  const float hi = round_tf32(v);
  float* o = out + (((long long)b * Ho + ho) * Wo + wo) * ldo + c;
  o[0] = hi; o[out_split] = round_tf32(v - hi); o[2 * out_split] = hi;
}

// ---------------------------------------------------------------------------
// BiGRU recurrence (rmvpe.py:8-20; torch.nn.GRU gate order r,z,n).
// grid = 2 clusters x CL CTAs; cluster d handles direction d.  CTA `rank` owns hidden units
// [rank*UPC, (rank+1)*UPC): its 3*UPC rows of W_hh stay in REGISTERS for the whole sequence
// (2 threads per row, 128 weights each); h_{t-1} (256 floats) is replicated in every CTA's
// shared memory and the freshly computed slice is pushed to all peers through DSMEM, double
// buffered so one cluster barrier per step suffices.
//   xp   [T, 2*3H]  : x W_ih^T + b_ih for both directions (dir d at column d*3H), precomputed by a GEMM
//   out  [T, 2*H]   : h_t, forward at columns [0,H), backward at [H,2H)
// ---------------------------------------------------------------------------
constexpr int GRU_H = 256;
constexpr int GRU_CL = 8;
constexpr int GRU_UPC = GRU_H / GRU_CL;      // 32 units per CTA
constexpr int GRU_ROWS = 3 * GRU_UPC;        // 96 W_hh rows per CTA
constexpr int GRU_THREADS = 2 * GRU_ROWS;    // 192

__global__ void __cluster_dims__(GRU_CL, 1, 1) __launch_bounds__(GRU_THREADS, 1)
bigru_kernel(const float* __restrict__ xp, const float* __restrict__ whh /*[2][3H][H]*/,
             const float* __restrict__ bhh /*[2][3H]*/, float* __restrict__ out, int T) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.x / GRU_CL;
  const int tid = threadIdx.x;
  const int row = tid >> 1;            // 0..95 : gate g = row / UPC, unit j = row % UPC
  const int half = tid & 1;            // which 128-wide half of the dot product
  const int g = row / GRU_UPC, j = row % GRU_UPC;
  const int unit = rank * GRU_UPC + j;
  const int wrow = g * GRU_H + unit;

  __shared__ __align__(16) float hbuf[2][GRU_H];
  __shared__ float gate[GRU_ROWS];

  // this thread's 128 recurrent weights
  float w[GRU_H / 2];
  {
    const float* src = whh + ((long long)dir * 3 * GRU_H + wrow) * GRU_H + half * (GRU_H / 2);
#pragma unroll
    for (int k = 0; k < GRU_H / 2; k += 4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(src + k));
      w[k] = v.x; w[k + 1] = v.y; w[k + 2] = v.z; w[k + 3] = v.w;
    }
  }
  const float bh = bhh[dir * 3 * GRU_H + wrow];
  for (int i = tid; i < 2 * GRU_H; i += GRU_THREADS) (&hbuf[0][0])[i] = 0.f;
  cluster.sync();

  const long long xp_ld = 2 * 3 * GRU_H;
  const float* xp_d = xp + dir * 3 * GRU_H;
  // prefetch x-projection for the first step
  int t = dir == 0 ? 0 : T - 1;
  float xv = (half == 0) ? __ldg(xp_d + (long long)t * xp_ld + wrow) : 0.f;
  // x-projection of the n gate for the unit this thread finalises (threads 0..UPC-1), also fetched one step ahead:
  // loaded inside the step it sat on the critical path of every one of the T sequential steps
  float xn = (tid < GRU_UPC) ? __ldg(xp_d + (long long)t * xp_ld + 2 * GRU_H + rank * GRU_UPC + tid) : 0.f;

  for (int s = 0; s < T; ++s) {
    const int cur = s & 1, nxt = cur ^ 1;
    t = dir == 0 ? s : T - 1 - s;
    const int tn = dir == 0 ? s + 1 : T - 2 - s;
    float xv_next = 0.f;
    if (half == 0 && s + 1 < T) xv_next = __ldg(xp_d + (long long)tn * xp_ld + wrow);
    float xn_next = 0.f;
    if (tid < GRU_UPC && s + 1 < T) xn_next = __ldg(xp_d + (long long)tn * xp_ld + 2 * GRU_H + rank * GRU_UPC + tid);

    // partial dot product W_hh[row, half*128 : +128] . h[half*128 : +128]
    const float* h = &hbuf[cur][half * (GRU_H / 2)];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int k = 0; k < GRU_H / 2; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h + k);
      a0 = fmaf(w[k], hv.x, a0);
      a1 = fmaf(w[k + 1], hv.y, a1);
      a2 = fmaf(w[k + 2], hv.z, a2);
      a3 = fmaf(w[k + 3], hv.w, a3);
    }
    float acc = (a0 + a1) + (a2 + a3);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (half == 0) {
      const float hp = acc + bh;                    // W_h* h + b_h*
      // r,z: sigma(x + hp) ; n: needs r first -> stash (x, hp) separately for the n gate
      if (g < 2) gate[row] = 1.f / (1.f + expf(-(xv + hp)));
      else       gate[row] = hp;                    // combined below with r
    }
    __syncthreads();
    if (tid < GRU_UPC) {
      // thread tid finalises unit rank*UPC + tid
      const int u = rank * GRU_UPC + tid;
      const float r = gate[tid], z = gate[GRU_UPC + tid], hpn = gate[2 * GRU_UPC + tid];
      const float n = tanhf(xn + r * hpn);
      const float hprev = hbuf[cur][u];
      const float hnew = (1.f - z) * n + z * hprev;
      out[(long long)t * (2 * GRU_H) + dir * GRU_H + u] = hnew;
#pragma unroll
      for (int dst = 0; dst < GRU_CL; ++dst) {
        float* peer = cluster.map_shared_rank(&hbuf[0][0], dst);
        peer[nxt * GRU_H + u] = hnew;
      }
    }
    xv = xv_next;
    xn = xn_next;
    cluster.sync();   // publishes hbuf[nxt] cluster-wide; also orders gate[] reuse
  }
}

// ---------------------------------------------------------------------------
// BiGRU v2: same decomposition (2 clusters x 8 CTAs, W_hh in registers) but the per-step exchange is one DSMEM hop:
//   * 512 threads = 16 warps x 2 units x (3 gates x 4 K-quarters): the twelve lanes of a unit sit in one warp, so the
//     gate pre-activations are combined with shuffles (no block barrier, no shared-memory gate buffer);
//   * the unit's leader lane pushes h_new to every CTA of the cluster with st.async ... mbarrier::complete_tx, i.e. the
//     data and its arrival signal travel together; each CTA waits on its OWN mbarrier for the 1024 bytes of the new h
//     (armed one step ahead) instead of a cluster-wide barrier.  Double-buffered h: a CTA can only start step s+1 after
//     every peer has SENT its step-s slice, which each peer does after its last read of the step-s input buffer.
// One st.async per (unit, peer) means 256 remote mbarrier updates per CTA and step, which can cost more than v1's one
// cluster barrier per step.  Not the default; v3 sends one 128-byte cp.async.bulk per peer instead.
// ---------------------------------------------------------------------------
constexpr int GRU2_THREADS = 512;

__device__ __forceinline__ uint32_t gru_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__global__ void __cluster_dims__(GRU_CL, 1, 1) __launch_bounds__(GRU2_THREADS, 1)
bigru_v2_kernel(const float* __restrict__ xp, const float* __restrict__ whh /*[2][3H][H]*/,
                const float* __restrict__ bhh /*[2][3H]*/, float* __restrict__ out, int T) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.x / GRU_CL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool active = lane < 24;
  const int ul = lane / 12;                         // unit within the warp (0/1); lanes 24..31 idle
  const int li = lane - ul * 12;                    // 0..11
  const int g = li >> 2, q = li & 3;                // gate (r,z,n), K quarter
  const int j = warp * 2 + (active ? ul : 0);       // unit inside this CTA, 0..31
  const int unit = rank * GRU_UPC + j;
  const int wrow = g * GRU_H + unit;
  const bool leader = active && li == 0;

  __shared__ __align__(16) float hbuf[2][GRU_H];
  __shared__ __align__(8) unsigned long long mbar[2];

  float w[GRU_H / 4];
  float bh = 0.f;
  if (active) {
    const float* src = whh + ((long long)dir * 3 * GRU_H + wrow) * GRU_H + q * (GRU_H / 4);
#pragma unroll
    for (int k = 0; k < GRU_H / 4; k += 4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(src + k));
      w[k] = v.x; w[k + 1] = v.y; w[k + 2] = v.z; w[k + 3] = v.w;
    }
    bh = bhh[dir * 3 * GRU_H + wrow];
  } else {
#pragma unroll
    for (int k = 0; k < GRU_H / 4; ++k) w[k] = 0.f;
  }
  for (int i = threadIdx.x; i < 2 * GRU_H; i += GRU2_THREADS) (&hbuf[0][0])[i] = 0.f;
  const uint32_t mb0 = gru_smem_u32(&mbar[0]), mb1 = gru_smem_u32(&mbar[1]);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb0));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster.sync();

  // remote addresses of every CTA's h buffers / barriers (leader lanes only)
  uint32_t peer_h[GRU_CL], peer_mb[GRU_CL];
#pragma unroll
  for (int d = 0; d < GRU_CL; ++d) {
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_h[d]) : "r"(gru_smem_u32(&hbuf[0][0])), "r"(d));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_mb[d]) : "r"(mb0), "r"(d));
  }

  const long long xp_ld = 2 * 3 * GRU_H;
  const float* xp_d = xp + dir * 3 * GRU_H;
  int t = dir == 0 ? 0 : T - 1;
  // x-projections of this thread's gate row, one step ahead (only the q == 0 lane of each gate uses it)
  float xv = (active && q == 0) ? __ldg(xp_d + (long long)t * xp_ld + wrow) : 0.f;

  for (int s = 0; s < T; ++s) {
    const int cur = s & 1, nxt = cur ^ 1;
    t = dir == 0 ? s : T - 1 - s;
    const int tn = dir == 0 ? s + 1 : T - 2 - s;
    // arm the barrier that will collect h_{s+1}: 256 floats from the 8 CTAs of the cluster (this one included)
    if (threadIdx.x == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(nxt ? mb1 : mb0), "r"(GRU_H * 4) : "memory");
    float xv_next = 0.f;
    if (active && q == 0 && s + 1 < T) xv_next = __ldg(xp_d + (long long)tn * xp_ld + wrow);

    const float* h = &hbuf[cur][q * (GRU_H / 4)];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int k = 0; k < GRU_H / 4; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h + k);
      a0 = fmaf(w[k], hv.x, a0);
      a1 = fmaf(w[k + 1], hv.y, a1);
      a2 = fmaf(w[k + 2], hv.z, a2);
      a3 = fmaf(w[k + 3], hv.w, a3);
    }
    float acc = (a0 + a1) + (a2 + a3);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    const float hp = acc + bh;                              // W_h* h + b_h*   (valid on the q == 0 lane of each gate)
    // gather (x, hp) of the three gates on the unit's leader lane
    const int base = ul * 12;
    const float hp_r = __shfl_sync(0xffffffffu, hp, base + 0), hp_z = __shfl_sync(0xffffffffu, hp, base + 4),
                hp_n = __shfl_sync(0xffffffffu, hp, base + 8);
    const float x_r = __shfl_sync(0xffffffffu, xv, base + 0), x_z = __shfl_sync(0xffffffffu, xv, base + 4),
                x_n = __shfl_sync(0xffffffffu, xv, base + 8);
    if (leader) {
      const float r = 1.f / (1.f + expf(-(x_r + hp_r)));
      const float z = 1.f / (1.f + expf(-(x_z + hp_z)));
      const float n = tanhf(x_n + r * hp_n);
      const float hprev = hbuf[cur][unit];
      const float hnew = (1.f - z) * n + z * hprev;
      out[(long long)t * (2 * GRU_H) + dir * GRU_H + unit] = hnew;
      const uint32_t off_h = (uint32_t)((nxt * GRU_H + unit) * 4), off_mb = (uint32_t)(nxt * 8);
#pragma unroll
      for (int d = 0; d < GRU_CL; ++d)
        asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(peer_h[d] + off_h),
                     "r"(__float_as_uint(hnew)), "r"(peer_mb[d] + off_mb)
                     : "memory");
    }
    xv = xv_next;
    // wait for all 256 floats of h_{s+1}
    {
      const uint32_t bar = nxt ? mb1 : mb0;
      const uint32_t parity = (uint32_t)((s >> 1) & 1);
      asm volatile(
          "{\n\t"
          ".reg .pred p;\n\t"
          "GRU_WAIT:\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
          "@p bra GRU_DONE;\n\t"
          "bra GRU_WAIT;\n\t"
          "GRU_DONE:\n\t"
          "}" ::"r"(bar), "r"(parity)
          : "memory");
    }
  }
  cluster.sync();      // no CTA may exit while a peer could still write into its shared memory
}

// BiGRU v3: v2's shuffle-combined gates, but the exchange is ONE 128-byte cp.async.bulk (shared::cta -> shared::cluster,
// mbarrier complete_tx) per peer and step instead of one st.async per (unit, peer): 8 remote transactions per CTA and step.
__global__ void __cluster_dims__(GRU_CL, 1, 1) __launch_bounds__(GRU2_THREADS, 1)
bigru_v3_kernel(const float* __restrict__ xp, const float* __restrict__ whh /*[2][3H][H]*/,
                const float* __restrict__ bhh /*[2][3H]*/, float* __restrict__ out, int T) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.x / GRU_CL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool active = lane < 24;
  const int ul = lane / 12;                         // unit within the warp (0/1); lanes 24..31 idle
  const int li = lane - ul * 12;                    // 0..11
  const int g = li >> 2, q = li & 3;                // gate (r,z,n), K quarter
  const int j = warp * 2 + (active ? ul : 0);       // unit inside this CTA, 0..31
  const int unit = rank * GRU_UPC + j;
  const int wrow = g * GRU_H + unit;
  const bool leader = active && li == 0;

  __shared__ __align__(16) float hbuf[2][GRU_H];
  __shared__ __align__(16) float hst[2][GRU_UPC];          // this CTA's new slice, staged for the bulk copies
  __shared__ __align__(8) unsigned long long mbar[2];

  float w[GRU_H / 4];
  float bh = 0.f;
  if (active) {
    const float* src = whh + ((long long)dir * 3 * GRU_H + wrow) * GRU_H + q * (GRU_H / 4);
#pragma unroll
    for (int k = 0; k < GRU_H / 4; k += 4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(src + k));
      w[k] = v.x; w[k + 1] = v.y; w[k + 2] = v.z; w[k + 3] = v.w;
    }
    bh = bhh[dir * 3 * GRU_H + wrow];
  } else {
#pragma unroll
    for (int k = 0; k < GRU_H / 4; ++k) w[k] = 0.f;
  }
  for (int i = threadIdx.x; i < 2 * GRU_H; i += GRU2_THREADS) (&hbuf[0][0])[i] = 0.f;
  const uint32_t mb0 = gru_smem_u32(&mbar[0]), mb1 = gru_smem_u32(&mbar[1]);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb0));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster.sync();

  // remote addresses of every CTA's h buffers / barriers (leader lanes only)
  uint32_t peer_h[GRU_CL], peer_mb[GRU_CL];
#pragma unroll
  for (int d = 0; d < GRU_CL; ++d) {
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_h[d]) : "r"(gru_smem_u32(&hbuf[0][0])), "r"(d));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_mb[d]) : "r"(mb0), "r"(d));
  }

  const long long xp_ld = 2 * 3 * GRU_H;
  const float* xp_d = xp + dir * 3 * GRU_H;
  int t = dir == 0 ? 0 : T - 1;
  // x-projections of this thread's gate row, one step ahead (only the q == 0 lane of each gate uses it)
  float xv = (active && q == 0) ? __ldg(xp_d + (long long)t * xp_ld + wrow) : 0.f;

  for (int s = 0; s < T; ++s) {
    const int cur = s & 1, nxt = cur ^ 1;
    t = dir == 0 ? s : T - 1 - s;
    const int tn = dir == 0 ? s + 1 : T - 2 - s;
    // arm the barrier that will collect h_{s+1}: 256 floats from the 8 CTAs of the cluster (this one included)
    if (threadIdx.x == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(nxt ? mb1 : mb0), "r"(GRU_H * 4) : "memory");
    float xv_next = 0.f;
    if (active && q == 0 && s + 1 < T) xv_next = __ldg(xp_d + (long long)tn * xp_ld + wrow);

    const float* h = &hbuf[cur][q * (GRU_H / 4)];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int k = 0; k < GRU_H / 4; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h + k);
      a0 = fmaf(w[k], hv.x, a0);
      a1 = fmaf(w[k + 1], hv.y, a1);
      a2 = fmaf(w[k + 2], hv.z, a2);
      a3 = fmaf(w[k + 3], hv.w, a3);
    }
    float acc = (a0 + a1) + (a2 + a3);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    const float hp = acc + bh;                              // W_h* h + b_h*   (valid on the q == 0 lane of each gate)
    // gather (x, hp) of the three gates on the unit's leader lane
    const int base = ul * 12;
    const float hp_r = __shfl_sync(0xffffffffu, hp, base + 0), hp_z = __shfl_sync(0xffffffffu, hp, base + 4),
                hp_n = __shfl_sync(0xffffffffu, hp, base + 8);
    const float x_r = __shfl_sync(0xffffffffu, xv, base + 0), x_z = __shfl_sync(0xffffffffu, xv, base + 4),
                x_n = __shfl_sync(0xffffffffu, xv, base + 8);
    if (leader) {
      const float r = 1.f / (1.f + expf(-(x_r + hp_r)));
      const float z = 1.f / (1.f + expf(-(x_z + hp_z)));
      const float n = tanhf(x_n + r * hp_n);
      const float hprev = hbuf[cur][unit];
      const float hnew = (1.f - z) * n + z * hprev;
      out[(long long)t * (2 * GRU_H) + dir * GRU_H + unit] = hnew;
      hst[nxt][j] = hnew;
    }
    xv = xv_next;
    __syncthreads();                                   // the 32 new values of this CTA are staged
    if (threadIdx.x == 0) {
      // generic-proxy writes -> async-proxy reads, then ONE 128-byte bulk copy per peer (data + arrival signal together)
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      const uint32_t src = gru_smem_u32(&hst[nxt][0]);
      const uint32_t off_h = (uint32_t)((nxt * GRU_H + rank * GRU_UPC) * 4), off_mb = (uint32_t)(nxt * 8);
#pragma unroll
      for (int d = 0; d < GRU_CL; ++d)
        asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(peer_h[d] + off_h),
                     "r"(src), "r"(GRU_UPC * 4), "r"(peer_mb[d] + off_mb)
                     : "memory");
    }
    // wait for all 256 floats of h_{s+1}
    {
      const uint32_t bar = nxt ? mb1 : mb0;
      const uint32_t parity = (uint32_t)((s >> 1) & 1);
      asm volatile(
          "{\n\t"
          ".reg .pred p;\n\t"
          "GRU3_WAIT:\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
          "@p bra GRU3_DONE;\n\t"
          "bra GRU3_WAIT;\n\t"
          "GRU3_DONE:\n\t"
          "}" ::"r"(bar), "r"(parity)
          : "memory");
    }
  }
  cluster.sync();      // no CTA may exit while a peer could still write into its shared memory
}

// ---------------------------------------------------------------------------
// to_local_average_cents + decode (rmvpe.py:359-364, 385-409) — one warp per frame, float64 where
// numpy is float64, and numpy's pairwise summation order for the 9-element reductions:
//   sum9(a) = (((a0+a1)+(a2+a3)) + ((a4+a5)+(a6+a7))) + a8
// ---------------------------------------------------------------------------
__global__ void rmvpe_decode_kernel(const float* __restrict__ sal, double* __restrict__ f0,
                                    double* __restrict__ cents_out, int T, int NB,
                                    long long ld, float thred) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= T) return;
  const float* s = sal + (long long)warp * ld;
  // argmax with numpy's first-occurrence tie rule
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int k = lane; k < NB; k += 32) {
    const float v = s[k];
    if (v > best) { best = v; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) {
    float sv[9];
    double pv[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int k = bi - 4 + i;
      const bool in = (k >= 0 && k < NB);
      sv[i] = in ? s[k] : 0.f;
      const double cents = in ? (20.0 * (double)k + 1997.3794084376191) : 0.0;
      pv[i] = __dmul_rn((double)sv[i], cents);   // no FMA contraction: numpy rounds the product first
    }
    const double psum = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(pv[0], pv[1]), __dadd_rn(pv[2], pv[3])),
                                            __dadd_rn(__dadd_rn(pv[4], pv[5]), __dadd_rn(pv[6], pv[7]))), pv[8]);
    const float wsum = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(sv[0], sv[1]), __fadd_rn(sv[2], sv[3])),
                                           __fadd_rn(__fadd_rn(sv[4], sv[5]), __fadd_rn(sv[6], sv[7]))), sv[8]);
    double cents = psum / (double)wsum;
    if (best <= thred) cents = 0.0;
    if (cents_out) cents_out[warp] = cents;
    double f = 10.0 * exp2(cents / 1200.0);
    if (f == 10.0) f = 0.0;
    f0[warp] = f;
  }
}

}  // namespace
}  // namespace b200vc

using namespace b200vc;

extern "C" {

int b200vc_reflect_pad_1d(const float* in, float* out, int64_t N, int64_t pad, void* stream) {
  B200VC_RECORD(b200vc_reflect_pad_1d(in, out, N, pad, stream));
  B200VC_REQUIRE(in && out && N > pad && pad >= 0, "reflect_pad_1d: bad args");
  const long long total = N + 2 * pad;
  reflect_pad_1d_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, N, pad, total);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_magnitude(const float* spec, float* mag, int64_t rows, int nb, int64_t lds, int64_t ldm, void* stream) {
  B200VC_RECORD(b200vc_magnitude(spec, mag, rows, nb, lds, ldm, stream));
  B200VC_REQUIRE(spec && mag && rows > 0 && nb > 0 && ldm >= nb, "magnitude: bad args");
  magnitude_kernel<<<blocks_for(rows * ldm, 256), 256, 0, (cudaStream_t)stream>>>(spec, mag, rows, nb, lds, ldm);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_logmel_affine_reflect(const float* x, float* out, int rows, int rows_total, int C, float clampv,
                                 float a, float b, void* stream) {
  B200VC_RECORD(b200vc_logmel_affine_reflect(x, out, rows, rows_total, C, clampv, a, b, stream));
  B200VC_REQUIRE(x && out && rows > 0 && rows_total >= rows && rows_total - rows < rows, "logmel: bad args");
  logmel_affine_reflect_kernel<<<blocks_for((long long)rows_total * C, 256), 256, 0, (cudaStream_t)stream>>>(
      x, out, rows, rows_total, C, clampv, a, b);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_avgpool2x2(const float* in, float* out, int B, int H, int W, int C, int64_t ldi, void* stream) {
  B200VC_RECORD(b200vc_avgpool2x2(in, out, B, H, W, C, ldi, stream));
  B200VC_REQUIRE(in && out && B > 0 && H % 2 == 0 && W % 2 == 0 && C > 0, "avgpool2x2: bad args");
  const long long n = (long long)B * (H / 2) * (W / 2) * C;
  avgpool2x2_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(in, out, B, H, W, C, ldi);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_avgpool2x2_split(const float* in, float* out, int B, int H, int W, int C, int64_t ldi, int64_t in_split,
                            int64_t ldo, int64_t out_split, void* stream) {
  B200VC_RECORD(b200vc_avgpool2x2_split(in, out, B, H, W, C, ldi, in_split, ldo, out_split, stream));
  B200VC_REQUIRE(in && out && B > 0 && H % 2 == 0 && W % 2 == 0 && C > 0, "avgpool2x2_split: bad args");
  const long long n = (long long)B * (H / 2) * (W / 2) * C;
  avgpool2x2_split_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(in, out, B, H, W, C, ldi, in_split, ldo, out_split);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_bigru(const float* xp, const float* whh, const float* bhh, float* out, int T, int hidden, void* stream) {
  B200VC_RECORD(b200vc_bigru(xp, whh, bhh, out, T, hidden, stream));
  B200VC_REQUIRE(xp && whh && bhh && out && T > 0, "bigru: bad args");
  B200VC_REQUIRE(hidden == GRU_H, "bigru: hidden size %d unsupported (kernel is specialised for %d)", hidden, GRU_H);
  // v2 (st.async + mbarrier per step) and v3 (bulk copy per peer) are kept behind B200VC_GRU=2 / 3 for experiments
  const char* e = getenv("B200VC_GRU");                 // 1 (default) | 2 | 3: exchange variant, see the kernels above
  const int ver = (e && (e[0] == '2' || e[0] == '3')) ? e[0] - '0' : 1;
  if (ver == 1) bigru_kernel<<<2 * GRU_CL, GRU_THREADS, 0, (cudaStream_t)stream>>>(xp, whh, bhh, out, T);
  else if (ver == 2) bigru_v2_kernel<<<2 * GRU_CL, GRU2_THREADS, 0, (cudaStream_t)stream>>>(xp, whh, bhh, out, T);
  else bigru_v3_kernel<<<2 * GRU_CL, GRU2_THREADS, 0, (cudaStream_t)stream>>>(xp, whh, bhh, out, T);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

int b200vc_rmvpe_decode(const float* salience, double* f0, double* cents, int T, int n_bins, int64_t ld, float thred,
                        void* stream) {
  B200VC_RECORD(b200vc_rmvpe_decode(salience, f0, cents, T, n_bins, ld, thred, stream));
  B200VC_REQUIRE(salience && f0 && T > 0 && n_bins > 0, "rmvpe_decode: bad args");
  rmvpe_decode_kernel<<<blocks_for((long long)T * 32, 256), 256, 0, (cudaStream_t)stream>>>(salience, f0, cents, T,
                                                                                           n_bins, ld, thred);
  count_launch();
  B200VC_LAUNCH_CHECK();
  return kOk;
}

}  // extern "C"
