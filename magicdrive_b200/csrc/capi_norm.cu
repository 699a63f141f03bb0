// GroupNorm(+SiLU) over NHWC (optionally over a two-source channel concat) and LayerNorm.  HBM-bound kernels:
// 16-byte vector loads along the contiguous channel axis, fp32 statistics, warp-shuffle / smem reductions.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdlib.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"
#include "ptx_cluster.cuh"

// Images of at least this many bytes take the pixel-major cluster GroupNorm when MDB_GN_ROWS is unset (the crossover against
// gn_fused_kernel; a larger threshold for inputs that only fit a 16-CTA cluster).  tools/bench_norm.py times both kernels on
// the shapes of one denoising step.
#ifndef MDB_GN_ROWS_MIN_BYTES
#define MDB_GN_ROWS_MIN_BYTES 850000LL
#endif
#ifndef MDB_GN_ROWS_MIN_BYTES_C16
#define MDB_GN_ROWS_MIN_BYTES_C16 2500000LL
#endif

namespace {

// F16 (the GroupNorm kernels' template flag): f16 activations (fp16 models) in place of bf16; statistics stay fp32
template <bool F16 = false>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  using A = mdb::Act<F16>;
  const typename A::T2* h = reinterpret_cast<const typename A::T2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = A::to_float2(h[i]);
    f[2 * i] = t.x, f[2 * i + 1] = t.y;
  }
}
template <bool F16 = false>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  using A = mdb::Act<F16>;
  uint4 u;
  u.x = A::pack(f[0], f[1]), u.y = A::pack(f[2], f[3]);
  u.z = A::pack(f[4], f[5]), u.w = A::pack(f[6], f[7]);
  return u;
}

// Shift of group g of an image for the two-kernel statistics: the image's first pixel, first channel of the group.  Sums of
// (x - shift) keep E[d^2] - E[d]^2 well conditioned: a sample of the group lies within a few standard deviations of its mean,
// whereas the plain E[x^2] - mean^2 in fp32 is off by several percent once |mean| is a few hundred standard deviations.
template <bool F16>
__device__ __forceinline__ float gn_shift(const typename mdb::Act<F16>::T* __restrict__ x0, int c0, int ld0,
                                          const typename mdb::Act<F16>::T* __restrict__ x1, int ld1, long long pix, int c) {
  return mdb::Act<F16>::to_float(c < c0 ? x0[pix * ld0 + c] : x1[pix * ld1 + (c - c0)]);
}

// ---- GroupNorm pass 1: per (image, group) sum / sum-of-squares of x - shift.  blockDim = vpp * R, thread = (pixel lane r,
// channel vector cv)
template <bool F16>
__device__ __forceinline__ void gn_stats(const typename mdb::Act<F16>::T* __restrict__ x0, int c0, int ld0,
                                         const typename mdb::Act<F16>::T* __restrict__ x1, int c1, int ld1, int hw, int groups,
                                         int vpp, int R, int pix_per_cta, float* __restrict__ stats) {
  extern __shared__ float sm[];  // [2][ctot]
  const int ctot = c0 + c1;
  const int cpg = ctot / groups;
  const int img = blockIdx.y;
  const int p_begin = blockIdx.x * pix_per_cta;
  const int p_end = min(hw, p_begin + pix_per_cta);
  for (int i = threadIdx.x; i < 2 * ctot; i += blockDim.x) sm[i] = 0.f;
  __syncthreads();
  const int cv = threadIdx.x % vpp;
  const int r = threadIdx.x / vpp;
  if (r < R) {
    const int ch = cv * 8;
    const typename mdb::Act<F16>::T* base;
    int ld, coff;
    if (ch < c0) base = x0, ld = ld0, coff = ch;
    else base = x1, ld = ld1, coff = ch - c0;
    float s[8], ss[8], k[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] = 0.f, ss[i] = 0.f;
      k[i] = gn_shift<F16>(x0, c0, ld0, x1, ld1, static_cast<long long>(img) * hw, (ch + i) / cpg * cpg);
    }
    for (int p = p_begin + r; p < p_end; p += R) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + (static_cast<long long>(img) * hw + p) * ld + coff));
      float f[8];
      unpack8<F16>(u, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[i] - k[i];
        s[i] += d, ss[i] += d * d;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      atomicAdd(&sm[ch + i], s[i]);
      atomicAdd(&sm[ctot + ch + i], ss[i]);
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) a += sm[c], b += sm[ctot + c];
    atomicAdd(&stats[(img * groups + g) * 2], a);
    atomicAdd(&stats[(img * groups + g) * 2 + 1], b);
  }
}

__global__ void gn_stats_kernel(const __nv_bfloat16* __restrict__ x0, int c0, int ld0, const __nv_bfloat16* __restrict__ x1,
                                int c1, int ld1, int hw, int groups, int vpp, int R, int pix_per_cta, float* __restrict__ stats) {
  gn_stats<false>(x0, c0, ld0, x1, c1, ld1, hw, groups, vpp, R, pix_per_cta, stats);
}
__global__ void gn_stats_f16_kernel(const __half* __restrict__ x0, int c0, int ld0, const __half* __restrict__ x1, int c1,
                                    int ld1, int hw, int groups, int vpp, int R, int pix_per_cta, float* __restrict__ stats) {
  gn_stats<true>(x0, c0, ld0, x1, c1, ld1, hw, groups, vpp, R, pix_per_cta, stats);
}

// ---- GroupNorm pass 2: mean = shift + E[x - shift], var = E[(x - shift)^2] - E[x - shift]^2;
// y = (x - mean) * rstd * gamma + beta, optional SiLU, bf16 out.
template <bool F16>
__device__ __forceinline__ void gn_apply(const typename mdb::Act<F16>::T* __restrict__ x0, int c0, int ld0,
                                         const typename mdb::Act<F16>::T* __restrict__ x1, int c1, int ld1, int hw, int groups,
                                         float eps, const float* __restrict__ gamma, const float* __restrict__ beta, int silu,
                                         const float* __restrict__ stats, typename mdb::Act<F16>::T* __restrict__ out, int ldo,
                                         int pix_per_cta) {
  extern __shared__ float sm[];  // scale[ctot], shift[ctot]
  const int ctot = c0 + c1;
  const int img = blockIdx.y;
  const int cpg = ctot / groups;
  const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(hw));
  for (int c = threadIdx.x; c < ctot; c += blockDim.x) {
    const int g = c / cpg;
    const float dmean = stats[(img * groups + g) * 2] * inv_cnt;  // mean of x - shift
    float var = stats[(img * groups + g) * 2 + 1] * inv_cnt - dmean * dmean;
    var = fmaxf(var, 0.f);
    const float mean = gn_shift<F16>(x0, c0, ld0, x1, ld1, static_cast<long long>(img) * hw, g * cpg) + dmean;
    const float rstd = rsqrtf(var + eps);
    const float a = rstd * gamma[c];
    sm[c] = a;
    sm[ctot + c] = beta[c] - mean * a;
  }
  __syncthreads();
  const int vpp = ctot / 8;
  const int p_begin = blockIdx.x * pix_per_cta;
  const int p_end = min(hw, p_begin + pix_per_cta);
  const int total = (p_end - p_begin) * vpp;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int p = p_begin + idx / vpp;
    const int ch = (idx % vpp) * 8;
    const long long pix = static_cast<long long>(img) * hw + p;
    const uint4 u = (ch < c0) ? __ldg(reinterpret_cast<const uint4*>(x0 + pix * ld0 + ch))
                              : __ldg(reinterpret_cast<const uint4*>(x1 + pix * ld1 + (ch - c0)));
    float f[8];
    unpack8<F16>(u, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float y = f[i] * sm[ch + i] + sm[ctot + ch + i];
      if (silu) y = y / (1.0f + __expf(-y));
      f[i] = y;
    }
    *reinterpret_cast<uint4*>(out + pix * ldo + ch) = pack8<F16>(f);
  }
}

__global__ void gn_apply_kernel(const __nv_bfloat16* __restrict__ x0, int c0, int ld0, const __nv_bfloat16* __restrict__ x1,
                                int c1, int ld1, int hw, int groups, float eps, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int silu, const float* __restrict__ stats,
                                __nv_bfloat16* __restrict__ out, int ldo, int pix_per_cta) {
  gn_apply<false>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta, silu, stats, out, ldo, pix_per_cta);
}
__global__ void gn_apply_f16_kernel(const __half* __restrict__ x0, int c0, int ld0, const __half* __restrict__ x1, int c1,
                                    int ld1, int hw, int groups, float eps, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, int silu, const float* __restrict__ stats,
                                    __half* __restrict__ out, int ldo, int pix_per_cta) {
  gn_apply<true>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta, silu, stats, out, ldo, pix_per_cta);
}

// ---- GroupNorm, single kernel: one CTA per (image, group).  The group's hw x cpg slab (a few tens of KB, L2-resident:
// it was just written by the producing GEMM) is copied once into shared memory with 4-byte cp.async (every load in
// flight at once, no registers, no unrolling: the first version cached the slab in 56 unrolled registers and spent
// most of its time in instruction-cache misses), mean and variance are computed exactly (two passes over smem),
// then normalise + affine (+SiLU) and store.  No atomics, no memset, no stats buffer.
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst_smem))),
               "l"(src)
               : "memory");
}

template <bool CACHED, bool F16 = false>
__global__ void __launch_bounds__(256) gn_fused_kernel(const typename mdb::Act<F16>::T* __restrict__ x0, int c0, int ld0,
                                                       const typename mdb::Act<F16>::T* __restrict__ x1, int c1, int ld1, int hw,
                                                       int groups, float eps, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int silu,
                                                       typename mdb::Act<F16>::T* __restrict__ out, int ldo, uint32_t inv_pp) {
  using A = mdb::Act<F16>;
  constexpr int T = 256;
  mdb::pdl_wait();
  mdb::pdl_launch_dependents();
  // [units] bf16x2 / f16x2 (CACHED only); 128-byte aligned like gn_rows_kernel's slab, which shares the dynamic region
  extern __shared__ __align__(128) uint32_t slab[];
  __shared__ float red[T / 32];
  __shared__ float bcast;
  const int g = blockIdx.x, img = blockIdx.y;
  const int ctot = c0 + c1;
  const int cpg = ctot / groups;
  const int pp = cpg >> 1;  // bf16x2 units per pixel
  const int units = hw * pp;
  const int cbase = g * cpg;
  const long long pix0 = static_cast<long long>(img) * hw;
  // u / pp by multiply-high with a host-computed reciprocal (exact for u * pp < 2^32)
  auto split = [&](int u, int& p, int& c) {
    p = (pp == 1) ? u : static_cast<int>(__umulhi(static_cast<uint32_t>(u), inv_pp));
    c = cbase + 2 * (u - p * pp);
  };
  auto src = [&](int u) -> const uint32_t* {
    int p, c;
    split(u, p, c);
    return (c < c0) ? reinterpret_cast<const uint32_t*>(x0 + (pix0 + p) * ld0 + c)
                    : reinterpret_cast<const uint32_t*>(x1 + (pix0 + p) * ld1 + (c - c0));
  };
  auto value = [&](int u) -> float2 {
    const uint32_t w = CACHED ? slab[u] : __ldg(src(u));
    return A::to_float2(*reinterpret_cast<const typename A::T2*>(&w));
  };
  auto block_sum = [&](float v) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = (threadIdx.x < T / 32) ? red[threadIdx.x] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) bcast = t;
    }
    __syncthreads();
    return bcast;
  };
  if (CACHED) {
    for (int u = threadIdx.x; u < units; u += T) cp_async4(&slab[u], src(u));
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
  }
  float s = 0.f;
#pragma unroll 4
  for (int u = threadIdx.x; u < units; u += T) {
    const float2 f = value(u);
    s += f.x + f.y;
  }
  const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(hw));
  const float mean = block_sum(s) * inv_cnt;
  float sq = 0.f;
#pragma unroll 4
  for (int u = threadIdx.x; u < units; u += T) {
    const float2 f = value(u);
    const float d0 = f.x - mean, d1 = f.y - mean;
    sq += d0 * d0 + d1 * d1;
  }
  const float rstd = rsqrtf(block_sum(sq) * inv_cnt + eps);
#pragma unroll 4
  for (int u = threadIdx.x; u < units; u += T) {
    int p, c;
    split(u, p, c);
    const float2 f = value(u);
    const float2 ga = __ldg(reinterpret_cast<const float2*>(gamma + c));
    const float2 be = __ldg(reinterpret_cast<const float2*>(beta + c));
    float y0 = (f.x - mean) * rstd * ga.x + be.x;
    float y1 = (f.y - mean) * rstd * ga.y + be.y;
    if (silu) {
      y0 = y0 / (1.0f + __expf(-y0));
      y1 = y1 / (1.0f + __expf(-y1));
    }
    *reinterpret_cast<uint32_t*>(out + (pix0 + p) * ldo + c) = A::pack(y0, y1);
  }
}

// ---- LayerNorm: one warp per row, values kept in registers (two-pass mean / variance like ATen).
template <int MAXV>
__global__ void layernorm_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int c, int ldx,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 __nv_bfloat16* __restrict__ out, int ldo) {
  mdb::pdl_wait();
  mdb::pdl_launch_dependents();
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nvec = c / 8;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + row * ldx + vi * 8));
      unpack8(u, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[i][j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / static_cast<float>(c);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        sq += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / static_cast<float>(c) + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float y[8];
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8 + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = (v[i][j] - mean) * rstd * gg[j] + bb[j];
      *reinterpret_cast<uint4*>(out + row * ldo + vi * 8) = pack8(y);
    }
  }
}


// ---- GroupNorm, pixel-major on a thread-block cluster per image (MDB_GN_ROWS=1 forces it, =0 disables it).  The image's
// pixels are split into contiguous runs, one per CTA of the cluster.  A CTA pulls its run into shared memory ONCE with bulk-async
// copies (cp.async.bulk: no registers, every byte in flight at once -- the per-thread 16-byte-load loop of the first cluster
// kernel was latency-bound at ~0.8 TB/s; a dense source is a handful of 16 KB copies, a strided one a copy per pixel row),
// computes per-group (mean, M2) of the run exactly (two passes over shared memory), publishes them in its own shared memory,
// and after ONE cluster barrier combines the runs of the image through distributed shared memory (Chan's parallel variance:
// no E[x^2] - mean^2 cancellation), normalises its run from shared memory (+ affine, + SiLU) and stores it with coalesced
// 16-byte stores.  One global read and one global write per element, both in full rows; gn_fused_kernel reads 20..80-byte
// channel slices per pixel instead.  blockDim = vpp * R (vpp = 16-byte vectors per pixel), thread = (pixel lane r, channel
// vector cv): a thread's 8 channels, their groups, gamma and beta are fixed for the whole kernel.
__device__ __forceinline__ float ld_dsmem_f32(uint32_t cluster_addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr));
  return v;
}
template <bool F16>
__device__ __forceinline__ void gn_rows(const typename mdb::Act<F16>::T* __restrict__ x0, int c0, int ld0,
                                        const typename mdb::Act<F16>::T* __restrict__ x1, int c1, int ld1, int hw, int groups,
                                        float eps, const float* __restrict__ gamma, const float* __restrict__ beta, int silu,
                                        typename mdb::Act<F16>::T* __restrict__ out, int ldo, int vpp, int R, int ctas_per_img,
                                        int pix_per_cta) {
  using namespace mdb;
  using Elt = typename Act<F16>::T;
  extern __shared__ __align__(128) uint4 gslab[];  // [pix_per_cta][c0] | [pix_per_cta][c1] bf16, then float red[R][ctot]
  const int ctot = c0 + c1, cpg = ctot / groups;
  float* red = reinterpret_cast<float*>(gslab + static_cast<size_t>(pix_per_cta) * vpp);  // [R][ctot]
  __shared__ float g_a[128], g_b[128];  // per group: mean / rstd of the image
  __shared__ float part[256];           // per group: (mean, M2) of this CTA's run -- read by the cluster peers
  __shared__ __align__(8) uint64_t full_bar;
  const int img = blockIdx.x / ctas_per_img, run = blockIdx.x % ctas_per_img;  // run == %cluster_ctarank (1-D clusters)
  const int p_begin = min(hw, run * pix_per_cta), p_end = min(hw, p_begin + pix_per_cta);
  const int npix = p_end - p_begin;
  const int cv = threadIdx.x % vpp, r0 = threadIdx.x / vpp;
  const int ch = cv * 8;
  const long long pix0 = static_cast<long long>(img) * hw + p_begin;
  // this thread's 8 channels inside the slab of their source: element p of the run at mine[p * pitch]
  const int vpp0 = c0 / 8;
  const uint4* mine = (ch < c0) ? gslab + cv : gslab + static_cast<size_t>(pix_per_cta) * vpp0 + (cv - vpp0);
  const int pitch = (ch < c0) ? vpp0 : vpp - vpp0;
  if (threadIdx.x == 0) {
    mbar_init(&full_bar, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&full_bar, static_cast<uint32_t>(npix) * ctot * 2);
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the producer's tail
  pdl_launch_dependents();
  // ---- the run of each source lands in its own slab ([pixel][c0] then [pixel][c1]): a dense source (row stride == channels,
  // every activation of the step) is ONE contiguous range, fetched as 16 KB bulk copies; a strided one row by row.
  // All copies complete on full_bar.
  {
    const uint32_t bar = smem_u32(&full_bar);
    auto fetch = [&](const Elt* src, int c, int ld, uint32_t dst) {
      if (c == 0) return;
      if (ld == c) {
        const uint32_t bytes = static_cast<uint32_t>(npix) * c * 2;
        const char* g = reinterpret_cast<const char*>(src + pix0 * ld);
        for (uint32_t off = threadIdx.x * 16384u; off < bytes; off += blockDim.x * 16384u) {
          const uint32_t n = min(16384u, bytes - off);
          asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst + off),
                       "l"(g + off), "r"(n), "r"(bar)
                       : "memory");
        }
      } else {
        for (int p = threadIdx.x; p < npix; p += blockDim.x)
          asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                           dst + static_cast<uint32_t>(p) * c * 2),
                       "l"(src + (pix0 + p) * ld), "r"(c * 2), "r"(bar)
                       : "memory");
      }
    };
    fetch(x0, c0, ld0, smem_u32(gslab));
    fetch(x1, c1, ld1, smem_u32(gslab) + static_cast<uint32_t>(pix_per_cta) * c0 * 2);
  }
  mbar_wait(&full_bar, 0);
  // ---- per-channel sums of the run -> per-group local mean
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int p = r0; p < npix; p += R) {
    float f[8];
    unpack8<F16>(mine[p * pitch], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += f[e];
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[r0 * ctot + ch + e] = acc[e];
  __syncthreads();
  const float cnt_local = static_cast<float>(npix) * static_cast<float>(cpg);
  for (int c = threadIdx.x; c < ctot; c += blockDim.x) {  // fold the R pixel lanes: red[0][c] = channel sum of the run
    float s = red[c];
    for (int r = 1; r < R; ++r) s += red[r * ctot + c];
    red[c] = s;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < cpg; ++c) s += red[g * cpg + c];
    part[2 * g] = npix > 0 ? s / cnt_local : 0.f;  // local mean
  }
  __syncthreads();
  // ---- local M2 around the local mean (second pass over shared memory)
  float lm[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) lm[e] = part[2 * ((ch + e) / cpg)], acc[e] = 0.f;
  for (int p = r0; p < npix; p += R) {
    float f[8];
    unpack8<F16>(mine[p * pitch], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = f[e] - lm[e];
      acc[e] = fmaf(d, d, acc[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[r0 * ctot + ch + e] = acc[e];
  __syncthreads();
  for (int c = threadIdx.x; c < ctot; c += blockDim.x) {
    float s = red[c];
    for (int r = 1; r < R; ++r) s += red[r * ctot + c];
    red[c] = s;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < cpg; ++c) s += red[g * cpg + c];
    part[2 * g + 1] = s;
  }
  // ---- every run's (mean, M2) is published: combine the runs of this image (Chan et al.):
  //      mean = sum n_i m_i / N,  M2 = sum M2_i + sum n_i (m_i - mean)^2
  if (ctas_per_img > 1) cluster_sync_all(); else __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float wsum = 0.f;
    for (int r = 0; r < ctas_per_img; ++r) {
      const int nb = min(hw, r * pix_per_cta), ne = min(hw, nb + pix_per_cta);
      const float m = (ctas_per_img > 1) ? ld_dsmem_f32(mapa_u32(smem_u32(&part[2 * g]), r)) : part[2 * g];
      wsum += static_cast<float>(ne - nb) * m;
    }
    const float mean = wsum / static_cast<float>(hw);
    float m2 = 0.f;
    for (int r = 0; r < ctas_per_img; ++r) {
      const int nb = min(hw, r * pix_per_cta), ne = min(hw, nb + pix_per_cta);
      float m, q;
      if (ctas_per_img > 1) {
        const uint32_t a = mapa_u32(smem_u32(&part[2 * g]), r);
        m = ld_dsmem_f32(a), q = ld_dsmem_f32(a + 4);
      } else {
        m = part[2 * g], q = part[2 * g + 1];
      }
      const float d = m - mean;
      m2 += q + static_cast<float>(ne - nb) * static_cast<float>(cpg) * d * d;
    }
    g_a[g] = mean;
    g_b[g] = rsqrtf(m2 / (static_cast<float>(hw) * static_cast<float>(cpg)) + eps);
  }
  // peers may still be reading this CTA's `part`: arrive now, wait before exit
  if (ctas_per_img > 1) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  __syncthreads();
  // ---- normalise + affine (+SiLU) from shared memory, coalesced 16-byte stores
  float sa[8], sb[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float rs = g_b[(ch + e) / cpg], mu = g_a[(ch + e) / cpg];
    sa[e] = rs * __ldg(gamma + ch + e);
    sb[e] = __ldg(beta + ch + e) - mu * sa[e];
  }
  Elt* dst = out + pix0 * ldo + ch;
  for (int p = r0; p < npix; p += R) {
    float f[8];
    unpack8<F16>(mine[p * pitch], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = fmaf(f[e], sa[e], sb[e]);
      if (silu) y = y / (1.0f + __expf(-y));
      f[e] = y;
    }
    *reinterpret_cast<uint4*>(dst + static_cast<long long>(p) * ldo) = pack8<F16>(f);
  }
  if (ctas_per_img > 1) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void gn_rows_kernel(const __nv_bfloat16* __restrict__ x0, int c0, int ld0, const __nv_bfloat16* __restrict__ x1,
                               int c1, int ld1, int hw, int groups, float eps, const float* __restrict__ gamma,
                               const float* __restrict__ beta, int silu, __nv_bfloat16* __restrict__ out, int ldo, int vpp, int R,
                               int ctas_per_img, int pix_per_cta) {
  gn_rows<false>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta, silu, out, ldo, vpp, R, ctas_per_img, pix_per_cta);
}
__global__ void gn_rows_f16_kernel(const __half* __restrict__ x0, int c0, int ld0, const __half* __restrict__ x1, int c1,
                                   int ld1, int hw, int groups, float eps, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, int silu, __half* __restrict__ out, int ldo, int vpp, int R,
                                   int ctas_per_img, int pix_per_cta) {
  gn_rows<true>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta, silu, out, ldo, vpp, R, ctas_per_img, pix_per_cta);
}

// the plain kernels of one element type (plain, not templates: the bf16 ones compile as they did before f16 existed)
template <bool F16> struct GnKernels {
  static constexpr auto stats = gn_stats_kernel;
  static constexpr auto apply = gn_apply_kernel;
  static constexpr auto rows = gn_rows_kernel;
};
template <> struct GnKernels<true> {
  static constexpr auto stats = gn_stats_f16_kernel;
  static constexpr auto apply = gn_apply_f16_kernel;
  static constexpr auto rows = gn_rows_f16_kernel;
};

// mdb_groupnorm (bf16) and mdb_groupnorm_f16: the same kernel choice for both element types
template <bool F16>
int groupnorm(const void* x0_, int c0, int ld0, const void* x1_, int c1, int ld1, int n_img, int hw, int groups, float eps,
              const float* gamma, const float* beta, int silu, void* out_, int ldo, float* stats_ws, void* stream) {
  using namespace mdb;
  using Elt = typename Act<F16>::T;
  const Elt* x0 = static_cast<const Elt*>(x0_);
  const Elt* x1 = static_cast<const Elt*>(x1_);
  Elt* out = static_cast<Elt*>(out_);
  const int ctot = c0 + c1;
  if (!x0 || !out || !stats_ws || !gamma || !beta) return set_error(MDB_ERR_INVALID, "mdb_groupnorm: null pointer");
  if (c0 % 8 || c1 % 8 || ld0 % 8 || (c1 && ld1 % 8) || ldo % 8 || ctot % groups || ctot > 4096)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_groupnorm: unsupported channel layout (c0=%d c1=%d groups=%d)", c0, c1,
                     groups);
  if (c1 > 0 && !x1) return set_error(MDB_ERR_INVALID, "mdb_groupnorm: c1>0 but x1 null");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  {
    // pixel-major cluster kernel: the default wherever an image is large enough that gn_fused_kernel's channel-slice reads
    // cost more than the cluster barrier (MDB_GN_ROWS_MIN_BYTES); MDB_GN_ROWS=1 forces it, =0 disables it
    const char* env = getenv("MDB_GN_ROWS");  // read per call: tests flip it inside one process
    const int mode = env ? ((env[0] == '1') ? 1 : 0) : -1;
    const int vpp = ctot / 8;
    const long long img_bytes = static_cast<long long>(hw) * ctot * 2;
    const bool want = mode == 1 || (mode == -1 && img_bytes >= MDB_GN_ROWS_MIN_BYTES);
    if (want && groups <= 128 && vpp <= 1024 && ld0 % 8 == 0 && (c1 == 0 || ld1 % 8 == 0)) {
      int R = 512 / vpp;
      if (R < 1) R = 1;
      // largest portable cluster (<= 8 CTAs per image: more SMs pull on the image) whose runs still give every pixel lane two
      // pixels and fit in shared memory; images too large for 8 CTAs (the 28x50 level's skip concats) take a 16-CTA cluster
      // (non-portable size: the driver is asked whether one fits a GPC before it is used)
      constexpr size_t kMaxSmem = 200 * 1024;
      static bool attr = false;
      static int max16 = -1;  // >0: 16-CTA clusters of this kernel can be co-scheduled
      if (!attr) {
        cudaFuncSetAttribute(GnKernels<F16>::rows, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kMaxSmem));
        max16 = (cudaFuncSetAttribute(GnKernels<F16>::rows, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) ? 1 : 0;
        cudaGetLastError();
        attr = true;
      }
      int cpi = 0, ppc = 0;
      size_t smem = 0;
      auto try_cluster = [&](int cand, bool allow_small_runs) {
        const int pp = (hw + cand - 1) / cand;
        const size_t need = static_cast<size_t>(pp) * ctot * 2 + static_cast<size_t>(R) * ctot * 4;
        if (need > kMaxSmem || (cand - 1) * pp >= hw) return false;   // does not fit / would leave an empty run
        if (!allow_small_runs && pp < 2 * R && cand > 1) return false;  // every pixel lane should get two pixels
        if (cand > 8) {  // non-portable size: ask the driver whether such a cluster can be co-scheduled at all
          if (max16 <= 0) return false;
          cudaLaunchConfig_t probe = {};
          probe.gridDim = dim3(cand * n_img), probe.blockDim = dim3(vpp * R), probe.dynamicSmemBytes = need;
          cudaLaunchAttribute pa[1];
          pa[0].id = cudaLaunchAttributeClusterDimension;
          pa[0].val.clusterDim.x = cand, pa[0].val.clusterDim.y = 1, pa[0].val.clusterDim.z = 1;
          probe.attrs = pa, probe.numAttrs = 1;
          int n_clusters = 0;
          const bool ok = cudaOccupancyMaxActiveClusters(&n_clusters, GnKernels<F16>::rows, &probe) == cudaSuccess && n_clusters >= 1;
          cudaGetLastError();
          if (!ok) return false;
        }
        cpi = cand, ppc = pp, smem = need;
        return true;
      };
      const char* cenv = getenv("MDB_GN_ROWS_CLUSTER");  // experiment knob: try this cluster size first
      const int forced = cenv ? atoi(cenv) : 0;
      bool found = forced >= 1 && forced <= 16 && try_cluster(forced, true);
      for (int cand = 8; cand >= 1 && !found; cand /= 2) found = try_cluster(cand, false);
      if (!found && (mode == 1 || img_bytes >= MDB_GN_ROWS_MIN_BYTES_C16)) found = try_cluster(16, true);
      if (cpi > 0) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cpi * n_img), cfg.blockDim = dim3(vpp * R), cfg.dynamicSmemBytes = smem, cfg.stream = st;
        cudaLaunchAttribute la[2];
        la[0].id = cudaLaunchAttributeClusterDimension;
        la[0].val.clusterDim.x = cpi, la[0].val.clusterDim.y = 1, la[0].val.clusterDim.z = 1;
        add_pdl_attr(cfg, la, 1);
        cudaError_t le = cudaLaunchKernelEx(&cfg, GnKernels<F16>::rows, x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta,
                                            silu, out, ldo, vpp, R, cpi, ppc);
        if (le != cudaSuccess) return set_error(MDB_ERR_CUDA, "gn_rows_kernel launch: %s", cudaGetErrorString(le));
        MDB_CHECK_LAUNCH("gn_rows_kernel");
        return MDB_OK;
      }
    }
  }
  if (((ctot / groups) & 1) == 0 && (c0 & 1) == 0 && !getenv("MDB_GN_TWO_KERNEL")) {
    const int pp = ctot / groups / 2;
    const long long units = static_cast<long long>(hw) * pp;
    const uint32_t inv_pp = static_cast<uint32_t>((0x100000000ULL + pp - 1) / pp);  // ceil(2^32 / pp)
    if (units * pp >= 0xffffffffLL) return set_error(MDB_ERR_UNSUPPORTED, "mdb_groupnorm: tensor too large");
    const size_t slab_bytes = static_cast<size_t>(units) * 4;
    if (slab_bytes <= 96 * 1024) {
      static bool attr = false;
      if (!attr) {
        cudaFuncSetAttribute(gn_fused_kernel<true, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        attr = true;
      }
      launch_pdl(gn_fused_kernel<true, F16>, dim3(groups, n_img), dim3(256), slab_bytes, st, x0, c0, ld0, x1, c1, ld1, hw,
                 groups, eps, gamma, beta, silu, out, ldo, inv_pp);
    } else {
      gn_fused_kernel<false, F16><<<dim3(groups, n_img), 256, 0, st>>>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta,
                                                                       silu, out, ldo, inv_pp);
    }
    MDB_CHECK_LAUNCH("gn_fused_kernel");
    return MDB_OK;
  }
  cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(float) * 2 * n_img * groups, st);
  if (e != cudaSuccess) return set_error(MDB_ERR_CUDA, "mdb_groupnorm memset: %s", cudaGetErrorString(e));
  const int vpp = ctot / 8;
  int R = 512 / vpp;
  if (R < 1) R = 1;
  if (R > 16) R = 16;
  const int threads = vpp * R;  // <= 512
  // enough CTAs to fill the machine: ~4 per SM over all images
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  int chunks = (sms * 4 + n_img - 1) / n_img;
  int pix_per_cta = (hw + chunks - 1) / chunks;
  if (pix_per_cta < R) pix_per_cta = R;
  chunks = (hw + pix_per_cta - 1) / pix_per_cta;
  const size_t smem = sizeof(float) * 2 * ctot;
  GnKernels<F16>::stats<<<dim3(chunks, n_img), threads, smem, st>>>(x0, c0, ld0, x1, c1, ld1, hw, groups, vpp, R, pix_per_cta,
                                                                   stats_ws);
  MDB_CHECK_LAUNCH("gn_stats_kernel");
  GnKernels<F16>::apply<<<dim3(chunks, n_img), 256, smem, st>>>(x0, c0, ld0, x1, c1, ld1, hw, groups, eps, gamma, beta, silu,
                                                                 stats_ws, out, ldo, pix_per_cta);
  MDB_CHECK_LAUNCH("gn_apply_kernel");
  return MDB_OK;
}

}  // namespace

extern "C" int mdb_groupnorm(const void* x0, int c0, int ld0, const void* x1, int c1, int ld1, int n_img, int hw,
                             int groups, float eps, const float* gamma, const float* beta, int silu, void* out, int ldo,
                             float* stats_ws, void* stream) {
  return groupnorm<false>(x0, c0, ld0, x1, c1, ld1, n_img, hw, groups, eps, gamma, beta, silu, out, ldo, stats_ws, stream);
}

extern "C" int mdb_groupnorm_f16(const void* x0, int c0, int ld0, const void* x1, int c1, int ld1, int n_img, int hw,
                                 int groups, float eps, const float* gamma, const float* beta, int silu, void* out, int ldo,
                                 float* stats_ws, void* stream) {
  return groupnorm<true>(x0, c0, ld0, x1, c1, ld1, n_img, hw, groups, eps, gamma, beta, silu, out, ldo, stats_ws, stream);
}

extern "C" int mdb_layernorm(const void* x, long long rows, int c, int ldx, const float* gamma, const float* beta,
                             float eps, void* out, int ldo, void* stream) {
  using namespace mdb;
  if (!x || !out || !gamma || !beta) return set_error(MDB_ERR_INVALID, "mdb_layernorm: null pointer");
  if (c % 8 || ldx % 8 || ldo % 8 || c > 8 * 32 * 8)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_layernorm: c must be a multiple of 8 and <= 2048 (c=%d)", c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int warps = 8;
  const unsigned blocks = static_cast<unsigned>((rows + warps - 1) / warps);
  const int nvec = c / 8;
  const __nv_bfloat16* xp = static_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* op = static_cast<__nv_bfloat16*>(out);
  if (nvec <= 64)
    launch_pdl(layernorm_kernel<2>, dim3(blocks), dim3(warps * 32), 0, st, xp, rows, c, ldx, gamma, beta, eps, op, ldo);
  else if (nvec <= 160)
    launch_pdl(layernorm_kernel<5>, dim3(blocks), dim3(warps * 32), 0, st, xp, rows, c, ldx, gamma, beta, eps, op, ldo);
  else
    launch_pdl(layernorm_kernel<8>, dim3(blocks), dim3(warps * 32), 0, st, xp, rows, c, ldx, gamma, beta, eps, op, ldo);
  MDB_CHECK_LAUNCH("layernorm_kernel");
  return MDB_OK;
}

// ---------------------------------------------------------------- row softmax (single-head VAE attention scores)
namespace {
// one warp per row: out[r, j] = exp(s[r, j] - max_r) / sum_r for j < cols, 0 for cols <= j < cols_out (bf16, or f16 with
// F16: an fp16 VAE)
template <bool F16>
__device__ __forceinline__ void softmax_rows(const float* __restrict__ s, int lds, long long rows, int cols,
                                             typename mdb::Act<F16>::T* __restrict__ out, int ldo, int cols_out) {
  using A = mdb::Act<F16>;
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* sr = s + row * lds;
  float mx = -INFINITY;
  for (int j = lane; j < cols; j += 32) mx = fmaxf(mx, sr[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < cols; j += 32) sum += __expf(sr[j] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  typename A::T* orow = out + row * ldo;
  for (int j = lane; j < cols_out; j += 32) orow[j] = A::from_float(j < cols ? __expf(sr[j] - mx) * inv : 0.f);
}
__global__ void softmax_rows_kernel(const float* __restrict__ s, int lds, long long rows, int cols,
                                    __nv_bfloat16* __restrict__ out, int ldo, int cols_out) {
  softmax_rows<false>(s, lds, rows, cols, out, ldo, cols_out);
}
__global__ void softmax_rows_f16_kernel(const float* __restrict__ s, int lds, long long rows, int cols,
                                        __half* __restrict__ out, int ldo, int cols_out) {
  softmax_rows<true>(s, lds, rows, cols, out, ldo, cols_out);
}

template <bool F16>
int softmax_rows_launch(const float* s, int lds, long long rows, int cols, void* out, int ldo, int cols_out, void* stream) {
  if (!s || !out) return mdb::set_error(MDB_ERR_INVALID, "mdb_softmax_rows: null pointer");
  if (rows <= 0 || cols <= 0 || cols_out < cols || lds < cols || ldo < cols_out)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_softmax_rows: bad shape");
  const int threads = 256;
  const long long blocks = (rows * 32 + threads - 1) / threads;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if constexpr (F16)
    softmax_rows_f16_kernel<<<static_cast<unsigned>(blocks), threads, 0, st>>>(s, lds, rows, cols, static_cast<__half*>(out),
                                                                               ldo, cols_out);
  else
    softmax_rows_kernel<<<static_cast<unsigned>(blocks), threads, 0, st>>>(s, lds, rows, cols,
                                                                           static_cast<__nv_bfloat16*>(out), ldo, cols_out);
  MDB_CHECK_LAUNCH("softmax_rows_kernel");
  return MDB_OK;
}
}  // namespace

extern "C" int mdb_softmax_rows(const float* s, int lds, long long rows, int cols, void* out, int ldo, int cols_out,
                                void* stream) {
  return softmax_rows_launch<false>(s, lds, rows, cols, out, ldo, cols_out, stream);
}

extern "C" int mdb_softmax_rows_f16(const float* s, int lds, long long rows, int cols, void* out, int ldo, int cols_out,
                                    void* stream) {
  return softmax_rows_launch<true>(s, lds, rows, cols, out, ldo, cols_out, stream);
}
