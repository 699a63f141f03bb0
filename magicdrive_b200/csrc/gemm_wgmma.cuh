// Persistent warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a (operand scheme: gemm_tc.cuh).
//
// One CTA per SM loops over output tiles (m fastest, so concurrently running CTAs share the same weight tile in L2).
//   warp 8:     TMA producer (one lane): A tile + B tile per 64-wide K block into a ring of shared-memory stages; the ring
//               keeps flowing across tile boundaries, so the loads of tile i+1 overlap the epilogue of tile i.
//   CTAS = 2:   CTA pairs.  The two CTAs of a cluster compute consecutive M tiles against the same weight tile; each loads
//               its own A tile and HALF of the B tile, multicast into both CTAs' shared memory, which halves the L2 -> SM
//               weight traffic.  A stage is refilled only once the consumers of BOTH CTAs have released it (every
//               consumer warp arrives on the empty barrier of both CTAs).
//   warps 0..7: two consumer warpgroups, rows [0, 64) and [64, 128) of the 128-row M tile: wgmma m64 x BLOCK_N x k16 with
//               the fp32 accumulator in registers, then the epilogue straight from those registers.
// Epilogue (per element, fp32):  out = A_row * acc + ((bias_n + shift_img,n) * scale + B_row * colsum_n) [+ residual]
//   with A_row = scale, B_row = 0, or -- LayerNorm folded into this GEMM -- A_row = rstd * scale, B_row = -mean * rstd * scale
//   from the per-row partial sums the producer of A emitted; ReLU launches store max(0, out).  GEGLU tiles hold
//   [128 value | 128 gate] columns.  Split-K
//   tiles write fp32 partials instead (summed in split order by splitk_finalize_kernel).
#pragma once
#include "common_host.h"
#include "gemm_tc.cuh"
#include "ptx_cluster.cuh"
#include "wgmma.cuh"

namespace mdb {

template <int BLOCK_N, int CTAS>
struct WgGemmCfg {
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kBRows = BLOCK_N / CTAS;  // B rows each CTA loads (and multicasts)
  static constexpr int kBPartBytes = kBRows * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kStagesFit = (232448 - 1024 - kBarBytes) / kStageBytes;  // 227 KB of opt-in shared memory per block
  static constexpr int kStages = kStagesFit > 8 ? 8 : kStagesFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + kBarBytes;
  static constexpr int kConsumerWarps = 8;
  static constexpr int kThreads = 32 * kConsumerWarps + 32;
  static constexpr int kAcc = BLOCK_N / 2;  // fp32 accumulator registers per consumer thread
  static_assert(kStages >= 3, "pipeline too shallow");
  static_assert(kBPartBytes % 1024 == 0, "B stage parts must keep the 1024-byte swizzle alignment");
};

__device__ __forceinline__ float2 ldg_f2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// RELU: the ReLU epilogue (EPI_RELU) is compiled only into its own instantiations, so the others are the plain kernel.
// F16: f16 operands, residual and output (fp16 models) in place of bf16; the accumulator and the epilogue stay fp32.
template <int BLOCK_N, int CTAS, bool RELU = false, bool F16 = false>
__global__ void __launch_bounds__(WgGemmCfg<BLOCK_N, CTAS>::kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                  const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = WgGemmCfg<BLOCK_N, CTAS>;
  using A = Act<F16>;
  using Elt = typename A::T;
  constexpr bool PAIR = CTAS == 2;
  constexpr int STAGES = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;
  uint8_t* smB = smem + STAGES * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cb_total = p.cblocks0 + p.cblocks1;
  const int kb_total = p.taps_h * p.taps_w * cb_total;
  const int total_tiles = p.m_groups * p.n_tiles * p.splits;
  const int rank = PAIR ? static_cast<int>(cluster_ctarank()) : 0;
  const int first_tile = static_cast<int>(blockIdx.x) / CTAS, tile_step = static_cast<int>(gridDim.x) / CTAS;

  if (warp == Cfg::kConsumerWarps && lane == 0) {
    prefetch_tmap(&tmA0);
    prefetch_tmap(&tmA1);
    prefetch_tmap(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CTAS * Cfg::kConsumerWarps);  // one arrive per consumer warp of every CTA of the cluster
    }
    fence_barrier_init();
  }
  // a pair's peer multicasts into this CTA's barriers: both must be initialised before either producer starts
  if constexpr (PAIR) cluster_sync_all(); else __syncthreads();
  // everything above overlapped the predecessor's tail; from here on we read its outputs
  pdl_wait();
  pdl_launch_dependents();

  if (warp == Cfg::kConsumerWarps) {
    // =========================== TMA producer ===========================
    if (lane == 0) {
      const uint32_t tx_bytes = kABytes + Cfg::kBBytes;  // out-of-bounds rows are zero-filled and still counted
      const int hw_out = p.h_out * p.w_out;
      int stage = 0;
      uint32_t phase = 0;
      for (int t = first_tile; t < total_tiles; t += tile_step) {
        const int mt = (t % p.m_groups) * CTAS + rank;  // >= m_tiles for the second tile of an odd pair: all OOB, zero-filled
        const int rest = t / p.m_groups;
        const int nt = rest % p.n_tiles;
        const int z = rest / p.n_tiles;
        // im2col start: input position of the tile's first output pixel (the top-left filter tap)
        const int pix0 = mt * kBlockM;
        const int img0 = pix0 / hw_out;
        const int oh0 = (pix0 - img0 * hw_out) / p.w_out;
        const int ow0 = pix0 - img0 * hw_out - oh0 * p.w_out;
        const int wc = ow0 * p.stride - p.pad_w, hc = oh0 * p.stride - p.pad_h;
        const int n0 = nt * BLOCK_N;
        const int kb_begin = z * p.kb_per_split;
        const int kb_end = min(kb_total, kb_begin + p.kb_per_split);
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const int tap = kb / cb_total;
          const int cb = kb - tap * cb_total;
          const int r = tap / p.taps_w, s = tap - r * p.taps_w;
          mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
          const CUtensorMap* tmA = cb < p.cblocks0 ? &tmA0 : &tmA1;
          const int c = (cb < p.cblocks0 ? cb : cb - p.cblocks0) * kBlockK;
          if (p.im2col)
            tma_load_im2col_4d(tmA, &full_bar[stage], smA + stage * kABytes, c, wc, hc, img0, static_cast<uint16_t>(s),
                               static_cast<uint16_t>(r));
          else
            tma_load_2d(tmA, &full_bar[stage], smA + stage * kABytes, c, pix0);
          if constexpr (PAIR)
            tma_load_2d_multicast(&tmB, &full_bar[stage], smB + stage * Cfg::kBBytes + rank * Cfg::kBPartBytes, kb * kBlockK,
                                  n0 + rank * Cfg::kBRows, 0x3);
          else
            tma_load_2d(&tmB, &full_bar[stage], smB + stage * Cfg::kBBytes, kb * kBlockK, n0);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
  // =========================== consumers (warpgroups 0 and 1) ===========================
  const int wg = warp >> 2;
  const int q = lane & 3;
  const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows: row0 and row0 + 8
  const int hw_out = p.h_out * p.w_out;
  const long long pixels_total = static_cast<long long>(p.n_img) * p.h_out * p.w_out;
  const float scale = p.out_scale;
  int stage = 0;
  uint32_t phase = 0;
  const uint32_t peer = rank ^ 1;
  auto release = [&](int s) {  // this warp is done with stage s (its MMAs retired): free it in every CTA that fills it
    if (lane == 0) {
      mbar_arrive(&empty_bar[s]);
      if constexpr (PAIR) mbar_arrive_cluster_release(mapa_u32(smem_u32(&empty_bar[s]), peer));
    }
  };
  for (int t = first_tile; t < total_tiles; t += tile_step) {
    const int mt = (t % p.m_groups) * CTAS + rank;
    const int rest = t / p.m_groups;
    const int nt = rest % p.n_tiles;
    const int z = rest / p.n_tiles;
    const int n0 = nt * BLOCK_N;
    const int kb_begin = z * p.kb_per_split;
    const int nkb = min(kb_total, kb_begin + p.kb_per_split) - kb_begin;

    // ---- main loop: wgmma on stage i while the TMA fills the following ones; stage i-1 is released once its MMAs retired
    float acc[Cfg::kAcc];
#pragma unroll
    for (int i = 0; i < Cfg::kAcc; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      const uint64_t adesc = make_sw128_kmajor_desc(smem_u32(smA + stage * kABytes + wg * (64 * 128)));
      const uint64_t bdesc = make_sw128_kmajor_desc(smem_u32(smB + stage * Cfg::kBBytes));
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) WgmmaSS<BLOCK_N, F16>::run(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) release(prev);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    if (prev >= 0) release(prev);

    // ---- epilogue from registers
    int img[2];
    long long pix[2];
    bool ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int px = mt * kBlockM + row0 + 8 * h;
      img[h] = px / hw_out;
      pix[h] = px;
      ok[h] = pix[h] < pixels_total;
    }
    if (p.epi_mode == EPI_PARTIAL_F32) {
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        if (col >= p.n_out) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (ok[h])
            *reinterpret_cast<float2*>(p.partial + (static_cast<long long>(z) * pixels_total + pix[h]) * p.n_out + col) =
                make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
      continue;
    }
    float rowA[2] = {scale, scale}, rowB[2] = {0.f, 0.f};
    if (p.ln_stats != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!ok[h]) continue;
        const float2* sp = reinterpret_cast<const float2*>(p.ln_stats) + pix[h] * p.ln_parts;
        float s = 0.f, ss = 0.f;
        for (int j = 0; j < p.ln_parts; ++j) {
          const float2 v = __ldg(sp + j);
          s += v.x, ss += v.y;
        }
        const float mean = s * p.ln_inv_c;
        const float rstd = rsqrtf(fmaxf(ss * p.ln_inv_c - mean * mean, 0.f) + p.ln_eps);
        rowA[h] = rstd * scale;
        rowB[h] = -mean * rowA[h];
      }
    }
    const bool has_ln = p.ln_stats != nullptr;
    if (p.epi_mode == EPI_GEGLU) {
      constexpr int HALF = BLOCK_N / 2;
      const int on0 = nt * HALF;
      Elt* out = static_cast<Elt*>(p.out);
#pragma unroll
      for (int j = 0; j < HALF / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const float2 bv = p.bias ? ldg_f2(p.bias + n0 + c) : make_float2(0.f, 0.f);
        const float2 bg = p.bias ? ldg_f2(p.bias + n0 + HALF + c) : make_float2(0.f, 0.f);
        const float2 cv = has_ln ? ldg_f2(p.ln_colsum + n0 + c) : make_float2(0.f, 0.f);
        const float2 cg = has_ln ? ldg_f2(p.ln_colsum + n0 + HALF + c) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!ok[h]) continue;
          const float a0 = fmaf(rowA[h], acc[4 * j + 2 * h], fmaf(rowB[h], cv.x, bv.x * scale));
          const float a1 = fmaf(rowA[h], acc[4 * j + 2 * h + 1], fmaf(rowB[h], cv.y, bv.y * scale));
          const float g0 = fmaf(rowA[h], acc[4 * (j + HALF / 8) + 2 * h], fmaf(rowB[h], cg.x, bg.x * scale));
          const float g1 = fmaf(rowA[h], acc[4 * (j + HALF / 8) + 2 * h + 1], fmaf(rowB[h], cg.y, bg.y * scale));
          *reinterpret_cast<uint32_t*>(out + pix[h] * p.ldo + on0 + c) = A::pack(a0 * gelu_erf(g0), a1 * gelu_erf(g1));
        }
      }
      continue;
    }
    if (p.epi_mode == EPI_QUICK_GELU) {  // its own loop, so the linear epilogue below stays as it is: plain bf16 output
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        if (col >= p.n_out) continue;
        const float2 b = p.bias ? ldg_f2(p.bias + col) : make_float2(0.f, 0.f);
        const float2 cs = has_ln ? ldg_f2(p.ln_colsum + col) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!ok[h]) continue;
          const float v0 = fmaf(rowA[h], acc[4 * j + 2 * h], fmaf(rowB[h], cs.x, b.x * scale));
          const float v1 = fmaf(rowA[h], acc[4 * j + 2 * h + 1], fmaf(rowB[h], cs.y, b.y * scale));
          *reinterpret_cast<uint32_t*>(static_cast<Elt*>(p.out) + pix[h] * p.ldo + col) =
              A::pack(quick_gelu(v0), quick_gelu(v1));
        }
      }
      continue;
    }
    if constexpr (RELU) {  // its own loop too: plain bf16 output, the linear epilogue below is untouched
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        if (col >= p.n_out) continue;
        const float2 b = p.bias ? ldg_f2(p.bias + col) : make_float2(0.f, 0.f);
        const float2 cs = has_ln ? ldg_f2(p.ln_colsum + col) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!ok[h]) continue;
          const float v0 = fmaf(rowA[h], acc[4 * j + 2 * h], fmaf(rowB[h], cs.x, b.x * scale));
          const float v1 = fmaf(rowA[h], acc[4 * j + 2 * h + 1], fmaf(rowB[h], cs.y, b.y * scale));
          *reinterpret_cast<uint32_t*>(static_cast<Elt*>(p.out) + pix[h] * p.ldo + col) =
              A::pack(fmaxf(v0, 0.f), fmaxf(v1, 0.f));
        }
      }
      continue;
    }
    float st_s[2] = {0.f, 0.f}, st_ss[2] = {0.f, 0.f};
    // The residual may be the output buffer itself, so a residual load cannot move above an earlier output store: loaded
    // one element at a time, every element would wait out its own round trip to L2.  Each batch of RES_J 8-column groups
    // loads all its residual pairs first (the thread reads only the elements it then overwrites), so one round trip
    // serves the whole batch.
    constexpr int RES_J = BLOCK_N == 256 ? 1 : 4;  // 256 columns of accumulators leave no registers for more
#pragma unroll
    for (int jb = 0; jb < BLOCK_N / 8; jb += RES_J) {
      typename A::T2 res[RES_J][2];
      if (p.residual) {
#pragma unroll
        for (int jj = 0; jj < RES_J; ++jj) {
          const int col = n0 + 8 * (jb + jj) + 2 * q;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (col < p.n_out && ok[h])
              res[jj][h] = *reinterpret_cast<const typename A::T2*>(static_cast<const Elt*>(p.residual) + pix[h] * p.ldr + col);
        }
      }
#pragma unroll
      for (int jj = 0; jj < RES_J; ++jj) {
        const int j = jb + jj;
        const int col = n0 + 8 * j + 2 * q;
        if (col >= p.n_out) continue;
        const float2 b = p.bias ? ldg_f2(p.bias + col) : make_float2(0.f, 0.f);
        const float2 cs = has_ln ? ldg_f2(p.ln_colsum + col) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!ok[h]) continue;
          float2 cb = b;
          if (p.rowbias) {
            const float2 rb = ldg_f2(p.rowbias + static_cast<long long>(img[h]) * p.rowbias_ld + col);
            cb.x += rb.x, cb.y += rb.y;
          }
          float v0 = fmaf(rowA[h], acc[4 * j + 2 * h], fmaf(rowB[h], cs.x, cb.x * scale));
          float v1 = fmaf(rowA[h], acc[4 * j + 2 * h + 1], fmaf(rowB[h], cs.y, cb.y * scale));
          if (p.residual) {
            const float2 r = A::to_float2(res[jj][h]);
            v0 += r.x, v1 += r.y;
          }
          if (p.out_is_f32) {
            *reinterpret_cast<float2*>(static_cast<float*>(p.out) + pix[h] * p.ldo + col) = make_float2(v0, v1);
          } else {
            const uint32_t pk = A::pack(v0, v1);
            *reinterpret_cast<uint32_t*>(static_cast<Elt*>(p.out) + pix[h] * p.ldo + col) = pk;
            // the row statistics describe the values as stored: the consumer's folded LayerNorm multiplies these
            if constexpr (F16) {
              const float2 sv = A::to_float2(*reinterpret_cast<const typename A::T2*>(&pk));
              v0 = sv.x, v1 = sv.y;
            } else {
              v0 = __uint_as_float(pk << 16), v1 = __uint_as_float(pk & 0xffff0000u);
            }
          }
          st_s[h] += v0 + v1;
          st_ss[h] = fmaf(v0, v0, fmaf(v1, v1, st_ss[h]));
        }
      }
    }
    if (p.stats_out != nullptr) {
      // one (sum, sum sq) slot per (row, N tile): the four lanes of a quad hold the row's columns of this tile
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        st_s[h] += __shfl_xor_sync(0xffffffffu, st_s[h], 1);
        st_s[h] += __shfl_xor_sync(0xffffffffu, st_s[h], 2);
        st_ss[h] += __shfl_xor_sync(0xffffffffu, st_ss[h], 1);
        st_ss[h] += __shfl_xor_sync(0xffffffffu, st_ss[h], 2);
        if (q == 0 && ok[h])
          reinterpret_cast<float2*>(p.stats_out)[pix[h] * p.n_tiles + nt] = make_float2(st_s[h], st_ss[h]);
      }
    }
  }
  }
  // a pair's CTAs multicast into / arrive on each other's shared memory until the end: neither may exit before the other
  __syncwarp();
  if constexpr (PAIR) cluster_sync_all();
}

}  // namespace mdb
