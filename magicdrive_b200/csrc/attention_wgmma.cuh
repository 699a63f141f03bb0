// wgmma fused attention forward (flash-style, online softmax in fp32) for sm_90a.
//
//   per CTA: a 128-query tile of one (batch, head); loop over BN-key tiles of the (possibly neighbouring) batch's K/V:
//     S = Q K^T          wgmma SS  (Q, K tiles K-major in 128B-swizzled smem via 4-D TMA; d zero-padded to 64-chunks by
//                                   TMA out-of-bounds fill, so head dims 40 / 80 / 160 need no repacking)
//     P = exp2(S*c - m)  in registers: the fp32 S fragment is rescaled, exponentiated and packed to bf16 pairs that ARE the
//                        A fragment of the next product (no shared-memory round trip)
//     O = O*corr + P V   wgmma RS  (A = P from registers, B = V tile MN-major straight from the [keys, d] layout)
//   warp 8: TMA producer (Q per query tile, K/V ring of STAGES), warps 0..7: two consumer warpgroups of 64 query rows each.
//   n_sets > 1 runs the loop once per KV batch (cross-view neighbours) and sums the normalised outputs in slot order (each
//   rounded to bf16 first, like the reference's per-branch outputs).  A kv_index entry < 0 is an empty slot: the producer
//   loads nothing for it and the consumers skip it, both deciding from tiles_of(kv_entry(set), q0); a row with no present
//   set is written as zeros.
//   kv_len (optional, per query batch): keys at or beyond min(max(kv_len[b], 0), lk) take no weight and key tiles wholly past
//   that count are neither loaded nor walked (the "concat" mode with uneven neighbour counts).
//   Multi-Q mode (p.q_step > 0): the CTA walks the query tiles blockIdx.x, blockIdx.x + q_step, ... of its (batch, head);
//   with a single K/V tile (lk <= BN, one set: the text / camera / box cross-attention) that tile is loaded once.
//   KVRES (multi-Q launches with kv_len, one set): the key count is only known on the device, so each CTA decides from its
//   own batch's tile count: up to STAGES key tiles (the whole ring) are loaded once and stay resident while the CTA walks its
//   query tiles; a batch with more tiles streams them through the ring per query tile.  Either way the tiles are walked in
//   ascending order with the same width and the same updates, so the output is bitwise that of the lk = kv_len[b] launch.
//   CAUSAL (self-attention with lq == lk, one set): key j is visible to query i iff j <= i.  A query tile walks only the key
//   tiles up to the one holding its last row's diagonal (ascending, so tile 0, which holds key 0, always comes first), and
//   producer and consumers derive that count from the same q0.
#pragma once
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mdb {

constexpr int ATT_BM = 128;  // query rows per CTA tile

// K/V of a call may live in up to three buffers (this GPU's and, in view-sharded runs, the two ring-neighbour GPUs' buffers
// mapped through NVLink peer memory): kv_index entries are (source << 24) | batch index inside that source.
constexpr int ATT_MAX_SRC = 3;
struct AttnKvMaps {
  CUtensorMap k[ATT_MAX_SRC], v[ATT_MAX_SRC];
};

struct AttnParams {
  void* out;  // bf16, or f16 in the F16 instantiations
  int ldo;
  int lq, lk;
  const int* kv_index;  // [b, n_sets]: (source << 24) | batch, or < 0 for an empty slot; nullptr = batch b, one set
  int n_sets;
  const int* kv_len;    // [b] keys of each query batch's K/V (clamped to [0, lk]); nullptr = lk
  int n_src;
  float scale_log2;
  int q_step;  // > 0: query tiles per CTA walk stride (multi-Q mode); 0 = one query tile per CTA
};

// Key-tile width BN_ (0 = by head dim): 128 keys keep the S fragment at 64 registers per thread; head dims above 64 take
// 64-key tiles by default so that S, P and the O accumulator together stay within the register budget of 288-thread CTAs.
template <int D, int BN_ = 0>
struct AttnCfg {
  static constexpr int KD = (D + 63) / 64;        // 64-wide chunks of the head dim
  static constexpr int D16 = (D + 15) / 16 * 16;  // wgmma N of the PV product / k extent of QK^T
  static constexpr int BN = BN_ ? BN_ : ((D16 <= 64) ? 128 : 64);
  static constexpr int TILE_Q = ATT_BM * 128;     // bytes of one [128 rows][64 bf16] swizzled tile
  static constexpr int TILE_KV = BN * 128;
  static constexpr int SMEM_Q = KD * TILE_Q;
  static constexpr int STAGES_FIT = (232448 - 1024 - 256 - SMEM_Q) / (2 * KD * TILE_KV);  // K/V ring depth that fits
  static constexpr int STAGES = STAGES_FIT > 4 ? 4 : STAGES_FIT;
  static constexpr int SMEM_KV = STAGES * 2 * KD * TILE_KV;
  static constexpr int kSmemBytes = SMEM_Q + SMEM_KV + 1024 + 256;
  static constexpr int kConsumerWarps = 8;
  static constexpr int kThreads = 32 * kConsumerWarps + 32;
  static constexpr int SACC = BN / 2;   // S registers per thread
  static constexpr int OACC = D16 / 2;  // O registers per thread
  static_assert(STAGES >= 1 && kSmemBytes <= 232448, "shared memory");
};

// F16: f16 Q/K/V and output (fp16 models); P is packed to f16 pairs for the P V product, the softmax stays fp32.
template <int D, int BN_, bool CAUSAL = false, bool KVRES = false, bool F16 = false>
__global__ void __launch_bounds__(AttnCfg<D, BN_>::kThreads, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ AttnKvMaps kvm, const AttnParams p) {
  using Cfg = AttnCfg<D, BN_>;
  using A = Act<F16>;
  using Elt = typename A::T;
  constexpr int KD = Cfg::KD, D16 = Cfg::D16, BN = Cfg::BN, STAGES = Cfg::STAGES;
  constexpr int TILE_Q = Cfg::TILE_Q, TILE_KV = Cfg::TILE_KV;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smQ = smem;
  uint8_t* smK = smQ + Cfg::SMEM_Q;                   // [STAGES][KD][TILE_KV]
  uint8_t* smV = smK + STAGES * KD * TILE_KV;         // [STAGES][KD][TILE_KV]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smV + STAGES * KD * TILE_KV);
  uint64_t* q_full = bars;               // TMA -> consumers: Q tile landed
  uint64_t* q_empty = bars + 1;          // consumers (8 warps) -> TMA: Q tile no longer read
  uint64_t* kv_full = bars + 2;          // [STAGES]
  uint64_t* kv_empty = bars + 2 + STAGES;  // [STAGES] (8 warps)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.z, head = blockIdx.y;
  const int nq = (p.lq + ATT_BM - 1) / ATT_BM;
  const int q_step = p.q_step > 0 ? p.q_step : nq;
  const int n_own = (nq - static_cast<int>(blockIdx.x) + q_step - 1) / q_step;  // query tiles of this CTA
  auto q0_of = [&](int o) { return (static_cast<int>(blockIdx.x) + o * q_step) * ATT_BM; };

  if (warp == Cfg::kConsumerWarps && lane == 0) {
    prefetch_tmap(&tmQ);
    for (int i = 0; i < p.n_src; ++i) {
      prefetch_tmap(&kvm.k[i]);
      prefetch_tmap(&kvm.v[i]);
    }
    mbar_init(q_full, 1);
    mbar_init(q_empty, Cfg::kConsumerWarps);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], Cfg::kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");  // PDL: prologue above overlapped the predecessor's tail
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // kv_index / kv_len may be written by the predecessor kernel: read only after the PDL wait
  const int lkb = p.kv_len ? min(max(p.kv_len[b], 0), p.lk) : p.lk;  // keys of this batch; the maps never go past lk
  const int ntiles = (lkb + BN - 1) / BN;
  static_assert(!(CAUSAL && KVRES), "resident key tiles: every query tile walks all of them");
  const bool kv_resident = (KVRES ? ntiles <= STAGES : ntiles == 1) && p.n_sets == 1 && n_own > 1;
  auto kv_entry = [&](int set) { return p.kv_index ? p.kv_index[b * p.n_sets + set] : b; };
  // key tiles the set with kv_index entry kve reads for the query tile starting at q0: none for an empty slot; causal tiles
  // stop at the one holding key min(q0 + ATT_BM, lq) - 1.  Producer and consumers both take their counts from here.
  auto tiles_of = [&](int kve, int q0) {
    return kve < 0 ? 0 : CAUSAL ? min(ntiles, (min(q0 + ATT_BM, p.lq) - 1) / BN + 1) : ntiles;
  };

  if (warp == Cfg::kConsumerWarps) {
    // =========================== TMA producer ===========================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int o = 0; o < n_own; ++o) {
        if (o > 0) mbar_wait(q_empty, static_cast<uint32_t>(o - 1) & 1u);
        mbar_arrive_expect_tx(q_full, KD * TILE_Q);
#pragma unroll
        for (int c = 0; c < KD; ++c) tma_load_4d(&tmQ, q_full, smQ + c * TILE_Q, c * 64, head, q0_of(o), b);
        if (kv_resident && o > 0) continue;
        for (int set = 0; set < p.n_sets; ++set) {
          const int kve = kv_entry(set);
          const int nt = tiles_of(kve, q0_of(o));
          if (nt == 0) continue;
          const int kvb = kve & 0xffffff;
          const CUtensorMap* km = &kvm.k[kve >> 24];
          const CUtensorMap* vm = &kvm.v[kve >> 24];
          for (int j = 0; j < nt; ++j) {
            mbar_wait(&kv_empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&kv_full[stage], 2 * KD * TILE_KV);
#pragma unroll
            for (int c = 0; c < KD; ++c) {
              tma_load_4d(km, &kv_full[stage], smK + (stage * KD + c) * TILE_KV, c * 64, head, j * BN, kvb);
              tma_load_4d(vm, &kv_full[stage], smV + (stage * KD + c) * TILE_KV, c * 64, head, j * BN, kvb);
            }
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
    return;
  }

  // =========================== consumers: softmax + both products ===========================
  const int wg = warp >> 2;
  const int q = lane & 3;
  const int rloc = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // this thread's query rows: rloc and rloc + 8 of the tile
  const float sc = p.scale_log2;
  int stage = 0;
  uint32_t phase = 0;
  for (int o = 0; o < n_own; ++o) {
    const int q0 = q0_of(o);
    mbar_wait(q_full, static_cast<uint32_t>(o) & 1u);
    bool wrote = false;  // a present set was stored to this query tile's rows (uniform over the CTA)
    for (int set = 0; set < p.n_sets; ++set) {
      const int nt = tiles_of(kv_entry(set), q0);
      if (nt == 0) continue;
      float oacc[Cfg::OACC];
#pragma unroll
      for (int i = 0; i < Cfg::OACC; ++i) oacc[i] = 0.f;
      float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
      for (int j = 0; j < nt; ++j) {
        const int st = kv_resident ? (KVRES ? j : 0) : stage;  // resident tile j sits in ring slot j
        mbar_wait(&kv_full[st], kv_resident ? 0u : phase);
        // ---- S = Q K^T
        float s[Cfg::SACC];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D16 / 16; ++k) {
          const int c = k / 4, kk = k % 4;
          const uint64_t adesc = make_sw128_kmajor_desc(smem_u32(smQ + c * TILE_Q + wg * (64 * 128))) + 2 * kk;
          const uint64_t bdesc = make_sw128_kmajor_desc(smem_u32(smK + (st * KD + c) * TILE_KV)) + 2 * kk;
          WgmmaSS<BN, F16>::run(s, adesc, bdesc, k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        // ---- keys past this batch's key count (past lk: zero-filled by TMA) take no weight
        const int kbase = j * BN;
        if (kbase + BN > lkb) {
#pragma unroll
          for (int g = 0; g < BN / 8; ++g)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (kbase + 8 * g + 2 * q + e >= lkb) s[4 * g + e] = s[4 * g + 2 + e] = -INFINITY;
        }
        // ---- causal: keys after the query row take no weight (only tiles that reach past the tile's first row)
        if constexpr (CAUSAL) {
          if (kbase + BN - 1 > q0 + rloc) {
#pragma unroll
            for (int g = 0; g < BN / 8; ++g)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  if (kbase + 8 * g + 2 * q + e > q0 + rloc + 8 * h) s[4 * g + 2 * h + e] = -INFINITY;
          }
        }
        // ---- online softmax (row max over the quad that shares a row)
        float corr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float mx = -INFINITY;
#pragma unroll
          for (int g = 0; g < BN / 8; ++g) mx = fmaxf(mx, fmaxf(s[4 * g + 2 * h], s[4 * g + 2 * h + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          // sc > 0; finite: key kbase is always valid (causal: key 0 of tile 0, walked first, is visible to every row)
          const float m_new = fmaxf(m[h], mx * sc);
          corr[h] = exp2f(m[h] - m_new);
          m[h] = m_new;
        }
        uint32_t pa[BN / 16][4];
        float rs[2] = {0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) {
#pragma unroll
          for (int r = 0; r < 4; ++r) {  // r: (row h = r & 1, column half r >> 1) of the 16-key A fragment
            const int h = r & 1;
            const int i0 = 8 * kk + 4 * (r >> 1) + 2 * h;
            const float p0 = exp2f(fmaf(s[i0], sc, -m[h]));
            const float p1 = exp2f(fmaf(s[i0 + 1], sc, -m[h]));
            rs[h] += p0 + p1;
            pa[kk][r] = A::pack(p0, p1);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) l[h] = l[h] * corr[h] + rs[h];
#pragma unroll
        for (int g = 0; g < D16 / 8; ++g) {
          oacc[4 * g] *= corr[0], oacc[4 * g + 1] *= corr[0];
          oacc[4 * g + 2] *= corr[1], oacc[4 * g + 3] *= corr[1];
        }
        // ---- O += P V
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) {
          const uint64_t bdesc = make_sw128_mnmajor_desc(smem_u32(smV + st * KD * TILE_KV), TILE_KV) + (2048u >> 4) * kk;
          WgmmaRSBmn<D16, F16>::run(oacc, pa[kk], bdesc, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (!kv_resident) {
          if (lane == 0) mbar_arrive(&kv_empty[stage]);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
      // ---- normalise and store this set
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      }
      const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int qrow = q0 + rloc + 8 * h;
        if (qrow >= p.lq) continue;
        Elt* orow = static_cast<Elt*>(p.out) + (static_cast<long long>(b) * p.lq + qrow) * p.ldo + head * D;
#pragma unroll
        for (int g = 0; g < D16 / 8; ++g) {
          const int col = 8 * g + 2 * q;
          if (col >= D) continue;
          float f0 = oacc[4 * g + 2 * h] * inv[h], f1 = oacc[4 * g + 2 * h + 1] * inv[h];
          if (wrote) {
            // every branch rounded to the storage type before the sum, like the reference's per-branch attention outputs
            const float2 pf = A::to_float2(*reinterpret_cast<const typename A::T2*>(orow + col));
            f0 = A::to_float(A::from_float(f0)) + pf.x;
            f1 = A::to_float(A::from_float(f1)) + pf.y;
          }
          *reinterpret_cast<uint32_t*>(orow + col) = A::pack(f0, f1);
        }
      }
      wrote = true;
    }
    if (!wrote) {  // no present set: the sum over no neighbours is zero
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int qrow = q0 + rloc + 8 * h;
        if (qrow >= p.lq) continue;
        Elt* orow = static_cast<Elt*>(p.out) + (static_cast<long long>(b) * p.lq + qrow) * p.ldo + head * D;
#pragma unroll
        for (int g = 0; g < D16 / 8; ++g)
          if (8 * g + 2 * q < D) *reinterpret_cast<uint32_t*>(orow + 8 * g + 2 * q) = 0u;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(q_empty);
  }
}

}  // namespace mdb
