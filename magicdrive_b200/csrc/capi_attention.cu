// Fused multi-head attention forward (flash-style, online softmax in fp32) on wgmma + TMA: C-ABI launchers.
//
// Layout: q/out [B, Lq, heads*D] (row strides ldq/ldo), k/v [Bkv, Lk, heads*D] (ldk/ldv): exactly what the fused
// QKV projection GEMM writes, so no head transpose is ever materialised.  With n_sets == 2 the kernel runs two
// independent softmaxes against two KV batches and writes their sum: the cross-view "add" mode of
// BasicMultiviewTransformerBlock (magicdrive/networks/blocks.py:112-121, 213-217).  K/V may be spread over up to three
// buffers (mdb_attention_multi): in view-sharded runs the neighbour views' K/V are read in place from the ring-neighbour
// GPUs' buffers through NVLink peer memory (the tensor maps simply point at peer-mapped addresses).
// mdb_attention_causal is the CLIP text encoder's masked self-attention (one set, one source, lq == lk).
// Kernel: attention_wgmma.cuh.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdlib.h>
#include <string.h>

#include "../../include/magicdrive_b200.h"
#define MDB_NEED_TENSORMAP
#include "common_host.h"
#include "attention_wgmma.cuh"

namespace {

// [B, L, heads*D] (row stride ld) as a 4-D map (d, head, token, batch); box = (64, 1, rows, 1): the head dim is
// zero-padded to 64-wide chunks by TMA out-of-bounds fill, rows beyond L are zero-filled too.
bool make_qkv_map(CUtensorMap* m, const void* ptr, int d, int heads, int l, int b, int ld, int rows) {
  mdb::EncodeTiledFn enc = mdb::get_encode();
  if (!enc) return false;
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)heads, (cuuint64_t)l, (cuuint64_t)b};
  cuuint64_t strides[3] = {(cuuint64_t)d * 2, (cuuint64_t)ld * 2, (cuuint64_t)l * ld * 2};
  cuuint32_t box[4] = {64u, 1u, (cuuint32_t)rows, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct KvSources {
  const void* k[mdb::ATT_MAX_SRC];
  const void* v[mdb::ATT_MAX_SRC];
  int ldk[mdb::ATT_MAX_SRC], ldv[mdb::ATT_MAX_SRC], b_kv[mdb::ATT_MAX_SRC];
  int n;
};

bool make_kv_maps(mdb::AttnKvMaps* m, const KvSources& s, int d, int heads, int lk, int rows) {
  for (int i = 0; i < mdb::ATT_MAX_SRC; ++i) {
    const int j = i < s.n ? i : 0;  // unused slots alias source 0
    if (!make_qkv_map(&m->k[i], s.k[j], d, heads, lk, s.b_kv[j], s.ldk[j], rows) ||
        !make_qkv_map(&m->v[i], s.v[j], d, heads, lk, s.b_kv[j], s.ldv[j], rows))
      return false;
  }
  return true;
}

int attn_num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

// Query tiles per CTA walk (AttnParams::q_step) when one K/V tile covers all keys: one CTA per SM, each keeping its K/V tile
// and walking ~nq / gx query tiles.  0 = one tile per CTA.  MDB_ATTN_MULTIQ=0 disables it.
int multi_q_step(int b, int heads, int lq, int lk, int n_sets, int bn) {
  if (lk > bn || n_sets != 1) return 0;
  const char* e = getenv("MDB_ATTN_MULTIQ");
  if (e && e[0] == '0') return 0;
  const int nq = (lq + mdb::ATT_BM - 1) / mdb::ATT_BM;
  const long long per_tile_ctas = static_cast<long long>(b) * heads;
  const long long slots = attn_num_sms();
  if (per_tile_ctas * nq <= slots) return 0;  // everything is co-resident anyway
  long long gx = slots / per_tile_ctas;
  if (gx < 1) gx = 1;
  if (gx >= nq) return 0;
  return static_cast<int>(gx);
}

template <int D, int BN_, bool CAUSAL>
int launch_attention(const void* q, int ldq, const KvSources& src, void* out, int ldo, int b, int heads, int lq, int lk,
                     const int* kv_index, int n_sets, float scale, cudaStream_t st) {
  using Cfg = mdb::AttnCfg<D, BN_>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(mdb::attention_wgmma_kernel<D, BN_, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return mdb::set_error(MDB_ERR_CUDA, "attention_wgmma_kernel smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  CUtensorMap tq;
  mdb::AttnKvMaps kvm;
  if (!make_qkv_map(&tq, q, D, heads, lq, b, ldq, mdb::ATT_BM) || !make_kv_maps(&kvm, src, D, heads, lk, Cfg::BN))
    return mdb::set_error(MDB_ERR_CUDA, "mdb_attention: cuTensorMapEncodeTiled failed (d=%d heads=%d lq=%d lk=%d)", D, heads, lq, lk);
  mdb::AttnParams p;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo, p.lq = lq, p.lk = lk, p.kv_index = kv_index, p.n_sets = n_sets, p.n_src = src.n;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.q_step = multi_q_step(b, heads, lq, lk, n_sets, Cfg::BN);
  dim3 grid(p.q_step > 0 ? p.q_step : (lq + mdb::ATT_BM - 1) / mdb::ATT_BM, heads, b);
  cudaError_t le = mdb::launch_pdl(mdb::attention_wgmma_kernel<D, BN_, CAUSAL>, grid, dim3(Cfg::kThreads), Cfg::kSmemBytes, st, tq, kvm, p);
  if (le != cudaSuccess) return mdb::set_error(MDB_ERR_CUDA, "attention_wgmma_kernel launch: %s", cudaGetErrorString(le));
  cudaError_t e2 = cudaGetLastError();
  if (e2 != cudaSuccess) return mdb::set_error(MDB_ERR_CUDA, "attention_wgmma_kernel: %s", cudaGetErrorString(e2));
  return MDB_OK;
}

template <int BN_, bool CAUSAL>
int attention_dispatch_bn(const void* q, int ldq, const KvSources& src, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                          const int* kv_index, int n_sets, float scale, cudaStream_t st) {
  switch (d) {
    case 32: return launch_attention<32, BN_, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, kv_index, n_sets, scale, st);
    case 40: return launch_attention<40, BN_, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, kv_index, n_sets, scale, st);
    case 64: return launch_attention<64, BN_, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, kv_index, n_sets, scale, st);
    case 80: return launch_attention<80, BN_, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, kv_index, n_sets, scale, st);
    case 160: return launch_attention<160, BN_, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, kv_index, n_sets, scale, st);
    default: return mdb::set_error(MDB_ERR_UNSUPPORTED, "mdb_attention: head dim %d not instantiated (32, 40, 64, 80, 160)", d);
  }
}

// Key-tile width (A/B switch, read per call): MDB_ATTN_KERNEL = tc2 (default: 128 keys for head dims <= 64, 64 above) |
// tc2d (64-key tiles: smaller S fragment, deeper K/V ring) | tc (128-key tiles for every head dim).
template <bool CAUSAL = false>
int attention_dispatch(const void* q, int ldq, const KvSources& src, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                       const int* kv_index, int n_sets, float scale, cudaStream_t st) {
  const char* e = getenv("MDB_ATTN_KERNEL");
  if (e && !strcmp(e, "tc2d")) return attention_dispatch_bn<64, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, d, kv_index, n_sets, scale, st);
  if (e && !strcmp(e, "tc")) return attention_dispatch_bn<128, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, d, kv_index, n_sets, scale, st);
  if (e && *e && strcmp(e, "tc2"))
    return mdb::set_error(MDB_ERR_INVALID, "mdb_attention: MDB_ATTN_KERNEL must be tc2, tc2d or tc (got %s)", e);
  return attention_dispatch_bn<0, CAUSAL>(q, ldq, src, out, ldo, b, heads, lq, lk, d, kv_index, n_sets, scale, st);
}

}  // namespace

extern "C" int mdb_attention_multi(const void* q, int ldq, int n_src, const void* const* k, const int* ldk, const void* const* v,
                                   const int* ldv, const int* b_kv, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                                   const int* kv_index, int n_sets, float scale, void* stream) {
  using namespace mdb;
  if (!q || !k || !v || !ldk || !ldv || !b_kv || !out) return set_error(MDB_ERR_INVALID, "mdb_attention: null pointer");
  if (n_src < 1 || n_src > ATT_MAX_SRC) return set_error(MDB_ERR_INVALID, "mdb_attention: 1..%d K/V sources", ATT_MAX_SRC);
  if (n_sets < 1 || n_sets > 2 || (n_sets == 2 && !kv_index))
    return set_error(MDB_ERR_INVALID, "mdb_attention: n_sets must be 1 or 2 (2 needs kv_index)");
  if (scale <= 0.f) return set_error(MDB_ERR_INVALID, "mdb_attention: scale must be positive");
  if (lq <= 0 || lk <= 0 || b <= 0 || heads <= 0) return set_error(MDB_ERR_INVALID, "mdb_attention: bad shape");
  if (ldq % 8 || ldo % 8) return set_error(MDB_ERR_UNSUPPORTED, "mdb_attention: strides must be multiples of 8");
  KvSources src;
  src.n = n_src;
  for (int i = 0; i < n_src; ++i) {
    if (!k[i] || !v[i] || b_kv[i] <= 0) return set_error(MDB_ERR_INVALID, "mdb_attention: bad K/V source %d", i);
    if (ldk[i] % 8 || ldv[i] % 8) return set_error(MDB_ERR_UNSUPPORTED, "mdb_attention: strides must be multiples of 8");
    src.k[i] = k[i], src.v[i] = v[i], src.ldk[i] = ldk[i], src.ldv[i] = ldv[i], src.b_kv[i] = b_kv[i];
  }
  if (!kv_index && (n_src != 1 || b_kv[0] != b)) return set_error(MDB_ERR_INVALID, "mdb_attention: b_kv != b or several sources need kv_index");
  return attention_dispatch(q, ldq, src, out, ldo, b, heads, lq, lk, d, kv_index, n_sets, scale, static_cast<cudaStream_t>(stream));
}

extern "C" int mdb_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int b,
                             int b_kv, int heads, int lq, int lk, int d, const int* kv_index, int n_sets, float scale,
                             void* stream) {
  return mdb_attention_multi(q, ldq, 1, &k, &ldk, &v, &ldv, &b_kv, out, ldo, b, heads, lq, lk, d, kv_index, n_sets, scale, stream);
}

extern "C" int mdb_attention_causal(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo,
                                    int b, int heads, int lq, int lk, int d, float scale, void* stream) {
  using namespace mdb;
  if (!q || !k || !v || !out) return set_error(MDB_ERR_INVALID, "mdb_attention_causal: null pointer");
  if (lq != lk) return set_error(MDB_ERR_INVALID, "mdb_attention_causal: lq (%d) must equal lk (%d)", lq, lk);
  if (scale <= 0.f) return set_error(MDB_ERR_INVALID, "mdb_attention_causal: scale must be positive");
  if (lq <= 0 || b <= 0 || heads <= 0) return set_error(MDB_ERR_INVALID, "mdb_attention_causal: bad shape");
  if (ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) return set_error(MDB_ERR_UNSUPPORTED, "mdb_attention_causal: strides must be multiples of 8");
  KvSources src;
  src.n = 1;
  src.k[0] = k, src.v[0] = v, src.ldk[0] = ldk, src.ldv[0] = ldv, src.b_kv[0] = b;
  return attention_dispatch<true>(q, ldq, src, out, ldo, b, heads, lq, lk, d, nullptr, 1, scale, static_cast<cudaStream_t>(stream));
}
