// CLIP text encoder input: token + position embedding (transformers models/clip/modeling_clip.py CLIPTextEmbeddings.forward,
// called from CLIPTextTransformer.forward), written as the bf16 residual stream together with the row statistics that the
// first layer's folded layer_norm1 consumes (mdb_gemm_desc.ln_stats with ln_parts = 1).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdint.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"

namespace {

// One warp per token row; each lane moves 8 bf16 (16 bytes) at a time.
__global__ void clip_embed_kernel(const void* __restrict__ ids, int ids_are_i64, long long rows, int len,
                                  const __nv_bfloat16* __restrict__ tok, int vocab, const __nv_bfloat16* __restrict__ pos,
                                  int dim, __nv_bfloat16* __restrict__ out, int ldo, float* __restrict__ stats) {
  mdb::pdl_wait();
  mdb::pdl_launch_dependents();
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long id = ids_are_i64 ? static_cast<const long long*>(ids)[row] : static_cast<const int*>(ids)[row];
  const int p = static_cast<int>(row % len);
  __nv_bfloat16* orow = out + row * ldo;
  if (id < 0 || id >= vocab) {  // never used as an address: the row and its statistics become NaN
    const __nv_bfloat16 nan = __float2bfloat16_rn(__int_as_float(0x7fc00000));
    for (int c = lane; c < dim; c += 32) orow[c] = nan;
    if (lane == 0) reinterpret_cast<float2*>(stats)[row] = make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
    return;
  }
  const __nv_bfloat16* trow = tok + id * dim;
  const __nv_bfloat16* prow = pos + static_cast<long long>(p) * dim;
  float s = 0.f, ss = 0.f;
  for (int c = 8 * lane; c < dim; c += 256) {
    const uint4 tv = *reinterpret_cast<const uint4*>(trow + c);
    const uint4 pv = *reinterpret_cast<const uint4*>(prow + c);
    const __nv_bfloat162* t2 = reinterpret_cast<const __nv_bfloat162*>(&tv);
    const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&pv);
    uint4 ov;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 a = __bfloat1622float2(t2[i]), b = __bfloat1622float2(p2[i]);
      o2[i] = __floats2bfloat162_rn(a.x + b.x, a.y + b.y);  // the fp32 sum rounded once, like torch's bf16 add
      const float2 r = __bfloat1622float2(o2[i]);            // statistics of the values stored
      s += r.x + r.y;
      ss = fmaf(r.x, r.x, fmaf(r.y, r.y, ss));
    }
    *reinterpret_cast<uint4*>(orow + c) = ov;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) reinterpret_cast<float2*>(stats)[row] = make_float2(s, ss);
}

}  // namespace

extern "C" int mdb_clip_embed(const void* ids, int ids_are_i64, int n_seq, int len, const void* tok_table_bf16, int vocab,
                              const void* pos_table_bf16, int dim, void* out_bf16, int ldo, float* stats_out, void* stream) {
  using namespace mdb;
  if (!ids || !tok_table_bf16 || !pos_table_bf16 || !out_bf16 || !stats_out)
    return set_error(MDB_ERR_INVALID, "mdb_clip_embed: null pointer");
  if (n_seq <= 0 || len <= 0 || vocab <= 0 || dim <= 0) return set_error(MDB_ERR_INVALID, "mdb_clip_embed: bad shape");
  if (dim % 8 || ldo % 8) return set_error(MDB_ERR_UNSUPPORTED, "mdb_clip_embed: dim and ldo must be multiples of 8");
  if ((reinterpret_cast<uintptr_t>(tok_table_bf16) | reinterpret_cast<uintptr_t>(pos_table_bf16) |
       reinterpret_cast<uintptr_t>(out_bf16) | reinterpret_cast<uintptr_t>(stats_out)) & 15)
    return set_error(MDB_ERR_INVALID, "mdb_clip_embed: pointers must be 16-byte aligned");
  const long long rows = static_cast<long long>(n_seq) * len;
  const int warps = 8;
  const unsigned blocks = static_cast<unsigned>((rows + warps - 1) / warps);
  cudaError_t e = launch_pdl(clip_embed_kernel, dim3(blocks), dim3(32 * warps), 0, static_cast<cudaStream_t>(stream), ids,
                             ids_are_i64, rows, len, static_cast<const __nv_bfloat16*>(tok_table_bf16), vocab,
                             static_cast<const __nv_bfloat16*>(pos_table_bf16), dim, static_cast<__nv_bfloat16*>(out_bf16), ldo,
                             stats_out);
  if (e != cudaSuccess) return set_error(MDB_ERR_CUDA, "clip_embed_kernel launch: %s", cudaGetErrorString(e));
  MDB_CHECK_LAUNCH("clip_embed_kernel");
  return MDB_OK;
}
