// Map images and view mosaics (include/magicdrive_b200.h: mdb_render_bev_map, mdb_place_map_u8, mdb_concat_views_u8,
// mdb_m11_to_u8): the pixels of the reference's test-run images (magicdrive/misc/test_utils.py `run_one_batch`), equal
// byte for byte to its numpy / Pillow route.  oracle/map_visualizer.py is the same arithmetic in numpy.
//
// mdb_render_bev_map: runner/map_visualizer.py `render_static` / `render_dynamic` / the composite of `visualize_map`,
// one thread per map pixel.  Besides the colours it gathers, per map, the classes the legend names (`semantic_used`) and
// the first pixel where the reference raises, with one 64-bit OR or min per warp.
// mdb_place_map_u8: `Image.rotate(90)` of the square resized map (Transpose.ROTATE_90) and the legend pasted to its right
// or below, one thread per output pixel, every map of a batch in one launch.
// mdb_concat_views_u8: runner/img_utils.py `concat_6_views`, one thread per mosaic pixel.
// mdb_m11_to_u8: torchvision's to_pil_image(img_m11_to_01(x)) of [-1, 1] camera views.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxClasses = 64;  // semantic_used is a 64-bit class mask
constexpr int kMaxSide = 32767;
constexpr unsigned long long kNone = ~0ull;

// On the bits, so that this file's flush-to-zero build neither drops a denormal nor takes it for 0
__device__ __forceinline__ bool active(float v) { return (__float_as_uint(v) & 0x7fffffffu) != 0; }
__device__ __forceinline__ bool active(uint8_t v) { return v != 0; }
__device__ __forceinline__ bool binary(float v) { return !active(v) || __float_as_uint(v) == 0x3f800000u; }
__device__ __forceinline__ bool binary(uint8_t v) { return v <= 1; }

__device__ __forceinline__ unsigned long long warp_or(unsigned long long v) {
  const unsigned lo = __reduce_or_sync(0xffffffffu, static_cast<unsigned>(v));
  const unsigned hi = __reduce_or_sync(0xffffffffu, static_cast<unsigned>(v >> 32));
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}

__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// info[m] = {semantic_used, status (bit 0: a value not 0 / 1), first rank error, first colour error}.  render_static
// raises at the first pixel, in raster order, where get_color_by_priority fails: ValueError when an active class has no
// STATIC_PRIORITY rank (the first such channel), else KeyError when the class it chooses has no colour.  It does so for
// every pixel with a static class set, whether or not a dynamic layer covers it.  Each error word is the smallest
// (pixel << 6 | class) where that error arises, all ones where it never does.
template <typename T>
__global__ void __launch_bounds__(kThreads) render_bev_map_kernel(const T* __restrict__ maps, int channels, int hw,
                                                                  int n_static, int n_dynamic,
                                                                  const int* __restrict__ priority,
                                                                  const uint8_t* __restrict__ colors,
                                                                  uint8_t* __restrict__ out,
                                                                  unsigned long long* __restrict__ info) {
  __shared__ int s_prio[kMaxClasses];
  __shared__ uint8_t s_col[kMaxClasses][4];
  for (int i = threadIdx.x; i < n_static + n_dynamic; i += blockDim.x) {
    s_prio[i] = i < n_static ? priority[i] : 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) s_col[i][c] = colors[i * 4 + c];
  }
  __syncthreads();
  const int m = blockIdx.y;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  unsigned long long used = 0, status = 0, no_rank = kNone, no_colour = kNone;
  if (p < hw) {
    const T* src = maps + static_cast<long long>(m) * channels * hw + p;
    // get_color_by_priority: the first maximum of the STATIC_PRIORITY ranks of the active classes
    int chosen = -1, best = INT_MIN;
    for (int c = 0; c < n_static; ++c) {
      const T v = src[static_cast<long long>(c) * hw];
      if (!binary(v)) status = 1;
      if (active(v)) {
        used |= 1ull << c;
        if (s_prio[c] < 0 && no_rank == kNone) no_rank = static_cast<unsigned long long>(p) << 6 | c;
        if (s_prio[c] > best) best = s_prio[c], chosen = c;
      }
    }
    if (chosen >= 0 && !s_col[chosen][3]) no_colour = static_cast<unsigned long long>(p) << 6 | chosen;
    // argmax over the dynamic layers: on a binary map the first layer set, 0 where none is
    int dyn = -1;
    for (int c = 0; c < n_dynamic; ++c) {
      const T v = src[static_cast<long long>(n_static + c) * hw];
      if (!binary(v)) status = 1;
      if (dyn < 0 && active(v)) dyn = c;
    }
    // np.unique(semantic_map) takes the argmax at every pixel, so the first object class is named wherever none is set
    if (n_dynamic > 0) used |= 1ull << (n_static + max(dyn, 0));
    uint8_t rgb[3] = {200, 200, 200};  // COLORS["nothing"]
    const int k = dyn >= 0 ? n_static + dyn : chosen;
    if (k >= 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) rgb[c] = s_col[k][c];
    }
    uint8_t* o = out + (static_cast<long long>(m) * hw + p) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = rgb[c];
  }
  used = warp_or(used);
  status = warp_or(status);
  no_rank = warp_min(no_rank);
  no_colour = warp_min(no_colour);
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* inf = info + m * 4;
    if (used) atomicOr(inf, used);
    if (status) atomicOr(inf + 1, status);
    if (no_rank != kNone) atomicMin(inf + 2, no_rank);
    if (no_colour != kNone) atomicMin(inf + 3, no_colour);
  }
}

// desc[m] = {legend address, lh, lw, right (1) or below (0), byte offset of map m's image in out}
__global__ void __launch_bounds__(kThreads) place_map_kernel(const uint8_t* __restrict__ resized, int s,
                                                             const long long* __restrict__ desc,
                                                             uint8_t* __restrict__ out) {
  const int m = blockIdx.y;
  const long long* d = desc + m * 5;
  const uint8_t* legend = reinterpret_cast<const uint8_t*>(d[0]);
  const int lh = static_cast<int>(d[1]), lw = static_cast<int>(d[2]);
  const bool right = d[3] != 0;
  const int ow = right ? s + lw : s;
  const long long n = static_cast<long long>(right ? s : s + lh) * ow;
  const long long p = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (p >= n) return;
  const int y = static_cast<int>(p / ow), x = static_cast<int>(p % ow);
  const uint8_t* src;
  if (y < s && x < s)
    src = resized + ((static_cast<long long>(m) * s + x) * s + (s - 1 - y)) * 3;  // np.rot90: out[y, x] = in[x, s-1-y]
  else if (right)
    src = legend + (static_cast<long long>(y) * lw + (x - s)) * 3;
  else
    src = legend + (static_cast<long long>(y - s) * s + x) * 3;
  uint8_t* o = out + d[4] + p * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = src[c];
}

// img_concat_v(img_concat_h(views[:3]), img_concat_h(views[3:])), or img_concat_h(views) with oneline; the uncovered
// part of the narrower row is Image.new(mode, size, "black"): (0, 0, 0), and alpha 255 in RGBA.
__global__ void __launch_bounds__(kThreads) concat_views_kernel(const uint8_t* __restrict__ views, int n_views, int h,
                                                                int w, int c, int oneline, int oh, int ow,
                                                                uint8_t* __restrict__ out) {
  const int s = blockIdx.y;
  const long long p = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (p >= static_cast<long long>(oh) * ow) return;
  const int y = static_cast<int>(p / ow), x = static_cast<int>(p % ow);
  int view = x / w;
  if (!oneline) {
    const int row = y / h;
    view = view < (row ? n_views - 3 : 3) ? row * 3 + view : -1;
  }
  uint8_t* o = out + (static_cast<long long>(s) * oh * ow + p) * c;
  if (view < 0) {
    for (int k = 0; k < c; ++k) o[k] = k == 3 ? 255 : 0;
    return;
  }
  const uint8_t* src = views + (((static_cast<long long>(s) * n_views + view) * h + y % h) * w + x % w) * c;
  for (int k = 0; k < c; ++k) o[k] = src[k];
}

// to_pil_image(img * 0.5 + 0.5): each of * 0.5, + 0.5 and * 255 rounded to fp32, then .byte() truncates toward zero
// (modulo 256, as torch's CPU cast of an out-of-range value does)
__global__ void __launch_bounds__(kThreads) m11_to_u8_kernel(const float* __restrict__ x, long long n_pixels, int hw,
                                                             uint8_t* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= n_pixels) return;
  const long long img = i / hw, p = i % hw;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __ldg(x + (img * 3 + c) * hw + p);
    const float f = __fmul_rn(__fadd_rn(__fmul_rn(v, 0.5f), 0.5f), 255.f);
    out[i * 3 + c] = static_cast<uint8_t>(__float2int_rz(f));
  }
}

inline unsigned blocks(long long n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }

}  // namespace

extern "C" int mdb_render_bev_map(const void* maps, int maps_is_f32, int n_maps, int channels, int h, int w, int n_static,
                                  int n_dynamic, const int* priority, const unsigned char* colors, unsigned char* out,
                                  long long* info, void* stream) {
  using namespace mdb;
  if (!maps || !priority || !colors || !out || !info) return set_error(MDB_ERR_INVALID, "mdb_render_bev_map: null pointer");
  if (n_maps <= 0 || h <= 0 || w <= 0 || n_static < 0 || n_dynamic < 0 || n_static + n_dynamic == 0 ||
      n_static + n_dynamic > channels)
    return set_error(MDB_ERR_INVALID, "mdb_render_bev_map: bad sizes (maps=%d channels=%d %dx%d static=%d dynamic=%d)",
                     n_maps, channels, h, w, n_static, n_dynamic);
  if (n_static + n_dynamic > kMaxClasses || h > kMaxSide || w > kMaxSide || n_maps > 65535)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_render_bev_map: %d classes above %d, %dx%d above %d a side or %d maps",
                     n_static + n_dynamic, kMaxClasses, h, w, kMaxSide, n_maps);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  // {used, status} = 0, both error words all ones, for every map
  if (cudaMemset2DAsync(info, 4 * sizeof(long long), 0, 2 * sizeof(long long), n_maps, st) != cudaSuccess ||
      cudaMemset2DAsync(info + 2, 4 * sizeof(long long), 0xff, 2 * sizeof(long long), n_maps, st) != cudaSuccess)
    return set_error(MDB_ERR_CUDA, "mdb_render_bev_map: %s", cudaGetErrorString(cudaGetLastError()));
  const dim3 grid(blocks(static_cast<long long>(h) * w), n_maps);
  unsigned long long* inf = reinterpret_cast<unsigned long long*>(info);
  if (maps_is_f32)
    render_bev_map_kernel<float><<<grid, kThreads, 0, st>>>(static_cast<const float*>(maps), channels, h * w, n_static,
                                                            n_dynamic, priority, colors, out, inf);
  else
    render_bev_map_kernel<uint8_t><<<grid, kThreads, 0, st>>>(static_cast<const uint8_t*>(maps), channels, h * w,
                                                              n_static, n_dynamic, priority, colors, out, inf);
  MDB_CHECK_LAUNCH("render_bev_map_kernel");
  return MDB_OK;
}

extern "C" int mdb_place_map_u8(const unsigned char* resized, int n_maps, int s, const long long* desc,
                                long long max_pixels, unsigned char* out, void* stream) {
  using namespace mdb;
  if (!resized || !desc || !out) return set_error(MDB_ERR_INVALID, "mdb_place_map_u8: null pointer");
  if (n_maps <= 0 || s <= 0 || max_pixels <= 0)
    return set_error(MDB_ERR_INVALID, "mdb_place_map_u8: bad sizes (maps=%d side=%d pixels=%lld)", n_maps, s, max_pixels);
  if (n_maps > 65535 || s > kMaxSide || blocks(max_pixels) > 0x7fffffffu)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_place_map_u8: %d maps, side %d or %lld pixels too large", n_maps, s,
                     max_pixels);
  place_map_kernel<<<dim3(blocks(max_pixels), n_maps), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(resized, s, desc,
                                                                                                         out);
  MDB_CHECK_LAUNCH("place_map_kernel");
  return MDB_OK;
}

extern "C" int mdb_concat_views_u8(const unsigned char* views, int n_scenes, int n_views, int h, int w, int c, int oneline,
                                   unsigned char* out, void* stream) {
  using namespace mdb;
  if (!views || !out) return set_error(MDB_ERR_INVALID, "mdb_concat_views_u8: null pointer");
  if (n_scenes <= 0 || h <= 0 || w <= 0 || (c != 3 && c != 4) || n_views < (oneline ? 2 : 5))
    return set_error(MDB_ERR_INVALID, "mdb_concat_views_u8: bad sizes (scenes=%d views=%d %dx%dx%d oneline=%d)", n_scenes,
                     n_views, h, w, c, oneline);
  const long long oh = oneline ? h : 2LL * h;
  const long long ow = static_cast<long long>(oneline ? n_views : max(3, n_views - 3)) * w;
  if (n_scenes > 65535 || oh > INT_MAX || ow > INT_MAX || blocks(oh * ow) > 0x7fffffffu)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_concat_views_u8: %d scenes or a %lldx%lld mosaic too large", n_scenes, oh,
                     ow);
  concat_views_kernel<<<dim3(blocks(oh * ow), n_scenes), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      views, n_views, h, w, c, oneline, static_cast<int>(oh), static_cast<int>(ow), out);
  MDB_CHECK_LAUNCH("concat_views_kernel");
  return MDB_OK;
}

extern "C" int mdb_m11_to_u8(const float* x, int n, int h, int w, unsigned char* out, void* stream) {
  using namespace mdb;
  if (!x || !out) return set_error(MDB_ERR_INVALID, "mdb_m11_to_u8: null pointer");
  if (n <= 0 || h <= 0 || w <= 0) return set_error(MDB_ERR_INVALID, "mdb_m11_to_u8: bad shape %d x %dx%d", n, h, w);
  const long long n_pixels = static_cast<long long>(n) * h * w;
  if (static_cast<long long>(h) * w > INT_MAX || blocks(n_pixels) > 0x7fffffffu)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_m11_to_u8: %d x %dx%d too large", n, h, w);
  m11_to_u8_kernel<<<blocks(n_pixels), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, n_pixels, h * w, out);
  MDB_CHECK_LAUNCH("m11_to_u8_kernel");
  return MDB_OK;
}
