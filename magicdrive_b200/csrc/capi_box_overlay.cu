// 3D-box overlays on camera views (include/magicdrive_b200.h: mdb_project_boxes, mdb_draw_box_edges_aa): the reference's
// `show_box` images (demo/helper.py:197-307, visualize_camera / show_box_on_views / draw_box_on_imgs), equal byte for
// byte to OpenCV's drawing.  oracle/box_overlay.py is the same arithmetic in numpy.
//
// mdb_project_boxes: per (scene, view), box corners in float32 with torch's operation order and no contraction, projected
// in float64 (the products of float32 values are exact; the sums run in the order numpy's matmul gives), kept when all
// 8 corners are in front, ordered far to near by a stable rank on the smallest depth, clipped, divided and truncated.
// numpy's argsort is an introsort: for more than 16 boxes its order among exactly equal smallest depths is not
// reproduced (here ties keep box order).
//
// mdb_draw_box_edges_aa: cv2.line(img, p0, p1, colour, 1, cv2.LINE_AA) for every edge of every drawn box, in draw order.
// One CTA owns one view.  Edges are set up (clipping, slope, end-point corrections) a chunk at a time, one per thread,
// then drawn one after another: within one edge each DDA step touches 3 pixels no other step of that edge touches, so
// the steps run in parallel, and a barrier between edges keeps OpenCV's order wherever edges overlap.  No atomics.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"

namespace {

constexpr int kXYShift = 16;
constexpr long long kXYOne = 1LL << kXYShift;
constexpr int kMaxBoxes = 4096;   // per scene: the projection ranks them in shared memory (8 bytes each)
constexpr int kMaxSide = 32767;   // image height / width
constexpr int kDrawThreads = 512;
constexpr int kEdgeChunk = 256;   // edges set up per pass (<= kDrawThreads)

// OpenCV's LineAA tables (imgproc/src/drawing.cpp)
__constant__ int kFilter[64] = {
    168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
    254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
    158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
    40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5};
__constant__ int kSlopeCorr[32] = {181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
                                   203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254};
// mmdet3d's corner order, relative origin (0.5, 0.5, 0), and visualize_camera's edge order
__constant__ float kCx[8] = {-0.5f, -0.5f, -0.5f, -0.5f, 0.5f, 0.5f, 0.5f, 0.5f};
__constant__ float kCy[8] = {-0.5f, -0.5f, 0.5f, 0.5f, -0.5f, -0.5f, 0.5f, 0.5f};
__constant__ float kCz[8] = {0.f, 1.f, 1.f, 0.f, 0.f, 1.f, 1.f, 0.f};
__constant__ int kEdges[12][2] = {{0, 1}, {0, 3}, {0, 4}, {1, 2}, {1, 5}, {3, 2}, {3, 7}, {4, 5}, {4, 7}, {2, 6}, {5, 6}, {6, 7}};

// ------------------------------------------------------------------------------------------------------------ project
// Corner k of box b (shifted to a gravity-centre origin) in the view's homogeneous image frame, float64.
__device__ __forceinline__ void project_corner(const float* b, float sn, float cs, const double* T, int k, double& u,
                                               double& v, double& z) {
  const float zc = __fadd_rn(b[2], __fmul_rn(b[5], -0.5f));  // tensor[:, :3] += dims * ((0.5, 0.5, 0) - (0.5, 0.5, 0.5))
  const float ox = __fmul_rn(b[3], kCx[k]), oy = __fmul_rn(b[4], kCy[k]), oz = __fmul_rn(b[5], kCz[k]);
  // einsum("aij,jka->aik") with rot_mat_T = [[cos, -sin, 0], [sin, cos, 0], [0, 0, 1]], then + centre
  const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(ox, cs), __fmul_rn(oy, sn)), __fmul_rn(oz, 0.f)), b[0]);
  const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(ox, -sn), __fmul_rn(oy, cs)), __fmul_rn(oz, 0.f)), b[1]);
  const float zz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(ox, 0.f), __fmul_rn(oy, 0.f)), __fmul_rn(oz, 1.f)), zc);
  const double p[3] = {x, y, zz};
  double r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], T[i * 4]), __dmul_rn(p[1], T[i * 4 + 1])), __dmul_rn(p[2], T[i * 4 + 2])),
                     T[i * 4 + 3]);
  u = r[0], v = r[1], z = r[2];
}

__global__ void project_boxes_kernel(const float* __restrict__ boxes, int box_dim, const float* __restrict__ sincos,
                                     const long long* __restrict__ labels, const int* __restrict__ box_offsets,
                                     const float* __restrict__ transforms, int n_views, int capacity,
                                     int* __restrict__ endpoints, int* __restrict__ colors, int* __restrict__ counts,
                                     int* __restrict__ status) {
  extern __shared__ double minz[];  // smallest depth of each box, -1 when a corner is not in front
  __shared__ double T[16];
  const int v = blockIdx.x, s = blockIdx.y;
  const long long sv = static_cast<long long>(s) * n_views + v;
  const int b0 = box_offsets[s], nb = box_offsets[s + 1] - b0;
  if (nb > capacity) {
    if (threadIdx.x == 0) counts[sv] = 0, status[sv] = 2;
    return;
  }
  if (threadIdx.x < 16) T[threadIdx.x] = transforms[sv * 16 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    const float* b = boxes + static_cast<long long>(b0 + i) * box_dim;
    const float sn = sincos[(b0 + i) * 2], cs = sincos[(b0 + i) * 2 + 1];
    double m = 0.0;
    bool front = true;
    for (int k = 0; k < 8; ++k) {
      double u, w, z;
      project_corner(b, sn, cs, T, k, u, w, z);
      front = front && z > 0.0;
      m = k == 0 ? z : fmin(m, z);
    }
    minz[i] = front ? m : -1.0;
  }
  __syncthreads();
  int drawn = 0;
  for (int base = 0; base < nb; base += blockDim.x)
    drawn += __syncthreads_count(base + threadIdx.x < nb && minz[base + threadIdx.x] > 0.0);
  bool bad = false;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    const double mi = minz[i];
    if (!(mi > 0.0)) continue;
    int rank = 0;  // np.argsort(-min z), stable
    for (int j = 0; j < nb; ++j) {
      const double mj = minz[j];
      rank += (mj > mi) || (mj == mi && j < i);
    }
    const float* b = boxes + static_cast<long long>(b0 + i) * box_dim;
    const float sn = sincos[(b0 + i) * 2], cs = sincos[(b0 + i) * 2 + 1];
    int* e = endpoints + (sv * capacity + rank) * 16;
    for (int k = 0; k < 8; ++k) {
      double u, w, z;
      project_corner(b, sn, cs, T, k, u, w, z);
      z = fmin(fmax(z, 1e-5), 1e5);
      const double x = trunc(__ddiv_rn(u, z)), y = trunc(__ddiv_rn(w, z));  // astype(int): toward zero
      const bool ok = x >= -2147483648.0 && x <= 2147483647.0 && y >= -2147483648.0 && y <= 2147483647.0;
      bad = bad || !ok;
      e[k * 2] = ok ? static_cast<int>(x) : 0;
      e[k * 2 + 1] = ok ? static_cast<int>(y) : 0;
    }
    colors[sv * capacity + rank] = static_cast<int>(labels[b0 + i]);
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) counts[sv] = drawn, status[sv] = bad ? 1 : 0;
}

// --------------------------------------------------------------------------------------------------------------- draw
struct Edge {         // one clipped edge, ready for its DDA (cv::LineAA)
  long long minor;    // 16.16 minor-axis position at step 0, + 1/2
  long long step;     // its increment per step
  int major0;         // major-axis pixel at step 0
  int ecount;         // steps - 1; -1 when the edge misses the image
  int x_major;
  int color;
  short ep[9];        // end-point corrections
};

__device__ __forceinline__ long long tdiv(long long a, long long b) { return a / b; }  // C division: toward zero

__device__ __forceinline__ long long clip_term(long long a, long long b, long long c) {  // (int64)((double)a * b / c)
  return __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(a), __ll2double_rn(b)), __ll2double_rn(c)));
}

// cv::clipLine on the (w << 16) x (h << 16) rectangle, then LineAA's set-up
__device__ Edge setup_edge(int h, int w, const int* p0, const int* p1, int color) {
  Edge e;
  e.color = color;
  e.ecount = -1;
  long long x1 = static_cast<long long>(p0[0]) << kXYShift, y1 = static_cast<long long>(p0[1]) << kXYShift;
  long long x2 = static_cast<long long>(p1[0]) << kXYShift, y2 = static_cast<long long>(p1[1]) << kXYShift;
  const long long right = (static_cast<long long>(w) << kXYShift) - 1, bottom = (static_cast<long long>(h) << kXYShift) - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    if (c1 & 12) {
      const long long a = c1 < 8 ? 0 : bottom;
      x1 += clip_term(a - y1, x2 - x1, y2 - y1);
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      const long long a = c2 < 8 ? 0 : bottom;
      x2 += clip_term(a - y2, x2 - x1, y2 - y1);
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        const long long a = c1 == 1 ? 0 : right;
        y1 += clip_term(a - x1, y2 - y1, x2 - x1);
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        const long long a = c2 == 1 ? 0 : right;
        y2 += clip_term(a - x2, y2 - y1, x2 - x1);
        x2 = a;
        c2 = 0;
      }
    }
  }
  if ((c1 | c2) != 0) return e;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long i, j;
  e.x_major = ax > ay;
  if (e.x_major) {
    if (dx < 0) {
      dy = -dy;
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    e.step = tdiv(dy * kXYOne, ax | 1);
    x2 += kXYOne;
    e.ecount = static_cast<int>((x2 >> kXYShift) - (x1 >> kXYShift));
    e.minor = y1 + ((e.step * -(x1 & (kXYOne - 1))) >> kXYShift) + (kXYOne >> 1);
    i = (x1 >> (kXYShift - 7)) & 0x78, j = (x2 >> (kXYShift - 7)) & 0x78;
    e.major0 = static_cast<int>(x1 >> kXYShift);
  } else {
    if (dy < 0) {
      dx = -dx;
      long long t = x1; x1 = x2; x2 = t;
      t = y1; y1 = y2; y2 = t;
    }
    e.step = tdiv(dx * kXYOne, ay | 1);
    y2 += kXYOne;
    e.ecount = static_cast<int>((y2 >> kXYShift) - (y1 >> kXYShift));
    e.minor = x1 + ((e.step * -(y1 & (kXYOne - 1))) >> kXYShift) + (kXYOne >> 1);
    i = (y1 >> (kXYShift - 7)) & 0x78, j = (y2 >> (kXYShift - 7)) & 0x78;
    e.major0 = static_cast<int>(y1 >> kXYShift);
  }
  int slope = static_cast<int>((e.step >> (kXYShift - 5)) & 0x3f) ^ (e.step < 0 ? 0x3f : 0);
  slope = (slope & 0x20) ? 0x100 : kSlopeCorr[slope];
  const long long t0 = slope << 7, t1 = ((0x78 - i) | 4) * slope, t2 = (j | 4) * slope;
  e.ep[0] = 0;
  e.ep[8] = static_cast<short>(slope);
  e.ep[1] = e.ep[3] = static_cast<short>(((((j - i) & 0x78) | 4) * slope >> 8) & 0x1ff);
  e.ep[2] = static_cast<short>((t1 >> 8) & 0x1ff);
  e.ep[4] = static_cast<short>(((((j - i) + 0x80) | 4) * slope >> 8) & 0x1ff);
  e.ep[5] = static_cast<short>(((t1 + t0) >> 8) & 0x1ff);
  e.ep[6] = static_cast<short>((t2 >> 8) & 0x1ff);
  e.ep[7] = static_cast<short>(((t2 + t0) >> 8) & 0x1ff);
  return e;
}

__device__ __forceinline__ void blend(uint8_t* p, const uint8_t* col, int a) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int v = p[c];
    v += ((col[c] - v) * a + 127) >> 8;  // OpenCV applies the blend twice
    v += ((col[c] - v) * a + 127) >> 8;
    p[c] = static_cast<uint8_t>(v);
  }
}

__global__ void __launch_bounds__(kDrawThreads) draw_box_edges_kernel(
    const void* __restrict__ images, int images_is_f32, int n_images, int h, int w, const int* __restrict__ endpoints,
    const int* __restrict__ colors, const int* __restrict__ counts, const int* __restrict__ status, int capacity,
    const uint8_t* __restrict__ palette, int n_colors, int transparent_bg, uint8_t* out) {
  __shared__ Edge edges[kEdgeChunk];
  __shared__ uint8_t pal[kEdgeChunk][3];
  const int img = blockIdx.x;
  // a view whose endpoints cv2 would refuse fails the whole call, which then writes nothing
  bool failed = false;
  for (int i = threadIdx.x; i < n_images; i += blockDim.x) failed = failed || status[i] != 0;
  if (__syncthreads_or(failed)) return;

  const int cs = transparent_bg ? 4 : 3;
  const long long hw = static_cast<long long>(h) * w;
  uint8_t* o = out + img * hw * cs;
  if (transparent_bg || images != out) {
    for (long long p = threadIdx.x; p < hw; p += blockDim.x) {
      uint8_t px[3] = {0, 0, 0};
      if (!transparent_bg) {
        for (int c = 0; c < 3; ++c) {
          const long long at = (img * hw + p) * 3 + c;
          if (images_is_f32) {
            const float f = rintf(__fmul_rn(static_cast<const float*>(images)[at], 255.f));  // numpy_to_pil
            px[c] = static_cast<uint8_t>(fminf(fmaxf(f, 0.f), 255.f));
          } else {
            px[c] = static_cast<const uint8_t*>(images)[at];
          }
        }
      }
      for (int c = 0; c < 3; ++c) o[p * cs + c] = px[c];
    }
  }
  __syncthreads();

  const int n_edges = min(counts[img], capacity) * 12;
  const int* ends = endpoints + static_cast<long long>(img) * capacity * 16;
  for (int base = 0; base < n_edges; base += kEdgeChunk) {
    const int k = base + threadIdx.x;
    if (threadIdx.x < kEdgeChunk && k < n_edges) {
      const int box = k / 12, ed = k % 12;
      const int col = colors[static_cast<long long>(img) * capacity + box];
      const bool ok = col >= 0 && col < n_colors;
      edges[threadIdx.x] = setup_edge(h, w, ends + box * 16 + kEdges[ed][0] * 2, ends + box * 16 + kEdges[ed][1] * 2, col);
      if (!ok) edges[threadIdx.x].ecount = -1;
      for (int c = 0; c < 3; ++c) pal[threadIdx.x][c] = ok ? palette[col * 3 + c] : 0;
    }
    __syncthreads();
    const int chunk = min(kEdgeChunk, n_edges - base);
    for (int q = 0; q < chunk; ++q) {
      const Edge& e = edges[q];
      const int major_n = e.x_major ? w : h, minor_n = e.x_major ? h : w;
      for (int st = threadIdx.x; st <= e.ecount; st += blockDim.x) {
        const int major = e.major0 + st;
        if (static_cast<unsigned>(major) >= static_cast<unsigned>(major_n)) continue;
        const long long m = e.minor + static_cast<long long>(st) * e.step;
        const int corr = e.ep[min(st, 2) * 3 + min(e.ecount - st, 2)];
        const int dist = static_cast<int>((m >> (kXYShift - 5)) & 31);
        const int first = static_cast<int>(m >> kXYShift) - 1;
        const int f[3] = {kFilter[dist + 32], kFilter[dist], kFilter[63 - dist]};
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const int mi = first + t;
          if (static_cast<unsigned>(mi) >= static_cast<unsigned>(minor_n)) continue;
          const int a = (corr * f[t] >> 8) & 0xff;
          const long long p = e.x_major ? static_cast<long long>(mi) * w + major : static_cast<long long>(major) * w + mi;
          blend(o + p * cs, pal[q], a);
        }
      }
      __syncthreads();
    }
  }

  if (transparent_bg) {
    for (long long p = threadIdx.x; p < hw; p += blockDim.x)
      o[p * 4 + 3] = (o[p * 4] | o[p * 4 + 1] | o[p * 4 + 2]) ? 255 : 0;
  }
}

}  // namespace

extern "C" int mdb_project_boxes(const float* boxes, int box_dim, const float* sincos, const long long* labels,
                                 const int* box_offsets, int n_scenes, const float* transforms, int n_views, int capacity,
                                 int* endpoints, int* colors, int* counts, int* status, void* stream) {
  using namespace mdb;
  if (!boxes || !sincos || !labels || !box_offsets || !transforms || !endpoints || !colors || !counts || !status)
    return set_error(MDB_ERR_INVALID, "mdb_project_boxes: null pointer");
  if (box_dim < 7 || n_scenes <= 0 || n_views <= 0 || capacity <= 0)
    return set_error(MDB_ERR_INVALID, "mdb_project_boxes: bad sizes (box_dim=%d scenes=%d views=%d capacity=%d)", box_dim,
                     n_scenes, n_views, capacity);
  if (capacity > kMaxBoxes || n_scenes > 65535)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_project_boxes: capacity %d above %d or %d scenes above 65535", capacity,
                     kMaxBoxes, n_scenes);
  project_boxes_kernel<<<dim3(n_views, n_scenes), 128, capacity * sizeof(double), static_cast<cudaStream_t>(stream)>>>(
      boxes, box_dim, sincos, labels, box_offsets, transforms, n_views, capacity, endpoints, colors, counts, status);
  MDB_CHECK_LAUNCH("project_boxes_kernel");
  return MDB_OK;
}

extern "C" int mdb_draw_box_edges_aa(const void* images, int images_is_f32, int n_images, int h, int w,
                                     const int* endpoints, const int* colors, const int* counts, const int* status,
                                     int capacity, const unsigned char* palette, int n_colors, int transparent_bg, void* out,
                                     void* stream) {
  using namespace mdb;
  if (!endpoints || !colors || !counts || !status || !palette || !out || (!transparent_bg && !images))
    return set_error(MDB_ERR_INVALID, "mdb_draw_box_edges_aa: null pointer");
  if (n_images <= 0 || h <= 0 || w <= 0 || capacity <= 0 || n_colors <= 0)
    return set_error(MDB_ERR_INVALID, "mdb_draw_box_edges_aa: bad sizes (images=%d %dx%d capacity=%d colours=%d)", n_images,
                     h, w, capacity, n_colors);
  if (h > kMaxSide || w > kMaxSide)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_draw_box_edges_aa: %dx%d above %d pixels a side", h, w, kMaxSide);
  if (!transparent_bg && images == out && images_is_f32)
    return set_error(MDB_ERR_INVALID, "mdb_draw_box_edges_aa: fp32 images cannot be drawn in place");
  draw_box_edges_kernel<<<n_images, kDrawThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      transparent_bg ? nullptr : images, images_is_f32, n_images, h, w, endpoints, colors, counts, status, capacity,
      static_cast<const uint8_t*>(palette), n_colors, transparent_bg, static_cast<uint8_t*>(out));
  MDB_CHECK_LAUNCH("draw_box_edges_kernel");
  return MDB_OK;
}
