// Baseline JPEG encoder (include/magicdrive_b200.h: mdb_jpeg_encode_u8): the files Pillow writes with
// Image.save(f, "JPEG", quality=q) at its defaults -- 4:2:0, the standard Huffman tables, no restart interval -- byte for
// byte.  oracle/jpeg_encode.py is the same coder in numpy.
//
// Nine launches per batch, all sized from the shapes alone:
//   coef       one CTA per 16 x 16 MCU: the forward half of capi_fid_protocol.cu's round trip, quantised int16
//              coefficients [n, mcus, 6, 64] in zigzag order, with libjpeg's dummy blocks past the luma plane's edge
//   bits       one warp per 8 x 8 block: the block's coded length, summed per MCU
//   scan_mcus  one CTA per image: int64 exclusive sum of the MCU lengths -> each MCU's first bit
//   layout     one CTA: each image's region of the bit buffer, whole 4 KiB chunks, int64 across the batch
//   zero       the used part of the bit buffer
//   pack       one warp per block again: each lane's (code, length) words ORed big-endian into the bit buffer, then the
//              1-bits that pad each image to a byte
//   ff_count   one CTA per chunk: 0xFF bytes
//   place      one CTA: each chunk's stuffed position, each file's length and its offset in `out`
//   scatter    one CTA per chunk: header, entropy-coded bytes with a 0x00 after every 0xFF, EOI
// A bit buffer or an output that is too small is found on the device: the kernels after it write nothing and `meta`
// says what was needed.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"
#include "jpeg_fdct.cuh"

namespace {

constexpr int kChunk = 4096;  // bytes of the bit buffer per stuffing CTA; each image's region is whole chunks
constexpr int kChunkGrid = 32;  // CTAs per image of the chunk kernels (grid-stride over the image's chunks)

// natural index of zigzag position k
__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ITU-T T.81 K.3: code counts of lengths 1..16 and the symbols in code order
constexpr uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                    {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
constexpr uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// symbol -> (code, length) of one table (T.81 Annex C)
struct HuffTable {
  uint16_t code[256];
  uint8_t len[256];
};
constexpr HuffTable make_table(const uint8_t* bits, const uint8_t* vals) {
  HuffTable t{};
  int code = 0, k = 0;
  for (int length = 1; length <= 16; ++length) {
    for (int i = 0; i < bits[length - 1]; ++i, ++k, ++code) {
      t.code[vals[k]] = static_cast<uint16_t>(code);
      t.len[vals[k]] = static_cast<uint8_t>(length);
    }
    code <<= 1;
  }
  return t;
}
// DC luma, AC luma, DC chroma, AC chroma
__constant__ HuffTable kHuff[4] = {make_table(kDcBits[0], kDcVals), make_table(kAcBits[0], kAcVals[0]),
                                   make_table(kDcBits[1], kDcVals), make_table(kAcBits[1], kAcVals[1])};

// ------------------------------------------------------------------------------------------------------ coefficients
// The forward DCT and quantisation of capi_fid_protocol.cu's jpeg_code_mcu_kernel, then the zigzag store.  Luma blocks
// wholly past ceil(w / 8) block columns or ceil(h / 8) block rows are libjpeg's dummy blocks (jccoefct.c, compress_data):
// zero AC and the DC of the block before them in the MCU.
__global__ void __launch_bounds__(256) jpeg_coef_kernel(const uint8_t* __restrict__ x, int h, int w, QuantTables qt,
                                                        int16_t* __restrict__ coef) {
  __shared__ int blk[6][64];
  __shared__ int dc[6];
  const int mcus_x = (w + 15) >> 4;
  const int my = blockIdx.x / mcus_x, mx = blockIdx.x % mcus_x, img = blockIdx.y;
  const int t = threadIdx.x;
  load_mcu(x, h, w, img, my, mx, blk);
  __syncthreads();
  const int b = t >> 3, k = t & 7;
  if (t < 48) fdct8<true>(&blk[b][k * 8], 1);
  __syncthreads();
  if (t < 48) {
    int* col = &blk[b][k];
    fdct8<false>(col, 8);
    const int* q = qt.q[b < 4 ? 0 : 1];
#pragma unroll
    for (int r = 0; r < 8; ++r) {  // round half away from zero
      const int v = col[8 * r], d = q[8 * r + k] * 8;
      const int a = ((v < 0 ? -v : v) + (d >> 1)) / d;
      col[8 * r] = v < 0 ? -a : a;
    }
  }
  __syncthreads();
  const int bw = (w + 7) >> 3, bh = (h + 7) >> 3;
  auto dummy = [&](int bb) { return bb < 4 && (2 * mx + (bb & 1) >= bw || 2 * my + (bb >> 1) >= bh); };
  if (t == 0) {
    for (int bb = 0; bb < 6; ++bb) dc[bb] = dummy(bb) ? dc[bb - 1] : blk[bb][0];  // block 0 is never a dummy
  }
  __syncthreads();
  int16_t* dst = coef + (static_cast<long long>(img) * gridDim.x + blockIdx.x) * 384;
  for (int i = t; i < 384; i += 256) {
    const int bb = i >> 6, kk = i & 63;
    const int v = kk == 0 ? dc[bb] : (dummy(bb) ? 0 : blk[bb][kZigzag[kk]]);
    dst[i] = static_cast<int16_t>(v);
  }
}

// ------------------------------------------------------------------------------------------------------ Huffman words
__device__ __forceinline__ int category(int v) { return 32 - __clz(v < 0 ? -v : v); }

// The (code, length) word of zigzag coefficient k of a block (length 0: nothing to code).  k = 0: the DC difference.
// k >= 1 nonzero: up to three ZRLs for the zeros before it, its run / size symbol and its bits.  k = 63 zero: EOB.
// Lengths stay below 64: 3 x 11 + 16 + 10 bits at most.
__device__ __forceinline__ int coef_word(int v, int k, int pred, unsigned long long ac_mask, int chroma, uint64_t* out) {
  const HuffTable& dct = kHuff[2 * chroma];
  const HuffTable& act = kHuff[2 * chroma + 1];
  if (k == 0) {
    const int d = v - pred, nb = category(d);
    *out = (static_cast<uint64_t>(dct.code[nb]) << nb) | (static_cast<unsigned>(d < 0 ? d - 1 : d) & ((1u << nb) - 1));
    return dct.len[nb] + nb;
  }
  if (v == 0) {
    if (k != 63) return 0;
    *out = act.code[0];
    return act.len[0];
  }
  const unsigned long long below = ac_mask & ((1ull << k) - 1);
  int r = k - 1 - (below ? 63 - __clzll(below) : 0);
  uint64_t c = 0;
  int len = 0;
  for (; r > 15; r -= 16) {
    c = (c << act.len[0xF0]) | act.code[0xF0];
    len += act.len[0xF0];
  }
  const int nb = category(v), sym = (r << 4) | nb;
  c = (c << act.len[sym]) | act.code[sym];
  c = (c << nb) | (static_cast<unsigned>(v < 0 ? v - 1 : v) & ((1u << nb) - 1));
  *out = c;
  return len + act.len[sym] + nb;
}

// OR the `len` (1..64) low bits of `code` into the big-endian bit buffer at bit `pos`
__device__ __forceinline__ void put_bits(uint32_t* buf, long long pos, uint64_t code, int len) {
  const uint64_t v = code << (64 - len);
  const int s = static_cast<int>(pos & 31);
  uint32_t* p = buf + (pos >> 5);
  const uint32_t high = static_cast<uint32_t>(v >> (32 + s));
  if (high) atomicOr(p, high);
  const uint32_t mid = static_cast<uint32_t>(v >> s), low = static_cast<uint32_t>(v << (32 - s));
  if (mid) atomicOr(p + 1, mid);
  if (low) atomicOr(p + 2, low);
}

struct ImageLayout {  // per image, int64
  long long bits;     // entropy-coded bits before the padding
  long long chunk0;   // first chunk of its bit-buffer region
  long long nchunks;  // chunks of that region
  long long file;     // file length
};

// One CTA of six warps per MCU, warp b on block b; lane l holds zigzag coefficients l and l + 32.
// kPack false: mcu_bits[img, mcu] = the MCU's coded length.  kPack true: the words ORed into the bit buffer.
template <bool kPack>
__global__ void __launch_bounds__(192) jpeg_blocks_kernel(const int16_t* __restrict__ coef, int* __restrict__ mcu_bits,
                                                          const long long* __restrict__ mcu_first,
                                                          const ImageLayout* __restrict__ layout,
                                                          const int* __restrict__ flags, uint32_t* __restrict__ bitbuf) {
  __shared__ int warp_bits[6];
  if (kPack && !flags[0]) return;
  const int mcus = gridDim.x, mcu = blockIdx.x, img = blockIdx.y;
  const int b = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m = static_cast<long long>(img) * mcus + mcu;
  const int16_t* blk = coef + (m * 6 + b) * 64;
  // the previous block of the same component in scan order; predictors start at 0 per image
  int pred = 0;
  if (b >= 1 && b <= 3) pred = blk[-64];
  else if (mcu > 0) pred = coef[((m - 1) * 6 + (b == 0 ? 3 : b)) * 64];
  const int v0 = blk[lane], v1 = blk[lane + 32];
  const unsigned long long ac_mask = (static_cast<unsigned long long>(__ballot_sync(~0u, v1 != 0)) << 32 |
                                      __ballot_sync(~0u, v0 != 0)) & ~1ull;
  const int chroma = b >= 4;
  uint64_t c0 = 0, c1 = 0;
  const int l0 = coef_word(v0, lane, pred, ac_mask, chroma, &c0);
  const int l1 = coef_word(v1, lane + 32, pred, ac_mask, chroma, &c1);
  int s0 = l0, s1 = l1;  // inclusive scans over the lanes
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int a0 = __shfl_up_sync(~0u, s0, d), a1 = __shfl_up_sync(~0u, s1, d);
    if (lane >= d) s0 += a0, s1 += a1;
  }
  const int half = __shfl_sync(~0u, s0, 31), total = half + __shfl_sync(~0u, s1, 31);
  if (lane == 0) warp_bits[b] = total;
  __syncthreads();
  if (!kPack) {
    if (threadIdx.x == 0) {
      int sum = 0;
      for (int i = 0; i < 6; ++i) sum += warp_bits[i];
      mcu_bits[m] = sum;
    }
    return;
  }
  long long pos = layout[img].chunk0 * (8LL * kChunk) + mcu_first[m];
  for (int i = 0; i < b; ++i) pos += warp_bits[i];
  if (l0) put_bits(bitbuf, pos + s0 - l0, c0, l0);
  if (l1) put_bits(bitbuf, pos + half + s1 - l1, c1, l1);
  if (mcu == 0 && threadIdx.x == 0) {  // 1-bits to the byte boundary (libjpeg's flush_bits)
    const long long bits = layout[img].bits;
    const int pad = static_cast<int>((8 - (bits & 7)) & 7);
    if (pad) put_bits(bitbuf, layout[img].chunk0 * (8LL * kChunk) + bits, (1u << pad) - 1, pad);
  }
}

// ------------------------------------------------------------------------------------------------------------ scans
// Exclusive prefix sum over the CTA (blockDim.x a multiple of 32, at most 1024); *total gets the CTA's sum.
__device__ long long cta_exclusive_scan(long long v, long long* total) {
  __shared__ long long warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  long long s = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long a = __shfl_up_sync(~0u, s, d);
    if (lane >= d) s += a;
  }
  __syncthreads();  // warp_sums may still be read from the previous call
  if (lane == 31) warp_sums[warp] = s;
  __syncthreads();
  long long before = 0, all = 0;
  for (int i = 0; i < warps; ++i) {
    if (i < warp) before += warp_sums[i];
    all += warp_sums[i];
  }
  *total = all;
  return before + s - v;
}

// one CTA per image: mcu_first[img, i] = the bits of MCUs 0..i-1; layout[img].bits = the image's
__global__ void __launch_bounds__(1024) jpeg_scan_mcus_kernel(const int* __restrict__ mcu_bits, int mcus,
                                                              long long* __restrict__ mcu_first,
                                                              ImageLayout* __restrict__ layout) {
  const long long base = static_cast<long long>(blockIdx.x) * mcus;
  long long carry = 0;
  for (int i0 = 0; i0 < mcus; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    long long tot;
    const long long ex = cta_exclusive_scan(i < mcus ? mcu_bits[base + i] : 0, &tot);
    if (i < mcus) mcu_first[base + i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) layout[blockIdx.x].bits = carry;
}

// one CTA: each image's bit-buffer region (whole chunks), flags[0] = whether they fit in `chunks`
__global__ void __launch_bounds__(1024) jpeg_layout_kernel(int n, long long chunks, ImageLayout* __restrict__ layout,
                                                           int* __restrict__ flags, long long* __restrict__ meta) {
  long long carry = 0;
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const long long bytes = i < n ? (layout[i].bits + 7) >> 3 : 0;
    const long long nc = (bytes + kChunk - 1) / kChunk;
    long long tot;
    const long long ex = cta_exclusive_scan(nc, &tot);
    if (i < n) {
      layout[i].chunk0 = carry + ex;
      layout[i].nchunks = nc;
      meta[3 * i] = bytes, meta[3 * i + 1] = -1, meta[3 * i + 2] = -1;
    }
    carry += tot;
  }
  if (threadIdx.x == 0) {
    flags[0] = carry <= chunks;  // the bit buffer holds every image
    flags[1] = 0;                // the files fit in `out`: set by jpeg_place_kernel
    *reinterpret_cast<long long*>(flags + 2) = carry;
  }
}

// the used part of the bit buffer
__global__ void jpeg_zero_kernel(const int* __restrict__ flags, uint4* __restrict__ bitbuf) {
  if (!flags[0]) return;
  const long long words = *reinterpret_cast<const long long*>(flags + 2) * (kChunk / 16);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < words;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    bitbuf[i] = make_uint4(0, 0, 0, 0);
}

// byte j of the bit buffer (words hold four bytes, the first in the high bits)
__device__ __forceinline__ uint32_t byte_at(const uint32_t* buf, long long j) {
  return (buf[j >> 2] >> (24 - 8 * (j & 3))) & 0xFF;
}

// Thread t of a 256-thread CTA covers bytes 16 t .. 16 t + 15 of a chunk: their 0xFF count.
__device__ __forceinline__ int count_ff(const uint32_t* chunk, long long valid) {
  const uint4 q = reinterpret_cast<const uint4*>(chunk)[threadIdx.x];
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
  int c = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i)
    c += (16LL * threadIdx.x + i < valid) && ((w[i >> 2] >> (24 - 8 * (i & 3))) & 0xFF) == 0xFF;
  return c;
}

__global__ void __launch_bounds__(256) jpeg_ff_count_kernel(const ImageLayout* __restrict__ layout,
                                                            const int* __restrict__ flags,
                                                            const uint32_t* __restrict__ bitbuf,
                                                            long long* __restrict__ chunk_ff) {
  if (!flags[0]) return;
  const ImageLayout L = layout[blockIdx.y];
  const long long bytes = (L.bits + 7) >> 3;
  for (long long j = blockIdx.x; j < L.nchunks; j += gridDim.x) {
    const uint32_t* chunk = bitbuf + (L.chunk0 + j) * (kChunk / 4);
    long long tot;
    cta_exclusive_scan(count_ff(chunk, bytes - j * kChunk), &tot);
    if (threadIdx.x == 0) chunk_ff[L.chunk0 + j] = tot;
  }
}

// one CTA: chunk_ff -> each chunk's first stuffed byte within its image's scan; file lengths and offsets in `out`
__global__ void __launch_bounds__(1024) jpeg_place_kernel(int n, long long out_bytes, ImageLayout* __restrict__ layout,
                                                          int* __restrict__ flags, long long* __restrict__ chunk_ff,
                                                          long long* __restrict__ meta) {
  if (!flags[0]) return;
  for (int img = 0; img < n; ++img) {
    const ImageLayout L = layout[img];
    long long carry = 0;
    for (long long j0 = 0; j0 < L.nchunks; j0 += blockDim.x) {
      const long long j = j0 + threadIdx.x;
      long long tot;
      const long long ex = cta_exclusive_scan(j < L.nchunks ? chunk_ff[L.chunk0 + j] : 0, &tot);
      if (j < L.nchunks) chunk_ff[L.chunk0 + j] = j * kChunk + carry + ex;
      carry += tot;
    }
    if (threadIdx.x == 0) layout[img].file = MDB_JPEG_HEADER_BYTES + ((L.bits + 7) >> 3) + carry + 2;
  }
  __syncthreads();
  long long carry = 0;
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    long long tot;
    const long long ex = cta_exclusive_scan(i < n ? layout[i].file : 0, &tot);
    if (i < n) meta[3 * i + 1] = layout[i].file, meta[3 * i + 2] = carry + ex;
    carry += tot;
  }
  const int fits = carry <= out_bytes;
  for (int i = threadIdx.x; i < n && !fits; i += blockDim.x) meta[3 * i + 2] = -1;
  if (threadIdx.x == 0) flags[1] = fits;
}

struct Header {
  uint8_t b[MDB_JPEG_HEADER_BYTES];
};

__global__ void __launch_bounds__(256) jpeg_scatter_kernel(const ImageLayout* __restrict__ layout,
                                                           const int* __restrict__ flags,
                                                           const uint32_t* __restrict__ bitbuf,
                                                           const long long* __restrict__ chunk_first,
                                                           const long long* __restrict__ meta, Header hdr,
                                                           uint8_t* __restrict__ out) {
  if (!flags[1]) return;
  const int img = blockIdx.y;
  const ImageLayout L = layout[img];
  uint8_t* file = out + meta[3 * img + 2];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < MDB_JPEG_HEADER_BYTES; i += blockDim.x) file[i] = hdr.b[i];
    if (threadIdx.x == 0) file[L.file - 2] = 0xFF, file[L.file - 1] = 0xD9;
  }
  const long long bytes = (L.bits + 7) >> 3;
  for (long long j = blockIdx.x; j < L.nchunks; j += gridDim.x) {
    const uint32_t* chunk = bitbuf + (L.chunk0 + j) * (kChunk / 4);
    const long long valid = bytes - j * kChunk;
    long long tot;
    long long p = MDB_JPEG_HEADER_BYTES + chunk_first[L.chunk0 + j] + cta_exclusive_scan(count_ff(chunk, valid), &tot);
    for (int i = 0; i < 16; ++i) {
      const long long jb = 16LL * threadIdx.x + i;
      if (jb >= valid) break;
      const uint32_t v = byte_at(chunk, jb);
      file[p + jb] = static_cast<uint8_t>(v);  // p counts the 0x00 bytes stuffed before this one
      if (v == 0xFF) file[p + jb + 1] = 0, ++p;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ host
struct Scratch {
  long long coef, mcu_bits, mcu_first, layout, flags, chunk_ff, bitbuf, total;
};

long long align256(long long v) { return (v + 255) & ~255LL; }

// byte offsets of the scratch regions for `chunks` 4 KiB chunks of bit buffer
Scratch scratch_layout(int n, int h, int w, long long chunks) {
  const long long mcus = static_cast<long long>((h + 15) / 16) * ((w + 15) / 16);
  Scratch s{};
  s.coef = 0;
  s.mcu_bits = align256(s.coef + n * mcus * 384 * 2);
  s.mcu_first = align256(s.mcu_bits + n * mcus * 4);
  s.layout = align256(s.mcu_first + n * mcus * 8);
  s.flags = align256(s.layout + n * static_cast<long long>(sizeof(ImageLayout)));
  s.chunk_ff = align256(s.flags + 64);
  s.bitbuf = align256(s.chunk_ff + chunks * 8);
  s.total = s.bitbuf + chunks * kChunk;
  return s;
}

void put16(uint8_t*& p, int v) { *p++ = static_cast<uint8_t>(v >> 8), *p++ = static_cast<uint8_t>(v); }

// SOI, APP0 JFIF 1.01 (no units, density 1 x 1, no thumbnail), DQT luma and chroma (8-bit, zigzag), SOF0 (components
// 1: 2x2 table 0, 2 and 3: 1x1 table 1), DHT DC0 AC0 DC1 AC1, SOS: what libjpeg writes before the scan for Pillow
Header make_header(int h, int w, const QuantTables& qt) {
  static const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  Header hd{};
  uint8_t* p = hd.b;
  const uint8_t app0[] = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  memcpy(p, app0, sizeof(app0));
  p += sizeof(app0);
  for (int t = 0; t < 2; ++t) {
    *p++ = 0xFF, *p++ = 0xDB;
    put16(p, 67);
    *p++ = static_cast<uint8_t>(t);
    for (int k = 0; k < 64; ++k) *p++ = static_cast<uint8_t>(qt.q[t][zz[k]]);
  }
  *p++ = 0xFF, *p++ = 0xC0;
  put16(p, 17);
  *p++ = 8;
  put16(p, h);
  put16(p, w);
  const uint8_t comps[] = {3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
  memcpy(p, comps, sizeof(comps));
  p += sizeof(comps);
  for (int t = 0; t < 4; ++t) {
    const int ac = t & 1, id = t >> 1;
    const uint8_t* bits = ac ? kAcBits[id] : kDcBits[id];
    const uint8_t* vals = ac ? kAcVals[id] : kDcVals;
    const int nv = ac ? 162 : 12;
    *p++ = 0xFF, *p++ = 0xC4;
    put16(p, 2 + 1 + 16 + nv);
    *p++ = static_cast<uint8_t>((ac << 4) | id);
    memcpy(p, bits, 16);
    memcpy(p + 16, vals, nv);
    p += 16 + nv;
  }
  const uint8_t sos[] = {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  memcpy(p, sos, sizeof(sos));
  return hd;
}

}  // namespace

extern "C" long long mdb_jpeg_scratch_bytes(int n, int h, int w, long long chunks) {
  if (n <= 0 || h < 1 || h > 65535 || w < 1 || w > 65535 || chunks < 0) return -1;
  return scratch_layout(n, h, w, chunks).total;
}

extern "C" int mdb_jpeg_encode_u8(const void* x, int n, int h, int w, int quality, void* scratch,
                                  long long scratch_bytes, void* out, long long out_bytes, long long* meta,
                                  void* stream) {
  if (!x || !scratch || !out || !meta) return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: null pointer");
  if (n <= 0 || n > 65535) return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: n = %d outside 1..65535", n);
  if (h < 1 || h > 65535 || w < 1 || w > 65535)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: %dx%d outside 1..65535", h, w);
  if (quality < 1 || quality > 100)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: quality %d outside 1..100", quality);
  if ((reinterpret_cast<uintptr_t>(scratch) & 255) || (reinterpret_cast<uintptr_t>(meta) & 7))
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: scratch must be 256-byte and meta 8-byte aligned");
  const Scratch s0 = scratch_layout(n, h, w, 0);
  long long chunks = scratch_bytes < s0.total ? -1 : (scratch_bytes - s0.total) / (kChunk + 8);
  while (chunks > 0 && scratch_layout(n, h, w, chunks).total > scratch_bytes) --chunks;  // the alignment padding
  if (chunks < n)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: scratch of %lld bytes, at least %lld needed",
                          scratch_bytes, scratch_layout(n, h, w, n).total);
  if (out_bytes < static_cast<long long>(n) * (MDB_JPEG_HEADER_BYTES + 3))
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_encode_u8: out of %lld bytes, at least %lld needed", out_bytes,
                          static_cast<long long>(n) * (MDB_JPEG_HEADER_BYTES + 3));
  const Scratch s = scratch_layout(n, h, w, chunks);
  uint8_t* base = static_cast<uint8_t*>(scratch);
  int16_t* coef = reinterpret_cast<int16_t*>(base + s.coef);
  int* mcu_bits = reinterpret_cast<int*>(base + s.mcu_bits);
  long long* mcu_first = reinterpret_cast<long long*>(base + s.mcu_first);
  ImageLayout* layout = reinterpret_cast<ImageLayout*>(base + s.layout);
  int* flags = reinterpret_cast<int*>(base + s.flags);
  long long* chunk_ff = reinterpret_cast<long long*>(base + s.chunk_ff);
  uint32_t* bitbuf = reinterpret_cast<uint32_t*>(base + s.bitbuf);
  const QuantTables qt = quant_tables(quality);
  const Header hdr = make_header(h, w, qt);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 mcu_grid(((h + 15) / 16) * ((w + 15) / 16), n), chunk_grid(kChunkGrid, n);
  const int mcus = static_cast<int>(mcu_grid.x);
  jpeg_coef_kernel<<<mcu_grid, 256, 0, st>>>(static_cast<const uint8_t*>(x), h, w, qt, coef);
  MDB_CHECK_LAUNCH("jpeg_coef_kernel");
  jpeg_blocks_kernel<false><<<mcu_grid, 192, 0, st>>>(coef, mcu_bits, nullptr, nullptr, nullptr, nullptr);
  MDB_CHECK_LAUNCH("jpeg_blocks_kernel<bits>");
  jpeg_scan_mcus_kernel<<<n, 1024, 0, st>>>(mcu_bits, mcus, mcu_first, layout);
  MDB_CHECK_LAUNCH("jpeg_scan_mcus_kernel");
  jpeg_layout_kernel<<<1, 1024, 0, st>>>(n, chunks, layout, flags, meta);
  MDB_CHECK_LAUNCH("jpeg_layout_kernel");
  jpeg_zero_kernel<<<264, 256, 0, st>>>(flags, reinterpret_cast<uint4*>(bitbuf));
  MDB_CHECK_LAUNCH("jpeg_zero_kernel");
  jpeg_blocks_kernel<true><<<mcu_grid, 192, 0, st>>>(coef, nullptr, mcu_first, layout, flags, bitbuf);
  MDB_CHECK_LAUNCH("jpeg_blocks_kernel<pack>");
  jpeg_ff_count_kernel<<<chunk_grid, 256, 0, st>>>(layout, flags, bitbuf, chunk_ff);
  MDB_CHECK_LAUNCH("jpeg_ff_count_kernel");
  jpeg_place_kernel<<<1, 1024, 0, st>>>(n, out_bytes, layout, flags, chunk_ff, meta);
  MDB_CHECK_LAUNCH("jpeg_place_kernel");
  jpeg_scatter_kernel<<<chunk_grid, 256, 0, st>>>(layout, flags, bitbuf, chunk_ff, meta, hdr,
                                                  static_cast<uint8_t*>(out));
  MDB_CHECK_LAUNCH("jpeg_scatter_kernel");
  return MDB_OK;
}
