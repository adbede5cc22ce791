// The loader transform of the reference (src/utils.py:165-183 get_transform) on decoded images and label maps of any
// size, for a batch in one launch each:
//
//     frame = Normalize(mean, std) . ToTensor . CenterCrop(res) . Resize(res, NEAREST)  (RGB image)
//     label = lut[ ToTargetTensor . CenterCrop(res) . Resize(res, NEAREST)  (L / P label map) ]
//
// The host (stego_b200/frames.py) computes Pillow's nearest-neighbour source index of every output row and column with
// the crop offset folded in, and packs the per-image records, those tables and the image bytes into one staging buffer.
// Each output pixel is then one gather: no resized intermediate is written, and only the source pixels the output
// needs are read.  A table entry of -1 is a pixel Pillow leaves at its fill value 0.
//
// frames_rgb8_kernel: one thread per 4 output pixels of a row, all three channels; the value is
//   ((float)x / 255 - mean[c]) / std[c], ToTensor's div(255) then Normalize's sub_ and div_, each rounded as torch
//   rounds it on the CPU (true divisions, no contraction).  float4 stores when res % 4 == 0.
// labels_u8_kernel: the same gather on one byte per pixel, then the optional 256-entry int64 table (shared memory),
//   written as int64; two 16-byte stores per thread when res % 4 == 0.
#include "common.cuh"
#include "host_util.h"

namespace stego {

constexpr int FR_THREADS = 256, FR_PIX = 4, FR_REC = 4;  // output pixels per thread; int64 words per record
enum : int { R_OFFSET = 0, R_H, R_W, R_TABLE };

struct FrameArgs {
  const unsigned char* staging;
  const long long* rec;  // [B][FR_REC]
  const int* tables;     // per record: res rows, then res columns
  int res, quads;        // quads = ceil(res / 4)
};

// The source pixel of output (y, x0 + k), k < FR_PIX, as a pointer to its first byte (nullptr: Pillow's fill).
template <int C>
__device__ __forceinline__ void gather(const FrameArgs& a, int b, int y, int x0, const unsigned char* (&src)[FR_PIX]) {
  const long long* r = a.rec + static_cast<size_t>(b) * FR_REC;
  const long long W = r[R_W];
  const int* t = a.tables + r[R_TABLE];
  const int sy = t[y];
  const unsigned char* row = sy >= 0 ? a.staging + r[R_OFFSET] + sy * W * C : nullptr;
#pragma unroll
  for (int k = 0; k < FR_PIX; ++k) {
    const int x = x0 + k;
    const int sx = x < a.res ? t[a.res + x] : -1;
    src[k] = (row && sx >= 0) ? row + static_cast<long long>(sx) * C : nullptr;
  }
}

__global__ void __launch_bounds__(FR_THREADS) frames_rgb8_kernel(FrameArgs a, float m0, float m1, float m2, float s0,
                                                                  float s1, float s2, float* out) {
  const int b = blockIdx.y;
  const int idx = blockIdx.x * FR_THREADS + threadIdx.x;
  if (idx >= a.res * a.quads) return;
  const int y = idx / a.quads, x0 = (idx - y * a.quads) * FR_PIX;
  const unsigned char* src[FR_PIX];
  gather<3>(a, b, y, x0, src);
  const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
  const size_t plane = static_cast<size_t>(a.res) * a.res;
  float* o = out + static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(y) * a.res + x0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v[FR_PIX];
#pragma unroll
    for (int k = 0; k < FR_PIX; ++k) {
      const float x = src[k] ? static_cast<float>(src[k][c]) : 0.0f;
      v[k] = __fdiv_rn(__fsub_rn(__fdiv_rn(x, 255.0f), mean[c]), stdv[c]);
    }
    float* oc = o + c * plane;
    if ((a.res & (FR_PIX - 1)) == 0) {
      *reinterpret_cast<float4*>(oc) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int k = 0; k < FR_PIX; ++k)
        if (x0 + k < a.res) oc[k] = v[k];
    }
  }
}

__global__ void __launch_bounds__(FR_THREADS) labels_u8_kernel(FrameArgs a, const long long* lut, long long* out) {
  __shared__ long long table[256];
  if (lut) {
    for (int i = threadIdx.x; i < 256; i += FR_THREADS) table[i] = lut[i];
    __syncthreads();
  }
  const int b = blockIdx.y;
  const int idx = blockIdx.x * FR_THREADS + threadIdx.x;
  if (idx >= a.res * a.quads) return;
  const int y = idx / a.quads, x0 = (idx - y * a.quads) * FR_PIX;
  const unsigned char* src[FR_PIX];
  gather<1>(a, b, y, x0, src);
  long long v[FR_PIX];
#pragma unroll
  for (int k = 0; k < FR_PIX; ++k) {
    const int id = src[k] ? *src[k] : 0;
    v[k] = lut ? table[id] : id;
  }
  long long* o = out + (static_cast<size_t>(b) * a.res + y) * a.res + x0;
  if ((a.res & (FR_PIX - 1)) == 0) {
    reinterpret_cast<longlong2*>(o)[0] = make_longlong2(v[0], v[1]);
    reinterpret_cast<longlong2*>(o)[1] = make_longlong2(v[2], v[3]);
  } else {
#pragma unroll
    for (int k = 0; k < FR_PIX; ++k)
      if (x0 + k < a.res) o[k] = v[k];
  }
}

// Checks the staging layout on its host copy (records, tables and every image inside the buffer) and fills `a`.
static int check_staging(const char* who, const void* host, const void* dev, long long bytes, int B, int res,
                         long long table_words, int channels, FrameArgs& a) {
  STEGO_CHECK_ARG(host && dev, "%s: null staging pointer", who);
  STEGO_CHECK_ARG(B >= 1 && B <= 65535, "%s: B=%d (1..65535)", who, B);
  STEGO_CHECK_ARG(res >= 1 && res <= 8192, "%s: res=%d (1..8192)", who, res);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(dev) % 8 == 0, "%s: staging must be 8-byte aligned", who);
  const long long head = 8ll * FR_REC * B;
  STEGO_CHECK_ARG(table_words >= 2ll * res && table_words <= (1ll << 40),
                  "%s: %lld table words (at least 2 res = %d)", who, table_words, 2 * res);
  const long long data = head + 4 * table_words;
  STEGO_CHECK_ARG(bytes >= data, "%s: %lld staging bytes hold no %lld-byte record and table block", who, bytes, data);
  const long long* rec = static_cast<const long long*>(host);
  const int* tables = reinterpret_cast<const int*>(static_cast<const char*>(host) + head);
  for (int b = 0; b < B; ++b) {
    const long long* r = rec + static_cast<size_t>(b) * FR_REC;
    const long long off = r[R_OFFSET], H = r[R_H], W = r[R_W], t = r[R_TABLE];
    STEGO_CHECK_ARG(H >= 1 && W >= 1 && H <= (1ll << 20) && W <= (1ll << 20), "%s: image %d is %lld x %lld (1..2^20)",
                    who, b, H, W);
    STEGO_CHECK_ARG(off >= data && off <= bytes && H * W * channels <= bytes - off,
                    "%s: image %d (%lld bytes at offset %lld) lies outside the %lld-byte staging data [%lld, %lld)",
                    who, b, H * W * channels, off, bytes, data, bytes);
    STEGO_CHECK_ARG(t >= 0 && t <= table_words - 2ll * res, "%s: image %d's tables start at word %lld of %lld", who,
                    b, t, table_words);
    for (int i = 0; i < res; ++i) {
      const int sy = tables[t + i], sx = tables[t + res + i];
      STEGO_CHECK_ARG(sy >= -1 && sy < H && sx >= -1 && sx < W,
                      "%s: image %d (%lld x %lld): output %d reads row %d / column %d", who, b, H, W, i, sy, sx);
    }
  }
  a.staging = static_cast<const unsigned char*>(dev);
  a.rec = static_cast<const long long*>(dev);
  a.tables = reinterpret_cast<const int*>(static_cast<const unsigned char*>(dev) + head);
  a.res = res;
  a.quads = (res + FR_PIX - 1) / FR_PIX;
  return STEGO_OK;
}

static dim3 frames_grid(const FrameArgs& a, int B) {
  return dim3(static_cast<unsigned>((static_cast<long long>(a.res) * a.quads + FR_THREADS - 1) / FR_THREADS), B);
}

}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contract.
extern "C" int stego_frames_rgb8(const void* staging_host, const void* staging_dev, long long bytes,
                                 long long table_words, int B, int res, float mean0, float mean1, float mean2,
                                 float std0, float std1, float std2, float* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(out, "stego_frames_rgb8: null output");
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0, "stego_frames_rgb8: out must be 16-byte aligned");
  FrameArgs a;
  const int rc = check_staging("stego_frames_rgb8", staging_host, staging_dev, bytes, B, res, table_words, 3, a);
  if (rc != STEGO_OK) return rc;
  frames_rgb8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, mean0, mean1, mean2, std0, std1, std2, out);
  STEGO_CHECK_LAUNCH("frames_rgb8_kernel launch");
  return STEGO_OK;
}

extern "C" int stego_labels_u8(const void* staging_host, const void* staging_dev, long long bytes,
                               long long table_words, int B, int res, const long long* lut, long long* out,
                               void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  STEGO_CHECK_ARG(out, "stego_labels_u8: null output");
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0, "stego_labels_u8: out must be 16-byte aligned");
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(lut) % 8 == 0, "stego_labels_u8: lut must be 8-byte aligned");
  FrameArgs a;
  const int rc = check_staging("stego_labels_u8", staging_host, staging_dev, bytes, B, res, table_words, 1, a);
  if (rc != STEGO_OK) return rc;
  labels_u8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, lut, out);
  STEGO_CHECK_LAUNCH("labels_u8_kernel launch");
  return STEGO_OK;
}
