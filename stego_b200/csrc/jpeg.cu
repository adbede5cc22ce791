// The JPEG round trip of the reference's crop script (src/crop_datasets.py:114-124: Image.save(path, "JPEG") with
// Pillow's defaults, then CroppedDataset's decode) on crop windows of decoded originals, and the training store's
// frames of the decoded crops, in two launches per batch of crops:
//
//   jpeg_codec_kernel: one CTA of 64 threads per 16 x 16 MCU of a crop (origin at the crop's top-left corner).
//     RGB -> YCbCr in fixed point, edge replication to the MCU grid, h2v2 chroma averaging with the alternating bias,
//     then per 8 x 8 block (4 luma, 1 Cb, 1 Cr) the islow FDCT, quantisation by the quality-75 tables, dequantisation
//     and the islow IDCT with the range limit.  Writes the decoded luma plane [h][w] and the two decoded chroma planes
//     [ceil(h / 2)][ceil(w / 2)] of the crop into the caller's workspace; padding samples are not written.
//   jpeg_store_rgb8_kernel: the decoded crop's pixels that get_transform(res, False, "center") reads (the index
//     tables of stego_b200/frames.py for the crop's size), each rebuilt from the workspace: h2v2 "fancy" (triangle)
//     chroma upsampling, or 2 x 2 replication when the chroma width is 1 or 2, then YCbCr -> RGB in fixed point.
//     Writes the raw bytes into row r0 + k of an n-row [n][3][res][res] store, as stego_frames_store_rgb8 does.
//
// Integer arithmetic only: libjpeg's islow DCT constants (13 fraction bits) and colour tables (16 fraction bits),
// restated by oracle/jpeg_oracle.py, which Pillow's own round trip judges.
#include <algorithm>

#include "common.cuh"
#include "host_util.h"

namespace stego {
namespace {

constexpr int JP_THREADS = 64;  // one MCU per CTA: 4 luma + 2 chroma blocks of 64 samples
constexpr int JP_REC = 9;       // int64 words per crop record
enum : int { J_SRC = 0, J_SH, J_SW, J_TOP, J_LEFT, J_H, J_W, J_TABLE, J_WS };

// ITU T.81 Annex K tables scaled for IJG quality 75 ((q * 50 + 50) / 100), natural order
__constant__ int kQuant[2][64] = {
    {8,  6,  5,  8,  12, 20, 26, 31, 6,  6,  7,  10, 13, 29, 30, 28, 7,  7,  8,  12, 20, 29,
     35, 28, 7,  9,  11, 15, 26, 44, 40, 31, 9,  11, 19, 28, 34, 55, 52, 39, 12, 18, 28, 32,
     41, 52, 57, 46, 25, 32, 39, 44, 52, 61, 60, 51, 36, 46, 48, 49, 56, 50, 52, 50},
    {9,  9,  12, 24, 50, 50, 50, 50, 9,  11, 13, 33, 50, 50, 50, 50, 12, 13, 28, 50, 50, 50,
     50, 50, 24, 33, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50,
     50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50, 50}};

constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// The odd-part rotation shared by the islow FDCT and IDCT (arguments in the FDCT's tmp4..tmp7 naming).
__device__ __forceinline__ void odd_part(int& t4, int& t5, int& t6, int& t7) {
  const int z1 = t4 + t7, z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * F1175;
  const int a1 = z1 * -F0899, a2 = z2 * -F2562, a3 = z3 * -F1961 + z5, a4 = z4 * -F0390 + z5;
  const int o4 = t4 * F0298 + a1 + a3, o5 = t5 * F2053 + a2 + a4, o6 = t6 * F3072 + a2 + a3,
            o7 = t7 * F1501 + a1 + a4;
  t4 = o4, t5 = o5, t6 = o6, t7 = o7;
}

// jpeg_fdct_islow along 8 samples d[0 * s] .. d[7 * s] in place (pass 1: rows, pass 2: columns).
template <bool PASS1>
__device__ __forceinline__ void fdct8(int* d, int s) {
  const int tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s], tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
  const int tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s], tmp3 = d[3 * s] + d[4 * s],
            tmp4 = d[3 * s] - d[4 * s];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  constexpr int sh = PASS1 ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS;
  if (PASS1) {
    d[0] = (tmp10 + tmp11) * (1 << PASS1_BITS);
    d[4 * s] = (tmp10 - tmp11) * (1 << PASS1_BITS);
  } else {
    d[0] = descale(tmp10 + tmp11, PASS1_BITS);
    d[4 * s] = descale(tmp10 - tmp11, PASS1_BITS);
  }
  const int z1 = (tmp12 + tmp13) * F0541;
  d[2 * s] = descale(z1 + tmp13 * F0765, sh);
  d[6 * s] = descale(z1 + tmp12 * -F1847, sh);
  int t4 = tmp4, t5 = tmp5, t6 = tmp6, t7 = tmp7;
  odd_part(t4, t5, t6, t7);
  d[7 * s] = descale(t4, sh);
  d[5 * s] = descale(t5, sh);
  d[3 * s] = descale(t6, sh);
  d[s] = descale(t7, sh);
}

// jpeg_idct_islow along 8 dequantised coefficients c[0 * s] .. c[7 * s] in place (pass 1: columns, pass 2: rows,
// before the + 128).
template <bool PASS1>
__device__ __forceinline__ void idct8(int* c, int s) {
  const int z1 = (c[2 * s] + c[6 * s]) * F0541;
  const int tmp2 = z1 + c[6 * s] * -F1847, tmp3 = z1 + c[2 * s] * F0765;
  const int tmp0 = (c[0] + c[4 * s]) * (1 << CONST_BITS), tmp1 = (c[0] - c[4 * s]) * (1 << CONST_BITS);
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  int t0 = c[7 * s], t1 = c[5 * s], t2 = c[3 * s], t3 = c[s];
  odd_part(t0, t1, t2, t3);
  constexpr int sh = PASS1 ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS + 3;
  c[0] = descale(tmp10 + t3, sh);
  c[7 * s] = descale(tmp10 - t3, sh);
  c[s] = descale(tmp11 + t2, sh);
  c[6 * s] = descale(tmp11 - t2, sh);
  c[2 * s] = descale(tmp12 + t1, sh);
  c[5 * s] = descale(tmp12 - t1, sh);
  c[3 * s] = descale(tmp13 + t0, sh);
  c[4 * s] = descale(tmp13 - t0, sh);
}

struct CropArgs {
  const unsigned char* staging;
  const long long* rec;  // [count][JP_REC]
  const int* tables;     // per record: res rows, then res columns of the crop
  unsigned char* ws;
  int res, quads;
};

__device__ __forceinline__ int ycc_y(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int ycc_cb(int r, int g, int b) {
  return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
}
__device__ __forceinline__ int ycc_cr(int r, int g, int b) {
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__global__ void __launch_bounds__(JP_THREADS) jpeg_codec_kernel(CropArgs a) {
  __shared__ int blk[6][64];  // luma blocks (tl, tr, bl, br), Cb, Cr
  const long long* r = a.rec + static_cast<size_t>(blockIdx.y) * JP_REC;
  const int h = static_cast<int>(r[J_H]), w = static_cast<int>(r[J_W]);
  const int mcu_w = (w + 15) >> 4, mcu_h = (h + 15) >> 4;
  if (static_cast<int>(blockIdx.x) >= mcu_w * mcu_h) return;
  const int my = blockIdx.x / mcu_w, mx = blockIdx.x - my * mcu_w;
  const long long SW = r[J_SW];
  const unsigned char* src = a.staging + r[J_SRC] + (r[J_TOP] * SW + r[J_LEFT]) * 3;
  const int t = threadIdx.x;
  const int ch = (h + 1) >> 1, cw = (w + 1) >> 1;
  // luma: 4 samples per thread, rows and columns replicated past the crop's edge
  for (int k = t; k < 256; k += JP_THREADS) {
    const int y = min((my << 4) + (k >> 4), h - 1), x = min((mx << 4) + (k & 15), w - 1);
    const unsigned char* p = src + (static_cast<long long>(y) * SW + x) * 3;
    const int bi = ((k >> 7) << 1) | ((k >> 3) & 1);  // block of (row k / 16, column k % 16)
    blk[bi][((k >> 4) & 7) * 8 + (k & 7)] = ycc_y(p[0], p[1], p[2]) - 128;
  }
  // chroma: one sample of each plane per thread.  Columns replicate at full resolution, rows to the 2-row group,
  // then the last chroma row repeats.
  {
    const int i = min((my << 3) + (t >> 3), ch - 1), j = (mx << 3) + (t & 7);
    int sb = 0, sr = 0;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int y = min(2 * i + dy, h - 1), x = min(2 * j + dx, w - 1);
        const unsigned char* p = src + (static_cast<long long>(y) * SW + x) * 3;
        sb += ycc_cb(p[0], p[1], p[2]);
        sr += ycc_cr(p[0], p[1], p[2]);
      }
    const int bias = 1 + (j & 1);
    blk[4][t] = ((sb + bias) >> 2) - 128;
    blk[5][t] = ((sr + bias) >> 2) - 128;
  }
  __syncthreads();
  const int b = t >> 3, l = t & 7;  // 48 threads: block b, row / column l
  if (b < 6) fdct8<true>(&blk[b][l * 8], 1);
  __syncthreads();
  if (b < 6) {
    int* col = &blk[b][l];
    fdct8<false>(col, 8);
    const int* q = kQuant[b >= 4];
#pragma unroll
    for (int v = 0; v < 8; ++v) {  // quantise (round half away from zero), dequantise
      const int qv = q[v * 8 + l], d = qv * 8, c = col[v * 8];
      const int m = (abs(c) + (d >> 1)) / d;
      col[v * 8] = (c < 0 ? -m : m) * qv;
    }
    idct8<true>(col, 8);
  }
  __syncthreads();
  if (b < 6) {
    int* row = &blk[b][l * 8];
    idct8<false>(row, 1);
    unsigned char* ws = a.ws + r[J_WS];
    int y, x0, pitch, rows;
    if (b < 4) {
      y = (my << 4) + ((b >> 1) << 3) + l, x0 = (mx << 4) + ((b & 1) << 3), pitch = w, rows = h;
    } else {
      y = (my << 3) + l, x0 = mx << 3, pitch = cw, rows = ch;
      ws += static_cast<long long>(h) * w + (b == 5 ? static_cast<long long>(ch) * cw : 0);
    }
    if (y < rows) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (x0 + k < pitch) ws[static_cast<long long>(y) * pitch + x0 + k] = static_cast<unsigned char>(
                                min(max(row[k] + 128, 0), 255));
    }
  }
}

// The decoder's upsampled chroma sample at pixel (y, x) of a plane c [ch][cw].
__device__ __forceinline__ int chroma_at(const unsigned char* c, int ch, int cw, int y, int x) {
  const int i = y >> 1, j = x >> 1;
  if (cw <= 2) return c[static_cast<long long>(i) * cw + j];
  const int near = (y & 1) ? min(i + 1, ch - 1) : max(i - 1, 0);
  const unsigned char* r0 = c + static_cast<long long>(i) * cw;
  const unsigned char* r1 = c + static_cast<long long>(near) * cw;
  const int jn = (x & 1) ? min(j + 1, cw - 1) : max(j - 1, 0);
  const int s = 3 * r0[j] + r1[j], sn = 3 * r0[jn] + r1[jn];
  return (3 * s + sn + 8 - (x & 1)) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_store_rgb8_kernel(CropArgs a, unsigned char* store, long long r0) {
  const int k = blockIdx.y;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= a.res * a.quads) return;
  const int y = idx / a.quads, x0 = (idx - y * a.quads) * 4;
  const long long* r = a.rec + static_cast<size_t>(k) * JP_REC;
  const int h = static_cast<int>(r[J_H]), w = static_cast<int>(r[J_W]);
  const int ch = (h + 1) >> 1, cw = (w + 1) >> 1;
  const int* t = a.tables + r[J_TABLE];
  const unsigned char* ly = a.ws + r[J_WS];
  const unsigned char* cb = ly + static_cast<long long>(h) * w;
  const unsigned char* cr = cb + static_cast<long long>(ch) * cw;
  const int sy = t[y];
  unsigned v[3][4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int x = x0 + q;
    const int sx = x < a.res ? t[a.res + x] : -1;
    if (sy < 0 || sx < 0) {
      v[0][q] = v[1][q] = v[2][q] = 0u;
      continue;
    }
    const int Y = ly[static_cast<long long>(sy) * w + sx];
    const int Cb = chroma_at(cb, ch, cw, sy, sx) - 128, Cr = chroma_at(cr, ch, cw, sy, sx) - 128;
    v[0][q] = min(max(Y + ((91881 * Cr + 32768) >> 16), 0), 255);
    v[1][q] = min(max(Y + ((-22554 * Cb - 46802 * Cr + 32768) >> 16), 0), 255);
    v[2][q] = min(max(Y + ((116130 * Cb + 32768) >> 16), 0), 255);
  }
  const size_t plane = static_cast<size_t>(a.res) * a.res;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    unsigned char* o = store + (static_cast<size_t>(r0 + k) * 3 + c) * plane + static_cast<size_t>(y) * a.res + x0;
    if ((a.res & 3) == 0) {
      *reinterpret_cast<uchar4*>(o) = make_uchar4(v[c][0], v[c][1], v[c][2], v[c][3]);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (x0 + q < a.res) o[q] = static_cast<unsigned char>(v[c][q]);
    }
  }
}

// Checks the crop staging on its host copy (records, windows, tables, image extents and workspace extents) and fills
// `a`; *max_mcus: the largest MCU count of a crop.
int check_crops(const char* who, const void* host, const void* dev, long long bytes, long long table_words, int count,
                int res, unsigned char* ws, long long ws_bytes, CropArgs& a, int* max_mcus) {
  STEGO_CHECK_ARG(host && dev && ws, "%s: null pointer", who);
  STEGO_CHECK_ARG(count >= 1 && count <= 65535, "%s: count=%d crops (1..65535)", who, count);
  STEGO_CHECK_ARG(res >= 0 && res <= 8192, "%s: res=%d (0..8192)", who, res);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(dev) % 8 == 0, "%s: staging must be 8-byte aligned", who);
  STEGO_CHECK_ARG(table_words >= 2ll * res && table_words <= (1ll << 40), "%s: %lld table words", who, table_words);
  const long long head = 8ll * JP_REC * count, data = head + 4 * table_words;
  STEGO_CHECK_ARG(bytes >= data, "%s: %lld staging bytes hold no %lld-byte record and table block", who, bytes, data);
  const long long* rec = static_cast<const long long*>(host);
  const int* tables = reinterpret_cast<const int*>(static_cast<const char*>(host) + head);
  *max_mcus = 0;
  for (int k = 0; k < count; ++k) {
    const long long* r = rec + static_cast<size_t>(k) * JP_REC;
    const long long off = r[J_SRC], SH = r[J_SH], SW = r[J_SW], top = r[J_TOP], left = r[J_LEFT], h = r[J_H],
                    w = r[J_W], t = r[J_TABLE], wo = r[J_WS];
    STEGO_CHECK_ARG(SH >= 1 && SW >= 1 && SH <= (1ll << 20) && SW <= (1ll << 20), "%s: crop %d's source is %lld x %lld",
                    who, k, SH, SW);
    STEGO_CHECK_ARG(off >= data && off <= bytes && SH * SW * 3 <= bytes - off,
                    "%s: crop %d's source (%lld bytes at offset %lld) lies outside the staging data [%lld, %lld)", who,
                    k, SH * SW * 3, off, data, bytes);
    STEGO_CHECK_ARG(h >= 1 && w >= 1 && top >= 0 && left >= 0 && top + h <= SH && left + w <= SW,
                    "%s: crop %d (top %lld, left %lld, %lld x %lld) is not inside its %lld x %lld source", who, k, top,
                    left, h, w, SH, SW);
    const long long need = h * w + 2 * ((h + 1) / 2) * ((w + 1) / 2);
    STEGO_CHECK_ARG(wo >= 0 && wo <= ws_bytes - need, "%s: crop %d's %lld workspace bytes at %lld exceed %lld", who, k,
                    need, wo, ws_bytes);
    const long long mcus = ((h + 15) / 16) * ((w + 15) / 16);
    STEGO_CHECK_ARG(mcus <= 0x7fffffffll, "%s: crop %d has %lld MCUs", who, k, mcus);
    *max_mcus = std::max(*max_mcus, static_cast<int>(mcus));
    if (res > 0) {
      STEGO_CHECK_ARG(t >= 0 && t <= table_words - 2ll * res, "%s: crop %d's tables start at word %lld of %lld", who,
                      k, t, table_words);
      for (int i = 0; i < res; ++i) {
        const int sy = tables[t + i], sx = tables[t + res + i];
        STEGO_CHECK_ARG(sy >= -1 && sy < h && sx >= -1 && sx < w,
                        "%s: crop %d (%lld x %lld): output %d reads row %d / column %d", who, k, h, w, i, sy, sx);
      }
    }
  }
  a.staging = static_cast<const unsigned char*>(dev);
  a.rec = static_cast<const long long*>(dev);
  a.tables = reinterpret_cast<const int*>(static_cast<const unsigned char*>(dev) + head);
  a.ws = ws;
  a.res = res;
  a.quads = (res + 3) / 4;
  return STEGO_OK;
}

}  // namespace
}  // namespace stego

using namespace stego;

// C-ABI: see include/stego_b200.h for the contract.
extern "C" int stego_jpeg_crops_codec(const void* staging_host, const void* staging_dev, long long bytes,
                                      long long table_words, int count, unsigned char* workspace,
                                      long long workspace_bytes, void* stream_) {
  CropArgs a;
  int max_mcus = 0;
  const int rc = check_crops("stego_jpeg_crops_codec", staging_host, staging_dev, bytes, table_words, count, 0,
                             workspace, workspace_bytes, a, &max_mcus);
  if (rc != STEGO_OK) return rc;
  jpeg_codec_kernel<<<dim3(max_mcus, count), JP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(a);
  STEGO_CHECK_LAUNCH("jpeg_codec_kernel launch");
  return STEGO_OK;
}

extern "C" int stego_jpeg_crops_store_rgb8(const void* staging_host, const void* staging_dev, long long bytes,
                                           long long table_words, int count, int res, const unsigned char* workspace,
                                           long long workspace_bytes, unsigned char* store, long long n, long long r0,
                                           void* stream_) {
  const char* who = "stego_jpeg_crops_store_rgb8";
  STEGO_CHECK_ARG(res >= 1, "%s: res=%d (1..8192)", who, res);
  CropArgs a;
  int max_mcus = 0;
  int rc = check_crops(who, staging_host, staging_dev, bytes, table_words, count, res,
                       const_cast<unsigned char*>(workspace), workspace_bytes, a, &max_mcus);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(store, "%s: null store", who);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(store) % 16 == 0, "%s: store must be 16-byte aligned", who);
  STEGO_CHECK_ARG(n >= 1 && r0 >= 0 && r0 <= n - count, "%s: rows %lld .. %lld of a %lld-row store", who, r0,
                  r0 + count, n);
  cudaPointerAttributes attr;
  const cudaError_t e = cudaPointerGetAttributes(&attr, store);
  if (e != cudaSuccess) return cuda_fail(e, who);
  unsigned char* dev = store;
  if (attr.type == cudaMemoryTypeHost) {
    STEGO_CHECK_ARG(attr.devicePointer, "%s: store is host memory that is not pinned", who);
    dev = static_cast<unsigned char*>(attr.devicePointer);
  } else {
    STEGO_CHECK_ARG(attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged,
                    "%s: store is neither device memory nor pinned host memory", who);
  }
  const dim3 grid(static_cast<unsigned>((static_cast<long long>(res) * a.quads + 255) / 256), count);
  jpeg_store_rgb8_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(a, dev, r0);
  STEGO_CHECK_LAUNCH("jpeg_store_rgb8_kernel launch");
  return STEGO_OK;
}
