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
// frames_rgb8_kernel<Op>: one thread per 4 output pixels of a row, all three channels.  FrameOut writes
//   ((float)x / 255 - mean[c]) / std[c], ToTensor's div(255) then Normalize's sub_ and div_, each rounded as torch
//   rounds it on the CPU (true divisions, no contraction); float4 stores when res % 4 == 0.  StoreOut writes the raw
//   bytes into row r0 + b of a resident store (stego_b200/dataset.py).
// labels_u8_kernel<Op>: the same gather on one byte per pixel, then the optional 256-entry int64 table (shared memory);
//   LabelOut writes int64 (two 16-byte stores per thread when res % 4 == 0), StoreOut the raw bytes.
//   With 7-word records (stego_store_rows_u8) each record carries its own output size and destination: the whole
//   Resize(res) output of an image, no crop, which RowOut writes as the uint8 [C][oh][ow] row of a ragged store.
// dataset_batch_kernel: a training batch from the resident store, one sample per blockIdx.y and 16 bytes per thread:
//   the frame through the same normalisation as FrameOut (fp32, or the bf16 round of it), the label through a
//   256-entry int64 table, and the data set's mask of that label.  The evaluation-set batches (stego_evalset_batch,
//   stego_b200/evalset.py) are the same kernel with a third mask rule, bool (label >= 0) for Coco.  The kernel is
//   templated on its row addressing: FixedRows reads [n][3][res][res] rows by index, WindowRows (stego_store_batch_window)
//   a res x res window of a ragged row.
#include "common.cuh"
#include "host_util.h"

namespace stego {

// output pixels per thread; int64 words per record (res x res outputs) and per ragged-row record
constexpr int FR_THREADS = 256, FR_PIX = 4, FR_REC = 4, FR_REC_ROWS = 7;
enum : int { R_OFFSET = 0, R_H, R_W, R_TABLE, R_OH, R_OW, R_DEST };

struct FrameArgs {
  const unsigned char* staging;
  const long long* rec;  // [B][rec_words]
  const int* tables;     // per record: its output rows' source rows, then its output columns' source columns
  int res, rec_words;
  int rows, quads;       // the grid: the tallest output's rows by the widest one's quads (ceil(width / 4))
};

// Output size of record r: res x res, or its own (oh, ow) with ragged-row records.
__device__ __forceinline__ void out_size(const FrameArgs& a, const long long* r, int& oh, int& ow) {
  oh = a.rec_words == FR_REC ? a.res : static_cast<int>(r[R_OH]);
  ow = a.rec_words == FR_REC ? a.res : static_cast<int>(r[R_OW]);
}

// The source pixel of output (y, x0 + k), k < FR_PIX, as a pointer to its first byte (nullptr: Pillow's fill).
template <int C>
__device__ __forceinline__ void gather(const FrameArgs& a, const long long* r, int oh, int ow, int y, int x0,
                                       const unsigned char* (&src)[FR_PIX]) {
  const long long W = r[R_W];
  const int* t = a.tables + r[R_TABLE];
  const int sy = t[y];
  const unsigned char* row = sy >= 0 ? a.staging + r[R_OFFSET] + sy * W * C : nullptr;
#pragma unroll
  for (int k = 0; k < FR_PIX; ++k) {
    const int x = x0 + k;
    const int sx = x < ow ? t[oh + x] : -1;
    src[k] = (row && sx >= 0) ? row + static_cast<long long>(sx) * C : nullptr;
  }
}

// ToTensor's div(255) then Normalize's sub_ and div_ of one byte, each an IEEE fp32 operation: the one definition both
// the loader frames and the resident-store batches use.
__device__ __forceinline__ float normalize_u8(unsigned x, float mean, float stdv) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(x), 255.0f), mean), stdv);
}

struct Norm {
  float mean[3], stdv[3];
};

// Output ops of the gather kernels: put(r, b, c, y, x0, v) writes output pixels (y, x0 .. x0 + FR_PIX) of channel c of
// image b (record r), v[k] being the gathered byte (frames) or its table value (labels); pixels past the output's width
// are not written.
struct FrameOut {  // fp32 [B][3][res][res], normalised
  Norm n;
  float* out;
  int res;
  __device__ __forceinline__ void put(const long long*, int b, int c, int y, int x0, const unsigned (&x)[FR_PIX]) const {
    float v[FR_PIX];
#pragma unroll
    for (int k = 0; k < FR_PIX; ++k) v[k] = normalize_u8(x[k], n.mean[c], n.stdv[c]);
    const size_t plane = static_cast<size_t>(res) * res;
    float* o = out + (static_cast<size_t>(b) * 3 + c) * plane + static_cast<size_t>(y) * res + x0;
    if ((res & (FR_PIX - 1)) == 0) {
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int k = 0; k < FR_PIX; ++k)
        if (x0 + k < res) o[k] = v[k];
    }
  }
};

struct LabelOut {  // int64 [B][res][res]
  long long* out;
  int res;
  __device__ __forceinline__ void put(const long long*, int b, int, int y, int x0, const long long (&v)[FR_PIX]) const {
    long long* o = out + (static_cast<size_t>(b) * res + y) * res + x0;
    if ((res & (FR_PIX - 1)) == 0) {
      reinterpret_cast<longlong2*>(o)[0] = make_longlong2(v[0], v[1]);
      reinterpret_cast<longlong2*>(o)[1] = make_longlong2(v[2], v[3]);
    } else {
#pragma unroll
      for (int k = 0; k < FR_PIX; ++k)
        if (x0 + k < res) o[k] = v[k];
    }
  }
};

struct StoreOut {  // uint8 rows [n][channels][res][res] of a resident store; image b goes to row r0 + b
  unsigned char* out;
  long long r0;
  int channels, res;
  template <typename T>
  __device__ __forceinline__ void put(const long long*, int b, int c, int y, int x0, const T (&v)[FR_PIX]) const {
    const size_t plane = static_cast<size_t>(res) * res;
    unsigned char* o = out + (static_cast<size_t>(r0 + b) * channels + c) * plane + static_cast<size_t>(y) * res + x0;
    if ((res & (FR_PIX - 1)) == 0) {
      *reinterpret_cast<uchar4*>(o) = make_uchar4(static_cast<unsigned char>(v[0]), static_cast<unsigned char>(v[1]),
                                                  static_cast<unsigned char>(v[2]), static_cast<unsigned char>(v[3]));
    } else {
#pragma unroll
      for (int k = 0; k < FR_PIX; ++k)
        if (x0 + k < res) o[k] = static_cast<unsigned char>(v[k]);
    }
  }
};

struct RowOut {  // uint8 [channels][oh][ow] rows of a ragged store, each at its record's byte offset R_DEST
  unsigned char* out;
  template <typename T>
  __device__ __forceinline__ void put(const long long* r, int, int c, int y, int x0, const T (&v)[FR_PIX]) const {
    const long long oh = r[R_OH], ow = r[R_OW];
    unsigned char* o = out + r[R_DEST] + (c * oh + y) * ow + x0;
#pragma unroll
    for (int k = 0; k < FR_PIX; ++k)
      if (x0 + k < ow) o[k] = static_cast<unsigned char>(v[k]);
  }
};

template <class Op>
__global__ void __launch_bounds__(FR_THREADS) frames_rgb8_kernel(FrameArgs a, Op op) {
  const int b = blockIdx.y;
  const int idx = blockIdx.x * FR_THREADS + threadIdx.x;
  if (idx >= a.rows * a.quads) return;
  const long long* r = a.rec + static_cast<size_t>(b) * a.rec_words;
  int oh, ow;
  out_size(a, r, oh, ow);
  const int y = idx / a.quads, x0 = (idx - y * a.quads) * FR_PIX;
  if (y >= oh || x0 >= ow) return;
  const unsigned char* src[FR_PIX];
  gather<3>(a, r, oh, ow, y, x0, src);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    unsigned x[FR_PIX];
#pragma unroll
    for (int k = 0; k < FR_PIX; ++k) x[k] = src[k] ? src[k][c] : 0u;
    op.put(r, b, c, y, x0, x);
  }
}

template <class Op>
__global__ void __launch_bounds__(FR_THREADS) labels_u8_kernel(FrameArgs a, const long long* lut, Op op) {
  __shared__ long long table[256];
  if (lut) {
    for (int i = threadIdx.x; i < 256; i += FR_THREADS) table[i] = lut[i];
    __syncthreads();
  }
  const int b = blockIdx.y;
  const int idx = blockIdx.x * FR_THREADS + threadIdx.x;
  if (idx >= a.rows * a.quads) return;
  const long long* r = a.rec + static_cast<size_t>(b) * a.rec_words;
  int oh, ow;
  out_size(a, r, oh, ow);
  const int y = idx / a.quads, x0 = (idx - y * a.quads) * FR_PIX;
  if (y >= oh || x0 >= ow) return;
  const unsigned char* src[FR_PIX];
  gather<1>(a, r, oh, ow, y, x0, src);
  long long v[FR_PIX];
#pragma unroll
  for (int k = 0; k < FR_PIX; ++k) {
    const int id = src[k] ? *src[k] : 0;
    v[k] = lut ? table[id] : id;
  }
  op.put(r, b, 0, y, x0, v);
}

// ---- training batches from a resident store ------------------------------------------------------------------------
constexpr int DB_THREADS = 256, DB_BYTES = 16;  // 16 store bytes (one 16-byte load) per thread
// bool (label == -1): CroppedDataset, CityscapesSeg; fp32 (label > 0): DirectoryDataset, Potsdam, PotsdamRaw;
// bool (label >= 0): Coco (evaluation sets only)
enum : int { MASK_IS_IGNORE = 0, MASK_IS_POSITIVE = 1, MASK_IS_NONNEG = 2 };

struct BatchArgs {
  const long long* lut;         // [256]
  Norm n;
  void* img;                    // [count][3][res][res] fp32 or bf16
  long long* label;             // [count][res][res]
  void* mask;                   // [count][res][res] bool or fp32
  int res, img_chunks, lab_chunks;
};

__device__ __forceinline__ void store16(float* o, const float (&v)[DB_BYTES]) {
#pragma unroll
  for (int k = 0; k < DB_BYTES; k += 4) *reinterpret_cast<float4*>(o + k) = make_float4(v[k], v[k + 1], v[k + 2], v[k + 3]);
}
__device__ __forceinline__ void store16(bf16* o, const float (&v)[DB_BYTES]) {
#pragma unroll
  for (int k = 0; k < DB_BYTES; k += 8) {
    uint4 w;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&w);
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[k + 2 * j], v[k + 2 * j + 1]);
    *reinterpret_cast<uint4*>(o + k) = w;
  }
}
__device__ __forceinline__ void put1(float* o, float v) { *o = v; }
__device__ __forceinline__ void put1(bf16* o, float v) { *o = __float2bfloat16_rn(v); }

// The 16 bytes at element e0 of a row of `len` bytes (fewer past its end), as 16-byte loads when rows are 16-byte
// multiples (res % 4 == 0), byte loads otherwise.
__device__ __forceinline__ void load16(const unsigned char* row, long long e0, long long len, bool vec,
                                       unsigned (&x)[DB_BYTES]) {
  if (vec) {
    const uint4 w = *reinterpret_cast<const uint4*>(row + e0);
    const unsigned words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < DB_BYTES; ++k) x[k] = (words[k >> 2] >> (8 * (k & 3))) & 0xffu;
  } else {
#pragma unroll
    for (int k = 0; k < DB_BYTES; ++k) x[k] = e0 + k < len ? row[e0 + k] : 0u;
  }
}

// The 16 bytes at p, any alignment: the aligned 16-byte block holding p and, unless p is aligned, the next one, shifted
// down by p's offset in its block.  The second block is read only when it holds some of the 16 bytes, so a buffer whose
// base is 16-byte aligned and whose size is a multiple of 16 is never read past.
__device__ __forceinline__ void load16_shifted(const unsigned char* p, unsigned (&x)[DB_BYTES]) {
  const uintptr_t at = reinterpret_cast<uintptr_t>(p);
  const uint4* q = reinterpret_cast<const uint4*>(at & ~static_cast<uintptr_t>(15));
  const int sh = static_cast<int>(at & 15);
  const uint4 lo = q[0];
  const uint4 hi = sh ? q[1] : make_uint4(0u, 0u, 0u, 0u);
  const unsigned w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  const int ws = sh >> 2;
  const unsigned bs = 8u * (sh & 3);
  unsigned v[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) v[j] = ws == 0 ? w[j] : ws == 1 ? w[j + 1] : ws == 2 ? w[j + 2] : w[j + 3];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned word = __funnelshift_r(v[j], v[j + 1], bs);
#pragma unroll
    for (int k = 0; k < 4; ++k) x[4 * j + k] = (word >> (8 * k)) & 0xffu;
  }
}

// Row addressing of dataset_batch_kernel.  fetch(s) runs in one thread and makes the block's only reads of sample s's
// (host-resident) record; image() / label() load the store bytes behind output elements e0 .. e0 + 16 of the sample's
// frame [3][res][res] / label map [res][res], 0 past its end.
struct FixedRows {  // images [n][3][res][res], labels [n][res][res]; the record is the row index
  const unsigned char* images;
  const unsigned char* labels;  // or null: every pixel reads id 0
  const long long* index;       // [count]
  int res;
  struct Row {
    long long row;
  };
  __device__ __forceinline__ Row fetch(int s) const { return Row{index[s]}; }
  __device__ __forceinline__ void image(const Row& r, long long e0, unsigned (&x)[DB_BYTES]) const {
    const long long len = 3ll * res * res;
    load16(images + r.row * len, e0, len, (res & 3) == 0, x);  // res % 4 == 0: every row is a 16-byte multiple
  }
  __device__ __forceinline__ void label(const Row& r, long long e0, unsigned (&x)[DB_BYTES]) const {
    const long long plane = static_cast<long long>(res) * res;
    load16(labels + r.row * plane, e0, plane, (res & 3) == 0, x);
  }
};

// A res x res window of a ragged row: the 16 output elements lie in one output row when res % 16 == 0 and are then 16
// consecutive source bytes at any alignment (load16_shifted: two aligned 16-byte loads and a funnel shift, instead of
// 16 byte loads, which read a host-resident store over PCIe once per byte); otherwise each byte is addressed alone.
__device__ __forceinline__ void window_load(const unsigned char* base, long long cstride, long long stride, int res,
                                            long long e0, int channels, unsigned (&x)[DB_BYTES]) {
  const long long plane = static_cast<long long>(res) * res;
  if ((res & 15) == 0) {
    const long long c = e0 / plane, yx = e0 - c * plane, y = yx / res;
    load16_shifted(base + c * cstride + y * stride + (yx - y * res), x);
  } else {
#pragma unroll
    for (int k = 0; k < DB_BYTES; ++k) {
      const long long e = e0 + k;
      if (e >= channels * plane) {
        x[k] = 0u;
      } else {
        const long long c = e / plane, yx = e - c * plane, y = yx / res;
        x[k] = base[c * cstride + y * stride + (yx - y * res)];
      }
    }
  }
}

struct WindowRows {  // a ragged store: row i is image uint8 [3][oh][ow] and label uint8 [lh][lw] at its byte offsets
  const unsigned char* images;
  const unsigned char* labels;  // or null: every pixel reads id 0
  const long long* rec;         // [count][WIN_REC]: row, image top, left, label top, left
  const long long* rows;        // [n][ROW_WORDS]: image byte offset, oh, ow, label byte offset, lh, lw
  int res;
  struct Row {
    long long img, img_plane, ow, lab, lw;  // window origins (bytes), the image's channel stride, the row strides
  };
  __device__ __forceinline__ Row fetch(int s) const;
  __device__ __forceinline__ void image(const Row& r, long long e0, unsigned (&x)[DB_BYTES]) const {
    window_load(images + r.img, r.img_plane, r.ow, res, e0, 3, x);
  }
  __device__ __forceinline__ void label(const Row& r, long long e0, unsigned (&x)[DB_BYTES]) const {
    window_load(labels + r.lab, 0, r.lw, res, e0, 1, x);
  }
};

constexpr int WIN_REC = 5, ROW_WORDS = 6;
enum : int { W_ROW = 0, W_TOP, W_LEFT, W_LTOP, W_LLEFT };
enum : int { RT_IMG = 0, RT_OH, RT_OW, RT_LAB, RT_LH, RT_LW };

__device__ __forceinline__ WindowRows::Row WindowRows::fetch(int s) const {
  const long long* q = rec + static_cast<size_t>(s) * WIN_REC;
  const long long* t = rows + q[W_ROW] * ROW_WORDS;
  Row r;
  r.ow = t[RT_OW];
  r.img_plane = t[RT_OH] * r.ow;
  r.img = t[RT_IMG] + q[W_TOP] * r.ow + q[W_LEFT];
  r.lw = t[RT_LW];
  r.lab = t[RT_LAB] + q[W_LTOP] * r.lw + q[W_LLEFT];
  return r;
}

template <typename T, int MASK, class Rows>
__global__ void __launch_bounds__(DB_THREADS) dataset_batch_kernel(BatchArgs a, Rows rows) {
  __shared__ long long table[256];
  __shared__ typename Rows::Row row;
  for (int i = threadIdx.x; i < 256; i += DB_THREADS) table[i] = a.lut[i];
  if (threadIdx.x == 0) row = rows.fetch(blockIdx.y);  // one read of the (possibly host-resident) record
  __syncthreads();
  const int s = blockIdx.y;
  const typename Rows::Row r = row;
  const long long plane = static_cast<long long>(a.res) * a.res;
  const bool vec = (a.res & 3) == 0;  // then every output plane is a multiple of 16 elements
  const int chunk = blockIdx.x * DB_THREADS + threadIdx.x;
  unsigned x[DB_BYTES];
  if (chunk < a.img_chunks) {
    const long long e0 = static_cast<long long>(chunk) * DB_BYTES, len = 3 * plane;
    rows.image(r, e0, x);
    T* o = static_cast<T*>(a.img) + s * len + e0;
    if (vec) {  // the 16 elements lie in one channel plane
      const int c = static_cast<int>(e0 / plane);
      float v[DB_BYTES];
#pragma unroll
      for (int k = 0; k < DB_BYTES; ++k) v[k] = normalize_u8(x[k], a.n.mean[c], a.n.stdv[c]);
      store16(o, v);
    } else {
#pragma unroll
      for (int k = 0; k < DB_BYTES; ++k) {
        if (e0 + k >= len) break;
        const int c = static_cast<int>((e0 + k) / plane);
        put1(o + k, normalize_u8(x[k], a.n.mean[c], a.n.stdv[c]));
      }
    }
  } else if (chunk - a.img_chunks < a.lab_chunks) {
    const long long e0 = static_cast<long long>(chunk - a.img_chunks) * DB_BYTES;
    if (rows.labels) {
      rows.label(r, e0, x);
    } else {
#pragma unroll
      for (int k = 0; k < DB_BYTES; ++k) x[k] = 0u;
    }
    long long v[DB_BYTES];
#pragma unroll
    for (int k = 0; k < DB_BYTES; ++k) v[k] = table[x[k]];
    long long* lo = a.label + s * plane + e0;
    if (vec) {
#pragma unroll
      for (int k = 0; k < DB_BYTES; k += 2) *reinterpret_cast<longlong2*>(lo + k) = make_longlong2(v[k], v[k + 1]);
      if (MASK != MASK_IS_POSITIVE) {
        unsigned w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int k = 0; k < DB_BYTES; ++k)
          w[k >> 2] |= static_cast<unsigned>(MASK == MASK_IS_IGNORE ? v[k] == -1 : v[k] >= 0) << (8 * (k & 3));
        *reinterpret_cast<uint4*>(static_cast<unsigned char*>(a.mask) + s * plane + e0) = make_uint4(w[0], w[1], w[2], w[3]);
      } else {
        float m[DB_BYTES];
#pragma unroll
        for (int k = 0; k < DB_BYTES; ++k) m[k] = v[k] > 0 ? 1.0f : 0.0f;
        store16(static_cast<float*>(a.mask) + s * plane + e0, m);
      }
    } else {
#pragma unroll
      for (int k = 0; k < DB_BYTES; ++k) {
        if (e0 + k >= plane) break;
        lo[k] = v[k];
        if (MASK == MASK_IS_IGNORE)
          static_cast<unsigned char*>(a.mask)[s * plane + e0 + k] = v[k] == -1;
        else if (MASK == MASK_IS_NONNEG)
          static_cast<unsigned char*>(a.mask)[s * plane + e0 + k] = v[k] >= 0;
        else
          static_cast<float*>(a.mask)[s * plane + e0 + k] = v[k] > 0 ? 1.0f : 0.0f;
      }
    }
  }
}

// Checks the staging layout on its host copy (records, tables and every image inside the buffer) and fills `a`.
// rec_words FR_REC: res x res outputs; FR_REC_ROWS: each record's own (oh, ow), res unused (the caller checks R_DEST).
static int check_staging(const char* who, const void* host, const void* dev, long long bytes, int B, int res,
                         long long table_words, int channels, FrameArgs& a, int rec_words = FR_REC) {
  STEGO_CHECK_ARG(host && dev, "%s: null staging pointer", who);
  STEGO_CHECK_ARG(B >= 1 && B <= 65535, "%s: B=%d (1..65535)", who, B);
  if (rec_words == FR_REC) STEGO_CHECK_ARG(res >= 1 && res <= 8192, "%s: res=%d (1..8192)", who, res);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(dev) % 8 == 0, "%s: staging must be 8-byte aligned", who);
  const long long head = 8ll * rec_words * B;
  const long long least = rec_words == FR_REC ? 2ll * res : 2;
  STEGO_CHECK_ARG(table_words >= least && table_words <= (1ll << 40), "%s: %lld table words (at least %lld)", who,
                  table_words, least);
  const long long data = head + 4 * table_words;
  STEGO_CHECK_ARG(bytes >= data, "%s: %lld staging bytes hold no %lld-byte record and table block", who, bytes, data);
  const long long* rec = static_cast<const long long*>(host);
  const int* tables = reinterpret_cast<const int*>(static_cast<const char*>(host) + head);
  long long rows = rec_words == FR_REC ? res : 0, width = rec_words == FR_REC ? res : 0;
  for (int b = 0; b < B; ++b) {
    const long long* r = rec + static_cast<size_t>(b) * rec_words;
    const long long off = r[R_OFFSET], H = r[R_H], W = r[R_W], t = r[R_TABLE];
    const long long oh = rec_words == FR_REC ? res : r[R_OH], ow = rec_words == FR_REC ? res : r[R_OW];
    STEGO_CHECK_ARG(oh >= 1 && ow >= 1 && oh <= (1ll << 20) && ow <= (1ll << 20), "%s: output %d is %lld x %lld", who,
                    b, oh, ow);
    rows = oh > rows ? oh : rows;
    width = ow > width ? ow : width;
    STEGO_CHECK_ARG(H >= 1 && W >= 1 && H <= (1ll << 20) && W <= (1ll << 20), "%s: image %d is %lld x %lld (1..2^20)",
                    who, b, H, W);
    STEGO_CHECK_ARG(off >= data && off <= bytes && H * W * channels <= bytes - off,
                    "%s: image %d (%lld bytes at offset %lld) lies outside the %lld-byte staging data [%lld, %lld)",
                    who, b, H * W * channels, off, bytes, data, bytes);
    STEGO_CHECK_ARG(t >= 0 && t <= table_words - (oh + ow), "%s: image %d's tables start at word %lld of %lld", who,
                    b, t, table_words);
    for (long long i = 0; i < oh; ++i) {
      const int sy = tables[t + i];
      STEGO_CHECK_ARG(sy >= -1 && sy < H, "%s: image %d (%lld x %lld): output row %lld reads row %d", who, b, H, W, i,
                      sy);
    }
    for (long long i = 0; i < ow; ++i) {
      const int sx = tables[t + oh + i];
      STEGO_CHECK_ARG(sx >= -1 && sx < W, "%s: image %d (%lld x %lld): output column %lld reads column %d", who, b, H,
                      W, i, sx);
    }
  }
  const long long quads = (width + FR_PIX - 1) / FR_PIX;
  STEGO_CHECK_ARG(rows * quads <= (1ll << 31) - FR_THREADS, "%s: a %lld x %lld output is too large", who, rows, width);
  a.staging = static_cast<const unsigned char*>(dev);
  a.rec = static_cast<const long long*>(dev);
  a.tables = reinterpret_cast<const int*>(static_cast<const unsigned char*>(dev) + head);
  a.res = res;
  a.rec_words = rec_words;
  a.rows = static_cast<int>(rows);
  a.quads = static_cast<int>(quads);
  return STEGO_OK;
}

static dim3 frames_grid(const FrameArgs& a, int B) {
  return dim3(static_cast<unsigned>((static_cast<long long>(a.rows) * a.quads + FR_THREADS - 1) / FR_THREADS), B);
}


// The address a kernel reads or writes `p` through: `p` itself for device memory, the mapped device pointer of pinned
// (page-locked) host memory.  Pageable host memory is refused.
static int device_view(const char* who, const char* what, const void* p, const void** dev, bool* on_host) {
  cudaPointerAttributes attr;
  const cudaError_t e = cudaPointerGetAttributes(&attr, p);
  if (e != cudaSuccess) return cuda_fail(e, who);
  if (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) {
    *dev = p;
    *on_host = false;
    return STEGO_OK;
  }
  STEGO_CHECK_ARG(attr.type == cudaMemoryTypeHost && attr.devicePointer,
                  "%s: %s is neither device memory nor pinned host memory", who, what);
  *dev = attr.devicePointer;
  *on_host = true;
  return STEGO_OK;
}

// Checks a store-build call (rows r0 .. r0 + B of an n-row store, 16-byte aligned) and resolves the store's address.
static int check_store(const char* who, unsigned char* store, long long n, long long r0, int B, unsigned char** dev) {
  STEGO_CHECK_ARG(store, "%s: null store", who);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(store) % 16 == 0, "%s: store must be 16-byte aligned", who);
  STEGO_CHECK_ARG(n >= 1 && r0 >= 0 && r0 <= n - B, "%s: rows %lld .. %lld of a %lld-row store", who, r0, r0 + B, n);
  const void* d = nullptr;
  bool on_host = false;
  const int rc = device_view(who, "store", store, &d, &on_host);
  if (rc != STEGO_OK) return rc;
  *dev = static_cast<unsigned char*>(const_cast<void*>(d));
  return STEGO_OK;
}


// The output checks of the batch entries, and BatchArgs filled from them.
static int check_batch(const char* who, int max_mask_kind, int res, int count, const long long* lut, const Norm& norm,
                       int out_bf16, int mask_kind, void* img, long long* label, void* mask, BatchArgs& a) {
  STEGO_CHECK_ARG(lut && img && label && mask, "%s: null pointer", who);
  STEGO_CHECK_ARG(res >= 1 && res <= 8192, "%s: res=%d (1..8192)", who, res);
  STEGO_CHECK_ARG(count >= 1 && count <= 65535, "%s: count=%d (1..65535)", who, count);
  STEGO_CHECK_ARG(out_bf16 == 0 || out_bf16 == 1, "%s: out_bf16=%d (0 or 1)", who, out_bf16);
  STEGO_CHECK_ARG(mask_kind >= 0 && mask_kind <= max_mask_kind, "%s: mask_kind=%d (0..%d)", who, mask_kind,
                  max_mask_kind);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(lut) % 8 == 0, "%s: lut must be 8-byte aligned", who);
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(img) % 16 == 0 && reinterpret_cast<uintptr_t>(label) % 16 == 0 &&
                      reinterpret_cast<uintptr_t>(mask) % 16 == 0,
                  "%s: outputs must be 16-byte aligned", who);
  a.lut = lut;
  a.n = norm;
  a.img = img;
  a.label = label;
  a.mask = mask;
  a.res = res;
  const long long plane = static_cast<long long>(res) * res;
  a.img_chunks = static_cast<int>((3 * plane + DB_BYTES - 1) / DB_BYTES);
  a.lab_chunks = static_cast<int>((plane + DB_BYTES - 1) / DB_BYTES);
  return STEGO_OK;
}

// The mapped address of a record the host has just checked: it must be pinned host memory.
static int host_record(const char* who, const char* what, const long long* p, const long long** dev) {
  bool on_host = false;
  const void* d = nullptr;
  const int rc = device_view(who, what, p, &d, &on_host);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(on_host, "%s: %s must be pinned host memory (it is checked on the host)", who, what);
  *dev = static_cast<const long long*>(d);
  return STEGO_OK;
}

// The store's address for the kernel (device memory or the mapped address of pinned host memory); null stays null.
static int store_view(const char* who, const char* what, const unsigned char* p, const unsigned char** dev) {
  *dev = nullptr;
  if (!p) return STEGO_OK;
  bool on_host = false;
  const void* d = nullptr;
  const int rc = device_view(who, what, p, &d, &on_host);
  if (rc != STEGO_OK) return rc;
  *dev = static_cast<const unsigned char*>(d);
  return STEGO_OK;
}

template <class Rows>
static int batch_launch(const BatchArgs& a, const Rows& rows, int count, int out_bf16, int mask_kind,
                        cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>((a.img_chunks + a.lab_chunks + DB_THREADS - 1) / DB_THREADS), count);
  if (out_bf16) {
    if (mask_kind == MASK_IS_IGNORE)
      dataset_batch_kernel<bf16, MASK_IS_IGNORE><<<grid, DB_THREADS, 0, stream>>>(a, rows);
    else if (mask_kind == MASK_IS_POSITIVE)
      dataset_batch_kernel<bf16, MASK_IS_POSITIVE><<<grid, DB_THREADS, 0, stream>>>(a, rows);
    else
      dataset_batch_kernel<bf16, MASK_IS_NONNEG><<<grid, DB_THREADS, 0, stream>>>(a, rows);
  } else {
    if (mask_kind == MASK_IS_IGNORE)
      dataset_batch_kernel<float, MASK_IS_IGNORE><<<grid, DB_THREADS, 0, stream>>>(a, rows);
    else if (mask_kind == MASK_IS_POSITIVE)
      dataset_batch_kernel<float, MASK_IS_POSITIVE><<<grid, DB_THREADS, 0, stream>>>(a, rows);
    else
      dataset_batch_kernel<float, MASK_IS_NONNEG><<<grid, DB_THREADS, 0, stream>>>(a, rows);
  }
  STEGO_CHECK_LAUNCH("dataset_batch_kernel launch");
  return STEGO_OK;
}

// The checks and the launch of stego_dataset_batch (mask kinds 0 and 1) and stego_evalset_batch (0, 1 and 2).
static int fixed_batch(const char* who, int max_mask_kind, const unsigned char* images, const unsigned char* labels,
                       long long n, int res, const long long* index, int count, const long long* lut, const Norm& norm,
                       int out_bf16, int mask_kind, void* img, long long* label, void* mask, cudaStream_t stream) {
  STEGO_CHECK_ARG(images && index, "%s: null pointer", who);
  STEGO_CHECK_ARG(n >= 1, "%s: n=%lld rows", who, n);
  BatchArgs a;
  int rc = check_batch(who, max_mask_kind, res, count, lut, norm, out_bf16, mask_kind, img, label, mask, a);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(images) % 16 == 0 && reinterpret_cast<uintptr_t>(labels) % 16 == 0,
                  "%s: the stores must be 16-byte aligned", who);
  FixedRows rows;
  rc = host_record(who, "index", index, &rows.index);
  if (rc != STEGO_OK) return rc;
  for (int i = 0; i < count; ++i)
    STEGO_CHECK_ARG(index[i] >= 0 && index[i] < n, "%s: index[%d]=%lld outside the %lld-row store", who, i, index[i],
                    n);
  rc = store_view(who, "images", images, &rows.images);
  if (rc != STEGO_OK) return rc;
  rc = store_view(who, "labels", labels, &rows.labels);
  if (rc != STEGO_OK) return rc;
  rows.res = res;
  return batch_launch(a, rows, count, out_bf16, mask_kind, stream);
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
  const FrameOut op{{{mean0, mean1, mean2}, {std0, std1, std2}}, out, res};
  frames_rgb8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, op);
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
  labels_u8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, lut, LabelOut{out, res});
  STEGO_CHECK_LAUNCH("labels_u8_kernel launch");
  return STEGO_OK;
}

extern "C" int stego_frames_store_rgb8(const void* staging_host, const void* staging_dev, long long bytes,
                                       long long table_words, int B, int res, unsigned char* store, long long n,
                                       long long r0, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  FrameArgs a;
  int rc = check_staging("stego_frames_store_rgb8", staging_host, staging_dev, bytes, B, res, table_words, 3, a);
  if (rc != STEGO_OK) return rc;
  unsigned char* dev = nullptr;
  rc = check_store("stego_frames_store_rgb8", store, n, r0, B, &dev);
  if (rc != STEGO_OK) return rc;
  frames_rgb8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, StoreOut{dev, r0, 3, res});
  STEGO_CHECK_LAUNCH("frames_rgb8_kernel<StoreOut> launch");
  return STEGO_OK;
}

extern "C" int stego_labels_store_u8(const void* staging_host, const void* staging_dev, long long bytes,
                                     long long table_words, int B, int res, unsigned char* store, long long n,
                                     long long r0, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  FrameArgs a;
  int rc = check_staging("stego_labels_store_u8", staging_host, staging_dev, bytes, B, res, table_words, 1, a);
  if (rc != STEGO_OK) return rc;
  unsigned char* dev = nullptr;
  rc = check_store("stego_labels_store_u8", store, n, r0, B, &dev);
  if (rc != STEGO_OK) return rc;
  labels_u8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, nullptr, StoreOut{dev, r0, 1, res});
  STEGO_CHECK_LAUNCH("labels_u8_kernel<StoreOut> launch");
  return STEGO_OK;
}

extern "C" int stego_dataset_batch(const unsigned char* images, const unsigned char* labels, long long n, int res,
                                   const long long* index, int count, const long long* lut, float mean0, float mean1,
                                   float mean2, float std0, float std1, float std2, int out_bf16, int mask_kind,
                                   void* img, long long* label, void* mask, void* stream) {
  return fixed_batch("stego_dataset_batch", MASK_IS_POSITIVE, images, labels, n, res, index, count, lut,
                      Norm{{mean0, mean1, mean2}, {std0, std1, std2}}, out_bf16, mask_kind, img, label, mask,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int stego_evalset_batch(const unsigned char* images, const unsigned char* labels, long long n, int res,
                                   const long long* index, int count, const long long* lut, float mean0, float mean1,
                                   float mean2, float std0, float std1, float std2, int out_bf16, int mask_kind,
                                   void* img, long long* label, void* mask, void* stream) {
  return fixed_batch("stego_evalset_batch", MASK_IS_NONNEG, images, labels, n, res, index, count, lut,
                      Norm{{mean0, mean1, mean2}, {std0, std1, std2}}, out_bf16, mask_kind, img, label, mask,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int stego_store_rows_u8(const void* staging_host, const void* staging_dev, long long bytes,
                                   long long table_words, int B, int channels, unsigned char* store,
                                   long long store_bytes, void* stream_) {
  const char* who = "stego_store_rows_u8";
  STEGO_CHECK_ARG(channels == 1 || channels == 3, "%s: channels=%d (1 or 3)", who, channels);
  FrameArgs a;
  int rc = check_staging(who, staging_host, staging_dev, bytes, B, 0, table_words, channels, a, FR_REC_ROWS);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(store && store_bytes >= 1, "%s: null or empty store", who);
  const long long* rec = static_cast<const long long*>(staging_host);
  for (int b = 0; b < B; ++b) {
    const long long* r = rec + static_cast<size_t>(b) * FR_REC_ROWS;
    const long long row = channels * r[R_OH] * r[R_OW];
    STEGO_CHECK_ARG(r[R_DEST] >= 0 && r[R_DEST] <= store_bytes - row,
                    "%s: image %d's %lld-byte row at offset %lld lies outside the %lld-byte store", who, b, row,
                    r[R_DEST], store_bytes);
  }
  const unsigned char* dev = nullptr;
  rc = store_view(who, "store", store, &dev);
  if (rc != STEGO_OK) return rc;
  const RowOut op{const_cast<unsigned char*>(dev)};
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (channels == 3)
    frames_rgb8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, op);
  else
    labels_u8_kernel<<<frames_grid(a, B), FR_THREADS, 0, stream>>>(a, nullptr, op);
  STEGO_CHECK_LAUNCH("stego_store_rows_u8 launch");
  return STEGO_OK;
}

extern "C" int stego_store_batch_window(const unsigned char* images, long long image_bytes,
                                        const unsigned char* labels, long long label_bytes, const long long* rows,
                                        long long n, int res, const long long* record, int count,
                                        const long long* lut, float mean0, float mean1, float mean2, float std0,
                                        float std1, float std2, int out_bf16, int mask_kind, void* img,
                                        long long* label, void* mask, void* stream) {
  const char* who = "stego_store_batch_window";
  STEGO_CHECK_ARG(images && rows && record, "%s: null pointer", who);
  STEGO_CHECK_ARG(n >= 1, "%s: n=%lld rows", who, n);
  BatchArgs a;
  int rc = check_batch(who, MASK_IS_NONNEG, res, count, lut, Norm{{mean0, mean1, mean2}, {std0, std1, std2}},
                       out_bf16, mask_kind, img, label, mask, a);
  if (rc != STEGO_OK) return rc;
  STEGO_CHECK_ARG(reinterpret_cast<uintptr_t>(images) % 16 == 0 && reinterpret_cast<uintptr_t>(labels) % 16 == 0 &&
                      image_bytes % 16 == 0 && (!labels || label_bytes % 16 == 0),
                  "%s: the stores must be 16-byte aligned and a multiple of 16 bytes long", who);
  WindowRows w;
  const long long* rows_dev = nullptr;
  rc = host_record(who, "rows", rows, &rows_dev);
  if (rc != STEGO_OK) return rc;
  rc = host_record(who, "record", record, &w.rec);
  if (rc != STEGO_OK) return rc;
  for (int s = 0; s < count; ++s) {
    const long long* q = record + static_cast<size_t>(s) * WIN_REC;
    const long long i = q[W_ROW];
    STEGO_CHECK_ARG(i >= 0 && i < n, "%s: record %d reads row %lld of a %lld-row store", who, s, i, n);
    const long long* t = rows + i * ROW_WORDS;
    const long long oh = t[RT_OH], ow = t[RT_OW];
    STEGO_CHECK_ARG(oh >= res && ow >= res && oh <= (1ll << 20) && ow <= (1ll << 20) && t[RT_IMG] >= 0 &&
                        t[RT_IMG] <= image_bytes - 3 * oh * ow,
                    "%s: row %lld (a %lld x %lld image at byte %lld) does not fit res %d in the %lld-byte store", who,
                    i, oh, ow, t[RT_IMG], res, image_bytes);
    STEGO_CHECK_ARG(q[W_TOP] >= 0 && q[W_TOP] <= oh - res && q[W_LEFT] >= 0 && q[W_LEFT] <= ow - res,
                    "%s: record %d's window (%lld, %lld) leaves row %lld's %lld x %lld image", who, s, q[W_TOP],
                    q[W_LEFT], i, oh, ow);
    if (labels) {
      const long long lh = t[RT_LH], lw = t[RT_LW];
      STEGO_CHECK_ARG(lh >= res && lw >= res && lh <= (1ll << 20) && lw <= (1ll << 20) && t[RT_LAB] >= 0 &&
                          t[RT_LAB] <= label_bytes - lh * lw,
                      "%s: row %lld (a %lld x %lld label at byte %lld) does not fit res %d in the %lld-byte store",
                      who, i, lh, lw, t[RT_LAB], res, label_bytes);
      STEGO_CHECK_ARG(q[W_LTOP] >= 0 && q[W_LTOP] <= lh - res && q[W_LLEFT] >= 0 && q[W_LLEFT] <= lw - res,
                      "%s: record %d's label window (%lld, %lld) leaves row %lld's %lld x %lld label", who, s,
                      q[W_LTOP], q[W_LLEFT], i, lh, lw);
    }
  }
  w.rows = rows_dev;
  rc = store_view(who, "images", images, &w.images);
  if (rc != STEGO_OK) return rc;
  rc = store_view(who, "labels", labels, &w.labels);
  if (rc != STEGO_OK) return rc;
  w.res = res;
  return batch_launch(a, w, count, out_bf16, mask_kind, reinterpret_cast<cudaStream_t>(stream));
}
