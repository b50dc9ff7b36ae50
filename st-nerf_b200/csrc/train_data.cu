// Training ray pool: per-image pixel selection with ordered compaction, and the batch kernel that turns pool indices into
// the trainer's (rays, rgbs, labels, bbox_labels, bboxes, near_far) (data/datasets/ray_dataset.py:339-460).
//
// Compiled with -fmad=false: a training ray is built by raygen.cuh's functions, which round like the reference's eager
// fp32 ops and like raygen_kernel, so a pool ray is bit-identical to the render ray of the same camera and pixel.
//
// A pool entry is 16 bytes and holds no ray (uint4):
//   x = pixel (row * W + col), y = camera | frame slot << 16, z = r | g << 8 | b << 16 | label << 24, w = layer.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "raygen.cuh"

namespace stnerf {

namespace {

constexpr int SEL_THREADS = 256;
constexpr int SEL_PER_THREAD = 8;
constexpr int SEL_TILE = SEL_THREADS * SEL_PER_THREAD;   // pixels of one tile; thread t owns pixels [8t, 8t+8) of it
constexpr int SCAN_THREADS = 1024;
constexpr int CAM_FLOATS = 24;                           // kinv 9 | rot 9 | org 3 | W | pad 2
constexpr int BOX_FLOATS = 24;

// Which pixels a (image, layer) keeps: label == layer (ray_sampling.py:194-240), or the box's projected rectangle
// rows [r0, r1) x cols [c0, c1) (:75-175).  A label map that is absent is the constant `const_label` (frame_dataset.py:283).
struct SelectArgs {
  const void* label;     // uint8 [H*W] or fp32 [H*W]; nullptr = constant map
  int label_is_float;
  int const_label;
  int H, W;
  int mode;              // STNERF_TD_BY_LABEL / STNERF_TD_BY_RECT
  int layer;
  int r0, r1, c0, c1;
};

__device__ __forceinline__ bool keep_pixel(const SelectArgs& a, long long p) {
  if (a.mode == STNERF_TD_BY_RECT) {
    const int r = (int)(p / a.W), c = (int)(p - (long long)r * a.W);
    return r >= a.r0 && r < a.r1 && c >= a.c0 && c < a.c1;
  }
  if (!a.label) return a.const_label == a.layer;
  if (a.label_is_float) return static_cast<const float*>(a.label)[p] == (float)a.layer;
  return static_cast<const uint8_t*>(a.label)[p] == (uint8_t)a.layer;
}

__device__ __forceinline__ int label_byte(const SelectArgs& a, long long p) {
  if (!a.label) return a.const_label & 255;
  if (a.label_is_float) return 0;                    // the float form writes pixel indices only
  return static_cast<const uint8_t*>(a.label)[p];
}

__global__ void __launch_bounds__(SEL_THREADS) select_count_kernel(SelectArgs a, int* __restrict__ tile_counts) {
  using Reduce = cub::BlockReduce<int, SEL_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long n = (long long)a.H * a.W;
  const long long base = (long long)blockIdx.x * SEL_TILE + (long long)threadIdx.x * SEL_PER_THREAD;
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < SEL_PER_THREAD; ++k)
    if (base + k < n && keep_pixel(a, base + k)) ++cnt;
  const int total = Reduce(tmp).Sum(cnt);
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = total;
}

// One block: exclusive scan of the tile counts in tile order; offsets[n_tiles] = the image's total.
__global__ void __launch_bounds__(SCAN_THREADS) select_scan_kernel(const int* __restrict__ tile_counts, int n_tiles,
                                                                   int* __restrict__ offsets) {
  using Scan = cub::BlockScan<int, SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int t0 = 0; t0 < n_tiles; t0 += SCAN_THREADS) {
    const int t = t0 + (int)threadIdx.x;
    const int v = t < n_tiles ? tile_counts[t] : 0;
    int ex, sum;
    Scan(tmp).ExclusiveSum(v, ex, sum);
    if (t < n_tiles) offsets[t] = carry + ex;
    carry += sum;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[n_tiles] = carry;
}

__global__ void __launch_bounds__(SEL_THREADS) select_write_kernel(SelectArgs a, const int* __restrict__ offsets,
                                                                   const uint8_t* __restrict__ rgb, uint32_t cam_frame,
                                                                   uint4* __restrict__ pool, int* __restrict__ pix) {
  using Scan = cub::BlockScan<int, SEL_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const long long n = (long long)a.H * a.W;
  const long long base = (long long)blockIdx.x * SEL_TILE + (long long)threadIdx.x * SEL_PER_THREAD;
  unsigned flags = 0;
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < SEL_PER_THREAD; ++k)
    if (base + k < n && keep_pixel(a, base + k)) { flags |= 1u << k; ++cnt; }
  int ex;
  Scan(tmp).ExclusiveSum(cnt, ex);
  long long o = (long long)offsets[blockIdx.x] + ex;
#pragma unroll
  for (int k = 0; k < SEL_PER_THREAD; ++k) {
    if (!(flags & (1u << k))) continue;
    const long long p = base + k;
    if (pool) {
      const uint8_t* c = rgb + 3 * p;
      const uint32_t z = (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | ((uint32_t)label_byte(a, p) << 24);
      pool[o] = make_uint4((uint32_t)p, cam_frame, z, (uint32_t)a.layer);
    }
    if (pix) pix[o] = (int)p;
    ++o;
  }
}

struct BatchTables {
  const float* cams;        // [n_geom][n_cams][CAM_FLOATS]
  const float* boxes;       // [n_layers][n_frames][BOX_FLOATS]
  const float* near_far;    // [n_layers][n_frames][n_cams][2]
  uint32_t geom_of_layer;    // 4 bits per layer (a register, not an indexed parameter array)
  int n_cams, n_frames;
  float frame_base;         // frame id of frame slot 0
  int time_col;
};

template <class Idx>
__global__ void __launch_bounds__(256) batch_kernel(const uint4* __restrict__ pool, const Idx* __restrict__ idx, long long B,
                                                    BatchTables t, float* __restrict__ rays, float* __restrict__ rgbs,
                                                    float* __restrict__ labels, float* __restrict__ bbox_labels,
                                                    float* __restrict__ bboxes, float* __restrict__ near_far) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const uint4 e = pool[(long long)idx[b]];
  const int cam = (int)(e.y & 0xffffu), frame = (int)(e.y >> 16), layer = (int)e.w;
  const float* cp = t.cams + ((long long)((t.geom_of_layer >> (4 * layer)) & 15u) * t.n_cams + cam) * CAM_FLOATS;
  const int W = (int)cp[21];
  const int row = (int)(e.x / (uint32_t)W), col = (int)(e.x - (uint32_t)row * (uint32_t)W);
  float c[3];
  raygen_dir(cp, (float)col, (float)row, c);
  const int stride = 6 + t.time_col;
  float* out = rays + b * stride;
  raygen_write(cp + 9, cp + 18, c, out);
  if (t.time_col) out[6] = t.frame_base + (float)frame;
  rgbs[3 * b + 0] = (float)(e.z & 255u) / 255.0f;
  rgbs[3 * b + 1] = (float)((e.z >> 8) & 255u) / 255.0f;
  rgbs[3 * b + 2] = (float)((e.z >> 16) & 255u) / 255.0f;
  labels[b] = (float)(e.z >> 24);
  bbox_labels[b] = (float)layer;
  const float* bx = t.boxes + ((long long)layer * t.n_frames + frame) * BOX_FLOATS;
#pragma unroll
  for (int k = 0; k < 24; ++k) bboxes[24 * b + k] = bx[k];
  const float* nf = t.near_far + (((long long)layer * t.n_frames + frame) * t.n_cams + cam) * 2;
  near_far[2 * b] = nf[0];
  near_far[2 * b + 1] = nf[1];
}

int select_args(const void* label, int label_is_float, int const_label, int H, int W, int mode, int layer,
                const int* rect_host, SelectArgs& a) {
  if (H <= 0 || W <= 0 || (long long)H * W >= (1LL << 31) || layer < 0 || layer >= STNERF_MAX_LAYERS) return STNERF_EINVAL;
  if (mode != STNERF_TD_BY_LABEL && mode != STNERF_TD_BY_RECT) return STNERF_EINVAL;
  if (mode == STNERF_TD_BY_RECT && !rect_host) return STNERF_EINVAL;
  a.label = label; a.label_is_float = label_is_float; a.const_label = const_label;
  a.H = H; a.W = W; a.mode = mode; a.layer = layer;
  a.r0 = a.r1 = a.c0 = a.c1 = 0;
  if (mode == STNERF_TD_BY_RECT) { a.r0 = rect_host[0]; a.r1 = rect_host[1]; a.c0 = rect_host[2]; a.c1 = rect_host[3]; }
  return STNERF_OK;
}

int n_tiles(int H, int W) { return (int)(((long long)H * W + SEL_TILE - 1) / SEL_TILE); }

}  // namespace
}  // namespace stnerf

using namespace stnerf;

extern "C" {

int64_t stnerf_td_select_scratch_ints(int H, int W) {
  if (H <= 0 || W <= 0) return 0;
  return 2 * (int64_t)n_tiles(H, W) + 1;
}

int stnerf_td_select_count(const void* label, int label_is_float, int const_label, int H, int W, int mode, int layer,
                           const int* rect_host, int* scratch, void* stream) {
  SelectArgs a;
  int rc = select_args(label, label_is_float, const_label, H, W, mode, layer, rect_host, a);
  if (rc != STNERF_OK || !scratch) return rc != STNERF_OK ? rc : STNERF_EINVAL;
  const int nt = n_tiles(H, W);
  cudaStream_t st = (cudaStream_t)stream;
  select_count_kernel<<<nt, SEL_THREADS, 0, st>>>(a, scratch);
  STNERF_LAUNCH_CHECK();
  select_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(scratch, nt, scratch + nt);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

int stnerf_td_select_write(const void* label, int label_is_float, int const_label, const uint8_t* rgb, int H, int W,
                           int mode, int layer, const int* rect_host, int camera, int frame_slot, const int* scratch,
                           void* pool, int* pixels, void* stream) {
  SelectArgs a;
  int rc = select_args(label, label_is_float, const_label, H, W, mode, layer, rect_host, a);
  if (rc != STNERF_OK) return rc;
  if (!scratch || (!pool && !pixels) || (pool && (!rgb || label_is_float)) || camera < 0 || camera > 0xffff ||
      frame_slot < 0 || frame_slot > 0xffff)
    return STNERF_EINVAL;
  const int nt = n_tiles(H, W);
  select_write_kernel<<<nt, SEL_THREADS, 0, (cudaStream_t)stream>>>(a, scratch + nt, rgb,
                                                                    (uint32_t)camera | ((uint32_t)frame_slot << 16),
                                                                    static_cast<uint4*>(pool), pixels);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

int stnerf_td_batch(const void* pool, const void* idx, int idx_is_64, int64_t B, const float* cams,
                    const int* geom_of_layer_host, int n_layers, int n_cams, const float* boxes, const float* near_far,
                    int n_frames, float frame_base, int time_col, float* rays, float* rgbs, float* labels,
                    float* bbox_labels, float* bboxes, float* near_far_out, void* stream) {
  if (B < 0 || n_layers < 1 || n_layers > STNERF_MAX_LAYERS || n_cams < 1 || n_frames < 1 || !geom_of_layer_host ||
      (time_col != 0 && time_col != 1))
    return STNERF_EINVAL;
  if (B == 0) return STNERF_OK;
  if (!pool || !idx || !cams || !boxes || !near_far || !rays || !rgbs || !labels || !bbox_labels || !bboxes || !near_far_out)
    return STNERF_EINVAL;
  BatchTables t;
  t.cams = cams; t.boxes = boxes; t.near_far = near_far;
  t.geom_of_layer = 0;
  for (int l = 0; l < n_layers; ++l) {
    if (geom_of_layer_host[l] < 0 || geom_of_layer_host[l] > 15) return STNERF_EINVAL;
    t.geom_of_layer |= (uint32_t)geom_of_layer_host[l] << (4 * l);
  }
  t.n_cams = n_cams; t.n_frames = n_frames; t.frame_base = frame_base; t.time_col = time_col;
  const int block = 256;
  const unsigned grid = (unsigned)((B + block - 1) / block);
  cudaStream_t st = (cudaStream_t)stream;
  if (idx_is_64)
    batch_kernel<long long><<<grid, block, 0, st>>>(static_cast<const uint4*>(pool), static_cast<const long long*>(idx), B, t,
                                                    rays, rgbs, labels, bbox_labels, bboxes, near_far_out);
  else
    batch_kernel<int><<<grid, block, 0, st>>>(static_cast<const uint4*>(pool), static_cast<const int*>(idx), B, t, rays, rgbs,
                                              labels, bbox_labels, bboxes, near_far_out);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // extern "C"
