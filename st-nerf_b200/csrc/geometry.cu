// Ray generation, ray/box clipping and stratified sampling kernels (HBM-bound, fp32, bit-parity arithmetic).
//
// Compiled with -fmad=false: the reference evaluates these expressions as separate ATen mul / add ops
// (layers/RaySamplePoint.py:17-32,98-105), and several results feed discontinuous tests (inclusive face
// tests, |bin_width| > 1e-5, t < 0), so products and sums must round separately exactly as eager PyTorch does.
#include "common.cuh"
#include "raygen.cuh"

namespace stnerf {

// ---------------------------------------------------------------------------------------------------------
// a3: layers/RaySamplePoint.py:8-62 -- six slab candidates, inclusive in-face tests, top-2.
// tlist is -1e3 * ones_like(rays) (:53): one slot per ray COLUMN, six face slots and a -1e3 sentinel per column beyond
// the sixth, and the top-2 (:60) runs over all of them.  `sentinels` = min(2, columns - 6) is how many of those take
// part: a 6-column ray has none, so when five or six faces are valid and all lie below -1e3 its top-2 is (-1e3, face) or
// two faces, where a ray with more columns gets (-1e3, -1e3).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ray_box_sentinels(int columns) { return min(2, columns - 6); }

__device__ __forceinline__ void ray_box(const float o[3], const float d[3], const float bmin[3], const float bmax[3],
                                        int sentinels, float& t_far, float& t_near) {
  const float eps = 2.220446049250313e-16f;   // np.finfo(float).eps cast to fp32 (:17-22)
  // an invalid face is a -1e3 candidate, so the six faces always fill both slots; -inf only marks a missing sentinel
  float m1 = sentinels > 0 ? -1000.0f : -INFINITY, m2 = sentinels > 1 ? -1000.0f : -INFINITY;
#pragma unroll
  for (int axis = 0; axis < 3; ++axis) {
    const int a1 = (axis + 1) % 3, a2 = (axis + 2) % 3;
    const float den = d[axis] + eps;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const float face = side ? bmax[axis] : bmin[axis];
      const float t = (face - o[axis]) / den;
      const float p1 = t * d[a1] + o[a1];
      const float p2 = t * d[a2] + o[a2];
      const bool ok = (p1 >= bmin[a1]) && (p1 <= bmax[a1]) && (p2 >= bmin[a2]) && (p2 <= bmax[a2]);
      const float v = ok ? t : -1000.0f;
      if (v > m1) { m2 = m1; m1 = v; } else if (v > m2) { m2 = v; }
    }
  }
  t_far = m1;
  t_near = m2;
}

// a4: start / width of the stratified bins of one (ray, box) (layers/RaySamplePoint.py:91-105)
__device__ __forceinline__ void ray_bins(const float o[3], const float d[3], const float bmin[3], const float bmax[3],
                                         int sentinels, bool is_bkgd, int n1, float& start, float& width, bool& hit) {
  float t_far, t_near;
  ray_box(o, d, bmin, bmax, sentinels, t_far, t_near);
  start = t_near;
  if (is_bkgd && start <= 0.0f) start = 0.0f;     // :93-95
  width = (t_far - start) / (float)n1;             // :100
  hit = fabsf(width) > 1e-5f;                      // :105
}

// ---------------------------------------------------------------------------------------------------------
// K2: coarse sampling of a chunk of rays against all layers.
//   block = 256 rays.  phase 1: thread-per-ray clipping, masks, ordered hit-list compaction (one atomic per
//   block per layer);  phase 2: the block writes t[layer][ray][k] fully coalesced.
// ---------------------------------------------------------------------------------------------------------
constexpr int SAMPLE_BLOCK = 256;

__global__ void __launch_bounds__(SAMPLE_BLOCK)
sample_kernel(const float* __restrict__ rays, long long n, int ray_stride, const DevScene scene,
              int n_layers, int n1, const float* __restrict__ jitter, long long jitter_layer_stride, uint64_t seed,
              long long ray_base, RayIdMap idmap, float* __restrict__ t_out, long long t_layer_stride, uint8_t* __restrict__ mask,
              long long mask_layer_stride, int* __restrict__ hit, long long hit_layer_stride, int* __restrict__ counts,
              int* __restrict__ lerp_flags, const float* __restrict__ box_table, int n_frames, const __grid_constant__ LayerRays lrays) {
  __shared__ float s_start[STNERF_MAX_LAYERS][SAMPLE_BLOCK];
  __shared__ float s_width[STNERF_MAX_LAYERS][SAMPLE_BLOCK];
  __shared__ int s_warp_hits[STNERF_MAX_LAYERS][SAMPLE_BLOCK / 32];
  __shared__ int s_base[STNERF_MAX_LAYERS];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long ray0 = (long long)blockIdx.x * SAMPLE_BLOCK;
  const long long r = ray0 + tid;
  const bool live = r < n;

  float o[3] = {0, 0, 0}, d[3] = {0, 0, 1};
  if (live) {
    const float* p = rays + r * ray_stride;
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
    d[0] = p[3]; d[1] = p[4]; d[2] = p[5];
  }
  unsigned my_hits = 0;
  // the rays' columns follow from the scene: [o, d, frame_id] with a shared frame id, else one frame id per layer
  const int sentinels = ray_box_sentinels(scene.fid_shared ? 7 : 6 + n_layers);
  // rays of a mixed-frame batch: the boxes of the ray's own frame, index_select(frame_id - 1) (layered_rfrender.py:193)
  const float* my_boxes = nullptr;
  if (box_table != nullptr && live) {
    int f = (int)rays[r * ray_stride + 6] - 1;                    // .type(torch.int64): truncation
    f = min(max(f, 0), n_frames - 1);
    my_boxes = box_table + (size_t)f * n_layers * 6;
  }
  for (int i = 0; i < n_layers; ++i) {
    float bmin[3] = {scene.bmin[i][0], scene.bmin[i][1], scene.bmin[i][2]};
    float bmax[3] = {scene.bmax[i][0], scene.bmax[i][1], scene.bmax[i][2]};
    if (my_boxes != nullptr) {
#pragma unroll
      for (int a = 0; a < 3; ++a) { bmin[a] = my_boxes[i * 6 + a]; bmax[a] = my_boxes[i * 6 + 3 + a]; }
    }
    float start, width;
    bool h;
    if (lrays.p[i] != rays) {         // a rotated layer: its own ray against the unrotated box == the oriented-box clip
      float oi[3] = {0, 0, 0}, di[3] = {0, 0, 1};
      if (live) {
        const float* q = lrays.p[i] + r * ray_stride;
        oi[0] = q[0]; oi[1] = q[1]; oi[2] = q[2];
        di[0] = q[3]; di[1] = q[4]; di[2] = q[5];
      }
      ray_bins(oi, di, bmin, bmax, sentinels, i == 0, n1, start, width, h);
    } else {
      ray_bins(o, d, bmin, bmax, sentinels, i == 0, n1, start, width, h);
    }
    h = h && live;
    s_start[i][tid] = start;
    s_width[i][tid] = width;
    if (live) mask[i * mask_layer_stride + r] = h ? 1 : 0;
    const unsigned b = __ballot_sync(0xffffffffu, h);
    if (lane == 0) s_warp_hits[i][warp] = __popc(b);
    if (h) my_hits |= 1u << i;
    // rank of this ray among the warp's hits
    // (stored for phase 1b in a register: popc of lower lanes)
    if (h && i > 0) {
      // MotionNet's batch-global "any fractional frame id" test (modeling/motion_net.py:53)
      const float f = rays[r * ray_stride + 6 + (scene.fid_shared ? 0 : i)];
      if (floorf(f) != f) atomicOr(&lerp_flags[i], 1);
    }
  }
  __syncthreads();
  if (tid < n_layers && tid > 0) {
    int tot = 0;
    for (int w = 0; w < SAMPLE_BLOCK / 32; ++w) tot += s_warp_hits[tid][w];
    s_base[tid] = tot ? atomicAdd(&counts[tid], tot) : 0;
  }
  __syncthreads();
  for (int i = 1; i < n_layers; ++i) {
    const bool h = (my_hits >> i) & 1u;
    const unsigned b = __ballot_sync(0xffffffffu, h);
    if (h) {
      int pos = s_base[i] + __popc(b & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) pos += s_warp_hits[i][w];
      hit[i * hit_layer_stride + pos] = (int)r;
    }
  }
  // phase 2: t = (k + U) * width + start, rounded op by op (layers/RaySamplePoint.py:102)
  const int rays_here = (int)min((long long)SAMPLE_BLOCK, n - ray0);
  const int total = rays_here * n1;
  for (int i = 0; i < n_layers; ++i) {
    float* tl = t_out + i * t_layer_stride + ray0 * n1;
    const float* jl = jitter ? jitter + i * jitter_layer_stride + ray0 * n1 : nullptr;
    for (int idx = tid; idx < total; idx += SAMPLE_BLOCK) {
      const int rr = idx / n1, k = idx - rr * n1;
      const float uu = jl ? jl[idx] : philox_uniform(seed, (uint32_t)i, idmap(ray_base + ray0 + rr), (uint32_t)k);
      const float a = (float)k + uu;
      tl[idx] = a * s_width[i][rr] + s_start[i][rr];
    }
  }
}

int launch_sample(const float* rays, long long n, int ray_stride, const DevScene& scene, int n_layers, int n1,
                  const float* jitter, long long jitter_layer_stride, uint64_t seed, long long ray_base, RayIdMap idmap,
                  float* t_coarse, long long t_layer_stride, uint8_t* mask, long long mask_layer_stride, int* hit,
                  long long hit_layer_stride, int* counts, int* lerp_flags, cudaStream_t st, const float* box_table,
                  int n_frames, const LayerRays* layer_rays) {
  if (n <= 0) return STNERF_OK;
  const int grid = (int)((n + SAMPLE_BLOCK - 1) / SAMPLE_BLOCK);
  LayerRays lr;
  for (int i = 0; i < STNERF_MAX_LAYERS; ++i) lr.p[i] = layer_rays ? layer_rays->p[i] : rays;
  sample_kernel<<<grid, SAMPLE_BLOCK, 0, st>>>(rays, n, ray_stride, scene, n_layers, n1, jitter,
                                               jitter_layer_stride, seed, ray_base, idmap, t_coarse, t_layer_stride, mask,
                                               mask_layer_stride, hit, hit_layer_stride, counts, lerp_flags,
                                               (scene.fid_shared && n_frames > 0) ? box_table : nullptr, n_frames, lr);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// The rays of a rotated layer (include/stnerf.h: stnerf_set_rotation): o' = c + R^T (o - c), d' = R^T d, frame ids copied.
// One thread per ray; a full-stride copy, so every consumer indexes it exactly like the caller's rays.
// ---------------------------------------------------------------------------------------------------------
__global__ void rotate_rays_kernel(const float* __restrict__ rays, long long n, int ray_stride, const RayRot rot,
                                   float* __restrict__ out) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* p = rays + r * ray_stride;
  float* q = out + r * ray_stride;
  const float o[3] = {p[0], p[1], p[2]}, d[3] = {p[3], p[4], p[5]};
  float o2[3], d2[3];
  rotate_back_point(rot, o, o2);
  rotate_back_dir(rot, d, d2);
#pragma unroll
  for (int a = 0; a < 3; ++a) { q[a] = o2[a]; q[3 + a] = d2[a]; }
  for (int k = 6; k < ray_stride; ++k) q[k] = p[k];
}

int launch_rotate_rays(const float* rays, long long n, int ray_stride, const RayRot& r, float* out, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  const int block = 256;
  rotate_rays_kernel<<<(unsigned)((n + block - 1) / block), block, 0, st>>>(rays, n, ray_stride, r, out);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Unit entry point: one box, explicit outputs (intersection() + RaySamplePoint.forward for one layer).
// ---------------------------------------------------------------------------------------------------------
struct Box6 { float lo[3], hi[3]; };

__global__ void intersect_sample_kernel(const float* __restrict__ rays, long long n, int ray_stride, Box6 box,
                                        int is_bkgd, int n1, const float* __restrict__ jitter, float* __restrict__ t,
                                        float* __restrict__ xyz, uint8_t* __restrict__ mask,
                                        float* __restrict__ tfar_tnear) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* p = rays + r * ray_stride;
  const float o[3] = {p[0], p[1], p[2]}, d[3] = {p[3], p[4], p[5]};
  const int sentinels = ray_box_sentinels(ray_stride);     // the rays are ray_stride columns wide
  if (tfar_tnear) {
    float tf, tn;
    ray_box(o, d, box.lo, box.hi, sentinels, tf, tn);
    tfar_tnear[2 * r] = tf;
    tfar_tnear[2 * r + 1] = tn;
  }
  float start, width;
  bool h;
  ray_bins(o, d, box.lo, box.hi, sentinels, is_bkgd != 0, n1, start, width, h);
  if (mask) mask[r] = h ? 1 : 0;
  for (int k = 0; k < n1; ++k) {
    const float a = (float)k + jitter[r * n1 + k];
    const float tt = a * width + start;
    if (t) t[r * n1 + k] = tt;
    if (xyz) {
      float* q = xyz + (r * n1 + k) * 3;
      q[0] = tt * d[0] + o[0];                 // :103
      q[1] = tt * d[1] + o[1];
      q[2] = tt * d[2] + o[2];
    }
  }
}

int launch_intersect_sample(const float* rays, long long n, int ray_stride, const float* bmin, const float* bmax,
                            int is_bkgd, int n1, const float* jitter, float* t, float* xyz, uint8_t* mask,
                            float* tfar_tnear, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  Box6 b;
  for (int a = 0; a < 3; ++a) { b.lo[a] = bmin[a]; b.hi[a] = bmax[a]; }
  const int block = 128, grid = (int)((n + block - 1) / block);
  intersect_sample_kernel<<<grid, block, 0, st>>>(rays, n, ray_stride, b, is_bkgd, n1, jitter, t, xyz, mask,
                                                  tfar_tnear);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// K1: ray generation (utils/render_helpers.py:96-123).  One thread per pixel; rays written with 6+F columns.
// ---------------------------------------------------------------------------------------------------------
struct RayGenParams {
  float kinv[9];
  float rot[9];
  float org[3];
  float fid[STNERF_MAX_LAYERS];
  int n_fid;
};

__global__ void raygen_kernel(RayGenParams P, int W, int row0, int row_step, int n_rows, float* __restrict__ rays,
                              int ray_stride) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)n_rows * W;
  if (idx >= total) return;
  const int rr = (int)(idx / W), j = (int)(idx - (long long)rr * W);
  const float px = (float)j, py = (float)(row0 + rr * row_step);
  float c[3];
  raygen_dir(P.kinv, px, py, c);        // dirs = K^-1 (col, row, 1)
  float* out = rays + idx * ray_stride;
  raygen_write(P.rot, P.org, c, out);
  for (int f = 0; f < P.n_fid; ++f) out[6 + f] = P.fid[f];
}

int launch_raygen(const float* Kinv, const float* T, int H, int W, int row0, int row_step, int n_rows,
                  const float* fids, int n_fids, float* rays, int ray_stride, cudaStream_t st) {
  if (n_rows <= 0 || W <= 0) return STNERF_OK;
  // rows past H-1 are extrapolated pixel rows (one padding row for equal shard sizes, see stnerf_render_views)
  if (n_fids > STNERF_MAX_LAYERS || ray_stride < 6 + n_fids || row0 >= H || row0 + (long long)(n_rows - 1) * row_step >= H + row_step)
    return STNERF_EINVAL;
  RayGenParams P;
  for (int i = 0; i < 9; ++i) P.kinv[i] = Kinv[i];
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) P.rot[3 * a + b] = T[4 * a + b];
    P.org[a] = T[4 * a + 3];
  }
  P.n_fid = n_fids;
  for (int f = 0; f < n_fids; ++f) P.fid[f] = fids[f];
  const long long total = (long long)n_rows * W;
  const int block = 256;
  raygen_kernel<<<(int)((total + block - 1) / block), block, 0, st>>>(P, W, row0, row_step, n_rows, rays, ray_stride);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// a6 unit entry point: utils/dimension_kernel.py:24-33
// ---------------------------------------------------------------------------------------------------------
__global__ void posenc_kernel(const float* __restrict__ x, long long P, int dim, int n_freq, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * dim) return;
  const long long p = idx / dim;
  const int c = (int)(idx - p * dim);
  const int width = dim * (1 + 2 * n_freq);
  const float v = x[idx];
  float* o = out + p * width;
  o[c] = v;
  float f = 1.0f;
  for (int k = 0; k < n_freq; ++k) {
    float s, cs;
    sincosf(v * f, &s, &cs);
    o[dim + 2 * k * dim + c] = s;
    o[dim + (2 * k + 1) * dim + c] = cs;
    f *= 2.0f;
  }
}

int launch_posenc(const float* x, long long P, int dim, int n_freq, float* out, cudaStream_t st) {
  if (P <= 0) return STNERF_OK;
  const long long total = P * dim;
  posenc_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(x, P, dim, n_freq, out);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // namespace stnerf
