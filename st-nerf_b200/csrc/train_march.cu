// Per-sample work of a training step outside the networks (stnerf_b200.train): ordered hit lists, the compact network
// inputs of one layer and pass, the masked scatter of the network outputs into the per-layer sample grid and its backward,
// and the Philox uniforms of the fine resampling.
//
// Compiled with -fmad=false like geometry.cu / composite.cu: the marched points must round op by op like eager PyTorch
// (they are march_point, shared with the networks' SRC_MARCH fetch), and the density masks and the alpha factor must give
// the very values composite_pass_kernel composites.
#include "common.cuh"

namespace stnerf {

constexpr int TM_BLOCK = 256;

// ---------------------------------------------------------------------------------------------------------
// Ordered hit compaction: the rays of each performer layer whose box was hit, in ascending ray order.
// sample_kernel's own lists are ordered within a block only (blocks claim their range with an atomicAdd), so the point order
// of a training step -- and with it the chunked weight-gradient sums of mlp_train.cu -- would change from call to call.
// Here: block counts, an exclusive scan in block order, then the writes.  No atomic is involved.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TM_BLOCK)
hit_count_kernel(const uint8_t* __restrict__ mask, long long n, int n_layers, const float* __restrict__ rays, int ray_stride,
                 int fid_shared, int nblk, int* __restrict__ block_counts, int* __restrict__ block_frac) {
  const long long r = (long long)blockIdx.x * TM_BLOCK + threadIdx.x;
  const bool live = r < n;
  for (int i = 1; i < n_layers; ++i) {
    const bool h = live && mask[i * n + r] != 0;
    bool frac = false;
    if (h) {                                      // MotionNet's batch-global "any fractional frame id" test (motion_net.py:53)
      const float f = rays[r * ray_stride + 6 + (fid_shared ? 0 : i)];
      frac = floorf(f) != f;
    }
    const int cnt = __syncthreads_count(h);
    const int any = __syncthreads_or(frac);
    if (threadIdx.x == 0) {
      block_counts[i * nblk + blockIdx.x] = cnt;
      block_frac[i * nblk + blockIdx.x] = any ? 1 : 0;
    }
  }
}

// one warp per performer layer: exclusive scan of the block counts in block order, the layer's total and its flag
__global__ void hit_scan_kernel(int* __restrict__ block_counts, const int* __restrict__ block_frac, int nblk,
                                int* __restrict__ totals, int* __restrict__ frac) {
  const int i = blockIdx.x + 1, lane = threadIdx.x;
  int carry = 0, any = 0;
  for (int b0 = 0; b0 < nblk; b0 += 32) {
    const int b = b0 + lane;
    const int v = b < nblk ? block_counts[i * nblk + b] : 0;
    any |= b < nblk ? block_frac[i * nblk + b] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (b < nblk) block_counts[i * nblk + b] = carry + x - v;
    carry += __shfl_sync(0xffffffffu, x, 31);
  }
  any = __any_sync(0xffffffffu, any);
  if (lane == 0) { totals[i] = carry; frac[i] = any; }
}

__global__ void __launch_bounds__(TM_BLOCK)
hit_write_kernel(const uint8_t* __restrict__ mask, long long n, int n_layers, const int* __restrict__ block_offsets, int nblk,
                 int* __restrict__ hit) {
  __shared__ int s_warp[TM_BLOCK / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long r = (long long)blockIdx.x * TM_BLOCK + tid;
  const bool live = r < n;
  for (int i = 1; i < n_layers; ++i) {
    const bool h = live && mask[i * n + r] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, h);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    if (h) {
      int pos = block_offsets[i * nblk + blockIdx.x] + __popc(b & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) pos += s_warp[w];
      hit[i * n + pos] = (int)r;
    }
    __syncthreads();
  }
}

size_t train_hits_scratch_ints(long long n, int n_layers) {
  const long long nblk = (n + TM_BLOCK - 1) / TM_BLOCK;
  return (size_t)(2 * nblk * n_layers + 2 * STNERF_MAX_LAYERS);
}

int launch_train_hits(const uint8_t* mask, long long n, int n_layers, const float* rays, int ray_stride, int fid_shared, int* hit,
                      int* scratch, int* totals_frac, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  const int nblk = (int)((n + TM_BLOCK - 1) / TM_BLOCK);
  int* block_counts = scratch;
  int* block_frac = scratch + (size_t)nblk * n_layers;
  hit_count_kernel<<<nblk, TM_BLOCK, 0, st>>>(mask, n, n_layers, rays, ray_stride, fid_shared, nblk, block_counts, block_frac);
  STNERF_LAUNCH_CHECK();
  if (n_layers > 1) {
    hit_scan_kernel<<<n_layers - 1, 32, 0, st>>>(block_counts, block_frac, nblk, totals_frac, totals_frac + STNERF_MAX_LAYERS);
    STNERF_LAUNCH_CHECK();
    hit_write_kernel<<<nblk, TM_BLOCK, 0, st>>>(mask, n, n_layers, block_counts, nblk, hit);
    STNERF_LAUNCH_CHECK();
  }
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Point assembly: the network inputs of one layer and pass, point p = (slot, k), ray = hit ? hit[slot] : slot.
// pos = march_point (the inverse edit included), dirs = d, times = frame-id column 6 + s.layer, xyzt = (pos, time).
// ---------------------------------------------------------------------------------------------------------
__global__ void train_points_kernel(const PointSrc s, long long P, float* __restrict__ pos, float* __restrict__ dirs,
                                    float* __restrict__ times, float* __restrict__ xyzt) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long slot = p / s.S;
  const int k = (int)(p - slot * s.S);
  const long long ray = s.hit ? (long long)s.hit[slot] : slot;
  const float* rp = s.rays + ray * s.ray_stride;
  const float dx = rp[3], dy = rp[4], dz = rp[5], tm = rp[6 + s.layer];
  float v[3];
  march_point(s, rp, s.t[ray * s.S + k], dx, dy, dz, v);
  if (pos) { pos[3 * p] = v[0]; pos[3 * p + 1] = v[1]; pos[3 * p + 2] = v[2]; }
  if (dirs) { dirs[3 * p] = dx; dirs[3 * p + 1] = dy; dirs[3 * p + 2] = dz; }
  if (times) times[p] = tm;
  if (xyzt) { xyzt[4 * p] = v[0]; xyzt[4 * p + 1] = v[1]; xyzt[4 * p + 2] = v[2]; xyzt[4 * p + 3] = tm; }
}

int launch_train_points(const PointSrc& s, long long P, float* pos, float* dirs, float* times, float* xyzt, cudaStream_t st) {
  if (P <= 0) return STNERF_OK;
  train_points_kernel<<<(int)((P + 255) / 256), 256, 0, st>>>(s, P, pos, dirs, times, xyzt);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Masked scatter: the density of one pass and layer as composite_pass_kernel composites it and the factor of its mask
// (pass_sigma); the backward multiplies the dense gradient by that factor.
// ---------------------------------------------------------------------------------------------------------
__global__ void train_scatter_kernel(const PassMask m, int layer, int fine, const float* __restrict__ t, int S,
                                     const int* __restrict__ hit, long long P,
                                     const float* __restrict__ rgb_c, const float* __restrict__ sigma_c, float* __restrict__ rgb,
                                     float* __restrict__ sigma, float* __restrict__ factor) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long slot = p / S;
  const int k = (int)(p - slot * S);
  const long long ray = hit ? (long long)hit[slot] : slot;
  const long long q = ray * S + k;
  float f;
  sigma[q] = pass_sigma(m, layer, fine, t[q], sigma_c[p], f);
  rgb[3 * q] = rgb_c[3 * p]; rgb[3 * q + 1] = rgb_c[3 * p + 1]; rgb[3 * q + 2] = rgb_c[3 * p + 2];
  if (factor) factor[p] = f;
}

__global__ void train_gather_kernel(int S, const int* __restrict__ hit, long long P, const float* __restrict__ factor,
                                    const float* __restrict__ d_rgb, const float* __restrict__ d_sigma, float* __restrict__ d_rgb_c,
                                    float* __restrict__ d_sigma_c) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const long long slot = p / S;
  const int k = (int)(p - slot * S);
  const long long ray = hit ? (long long)hit[slot] : slot;
  const long long q = ray * S + k;
  const float f = factor[p];
  d_sigma_c[p] = (d_sigma && f != 0.0f) ? d_sigma[q] * f : 0.0f;
#pragma unroll
  for (int a = 0; a < 3; ++a) d_rgb_c[3 * p + a] = d_rgb ? d_rgb[3 * q + a] : 0.0f;
}

int launch_train_scatter(const DevScene& sc, int layer, int fine, const float* t, long long n, int S, const int* hit, long long P,
                         const float* rgb_c, const float* sigma_c, float* rgb, float* sigma, float* factor, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  STNERF_CUDA(cudaMemsetAsync(rgb, 0, (size_t)n * S * 3 * sizeof(float), st));        // rays that miss the box: zeros
  STNERF_CUDA(cudaMemsetAsync(sigma, 0, (size_t)n * S * sizeof(float), st));
  if (P <= 0) return STNERF_OK;
  train_scatter_kernel<<<(int)((P + 255) / 256), 256, 0, st>>>(pass_mask(sc), layer, fine, t, S, hit, P, rgb_c, sigma_c, rgb, sigma,
                                                               factor);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

int launch_train_gather(int S, const int* hit, long long P, const float* factor, const float* d_rgb, const float* d_sigma,
                        float* d_rgb_c, float* d_sigma_c, cudaStream_t st) {
  if (P <= 0) return STNERF_OK;
  train_gather_kernel<<<(int)((P + 255) / 256), 256, 0, st>>>(S, hit, P, factor, d_rgb, d_sigma, d_rgb_c, d_sigma_c);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Fine-pass uniforms of every layer: the stream composite_pass_kernel draws when none are injected (Philox stream 64 + layer,
// keyed by the ray id, utils/sample_pdf.py:31).  u: [layer][ray][n2].
// ---------------------------------------------------------------------------------------------------------
__global__ void train_uniforms_kernel(long long n, int n2, int n_layers, uint64_t seed, RayIdMap idmap, float* __restrict__ u) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per_layer = n * n2;
  if (idx >= per_layer * n_layers) return;
  const int i = (int)(idx / per_layer);
  const long long rem = idx - (long long)i * per_layer;
  const long long r = rem / n2;
  const int j = (int)(rem - r * n2);
  u[idx] = philox_uniform(seed, 64u + (uint32_t)i, idmap(r), (uint32_t)j);
}

int launch_train_uniforms(long long n, int n2, int n_layers, uint64_t seed, RayIdMap idmap, float* u, cudaStream_t st) {
  const long long total = n * n2 * n_layers;
  if (total <= 0) return STNERF_OK;
  train_uniforms_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(n, n2, n_layers, seed, idmap, u);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // namespace stnerf
