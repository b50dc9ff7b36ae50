// Alpha compositing, inverse-CDF resampling and the depth-ordered merge of all layers (warp-per-ray kernels).
//
// Restates layers/render_layer.py:8-58 (gen_weight / VolumeRenderer), utils/sample_pdf.py:18-63 and the
// sort-merge of modeling/layered_rfrender.py:425-448 (coarse) / :587-606 (fine).  fp32, compiled with
// -fmad=false so every product/sum rounds like the separate ATen ops of the reference.  Scans use warp
// shuffles (tree order), so results agree with torch.cumprod / cumsum to a few ulp, not bit for bit.
#include <algorithm>
#include <math_constants.h>
#include "common.cuh"
#include "resample.cuh"

namespace stnerf {

constexpr unsigned FULL = 0xffffffffu;
using rs::lower_bound_s;
using rs::upper_bound_s;
using rs::write_pixel;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
  return v;
}
__device__ __forceinline__ float warp_incl_mul(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float n = __shfl_up_sync(FULL, v, d);
    if (lane >= d) v = v * n;
  }
  return v;
}
__device__ __forceinline__ float warp_incl_add(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float n = __shfl_up_sync(FULL, v, d);
    if (lane >= d) v = v + n;
  }
  return v;
}
__device__ __forceinline__ float sigmoidf_ref(float x) { return 1.0f / (1.0f + expf(-x)); }

// order-preserving map float -> uint32 (total order incl. negatives; -0.0 and +0.0 share a key, as they compare equal in the
// reference's torch.sort and in the rank merge's <= / <)
__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t u = __float_as_uint(f + 0.0f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// In-shared-memory bitonic sort of P (power of two) elements by one warp.  Every lane owns whole compare-exchange pairs
// (pair m of a stride-j step = elements i and i|j with i = m's bits with a zero inserted at bit log2 j), so no lane idles.
template <typename T>
__device__ __forceinline__ void warp_bitonic_sort(T* a, int P, int lane) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int m = lane; m < (P >> 1); m += 32) {
        const int i = ((m & ~(j - 1)) << 1) | (m & (j - 1));
        const int p = i | j;
        const T x = a[i], y = a[p];
        const bool up = (i & k) == 0;
        if ((x > y) == up) { a[i] = y; a[p] = x; }
      }
      __syncwarp();
    }
  }
}

// warp-uniform: is a[0..n) non-decreasing?
__device__ __forceinline__ bool warp_is_ascending(const float* a, int n, int lane) {
  bool ok = true;
  for (int k = lane; k + 1 < n; k += 32) ok = ok && (a[k] <= a[k + 1]);
  return __all_sync(FULL, ok);
}

// gen_weight + VolumeRenderer.forward over `count` samples: sample j lives at position `at(j)` of the per-warp depth /
// density arrays and its colour is `rgb_at(j)` (already through the sigmoid).  All lanes return the reduced
// color/depth/acc.  If w_out != null, w_out[j] = weight.
template <typename At, typename Rgb>
__device__ __forceinline__ void composite_run(int count, At at, Rgb rgb_at, const float* s_t, const float* s_sig, float boarder,
                                              float near_cut, bool use_near_cut, float* w_out, int lane, float out[5]) {
  float carry = 1.0f;                      // cumprod of [1, 1-alpha+1e-10, ...][:-1]  (render_layer.py:15)
  float cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f, ca = 0.f;
  for (int base = 0; base < count; base += 32) {
    const int j = base + lane;
    const bool valid = j < count;
    float f = 1.0f, alpha = 0.0f, tj = 0.0f;
    if (valid) {
      const int pj = at(j);
      tj = s_t[pj];
      const float delta = (j == count - 1) ? boarder : (s_t[at(j + 1)] - tj);     // render_layer.py:37-40
      float sg = s_sig[pj];
      if (use_near_cut && tj < near_cut) sg = 0.0f;                                // layered_rfrender.py:605
      const float e = expf(-fmaxf(sg, 0.0f) * delta);                              // render_layer.py:11
      alpha = 1.0f - e;
      f = (1.0f - alpha) + 1e-10f;                                                 // render_layer.py:12
    }
    const float incl = warp_incl_mul(f, lane);
    float excl = __shfl_up_sync(FULL, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float T = carry * excl;
    carry = carry * __shfl_sync(FULL, incl, 31);
    if (valid) {
      const float w = alpha * T;
      if (w_out) w_out[j] = w;
      if (w != 0.0f) {                     // a zero weight adds exactly +0 to every sum: its colour is neither read nor squashed
        const float3 c = rgb_at(j);        // (most samples: empty space has sigma <= 0.  Only a NaN colour would differ.)
        cr += c.x * w;                                                             // render_layer.py:45
        cg += c.y * w;
        cb += c.z * w;
        cd += w * tj;                                                              // :46
        ca += w;                                                                   // :47
      }
    }
  }
  out[0] = warp_sum(cr); out[1] = warp_sum(cg); out[2] = warp_sum(cb);
  out[3] = warp_sum(cd); out[4] = warp_sum(ca);
}

// utils/sample_pdf.py:18-63 for one ray: t[n1] (any order), w[n1] full weights, n2 uniforms -> z written to
// zbuf[0..n2).  cdf is an (n1-1)-float scratch.
template <typename U>
__device__ __forceinline__ void sample_pdf_ray(const float* s_t, const float* s_w, int n1, int n2, U get_u,
                                               float* cdf, float* zbuf, int lane) {
  const int nb = n1 - 2;                      // weights[..., 1:-1]
  float part = 0.f;
  for (int m = lane; m < nb; m += 32) part += s_w[m + 1] + 1e-5f;                  // :21
  const float tot = warp_sum(part);
  float carry = 0.f;
  if (lane == 0) cdf[0] = 0.0f;                                                    // :24
  for (int base = 0; base < nb; base += 32) {
    const int m = base + lane;
    const float pdf = (m < nb) ? (s_w[m + 1] + 1e-5f) / tot : 0.0f;                // :22
    const float incl = warp_incl_add(pdf, lane);
    if (m < nb) cdf[m + 1] = carry + incl;                                         // :23
    carry = carry + __shfl_sync(FULL, incl, 31);
  }
  __syncwarp();
  const int nc = n1 - 1;                      // len(cdf) == len(bins)
  for (int j = lane; j < n2; j += 32) {
    const float uu = get_u(j);
    const int lo = upper_bound_s(cdf, nc, uu);                                     // :47
    const int below = max(lo - 1, 0);                                              // :48
    const int above = min(lo, nc - 1);                                             // :49
    const float cb = cdf[below], ca = cdf[above];
    const float bb = 0.5f * (s_t[below + 1] + s_t[below]);                         // :20
    const float ba = 0.5f * (s_t[above + 1] + s_t[above]);
    float den = ca - cb;
    if (den < 1e-5f) den = 1.0f;                                                   // :59
    const float tt = (uu - cb) / den;
    zbuf[j] = bb + tt * (ba - bb);                                                 // :61
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------------------
// K5 / K6: one pass (coarse or fine) of per-layer + merged compositing for a chunk of rays.
// ---------------------------------------------------------------------------------------------------------
// Per warp in shared memory: depth and (masked) density of every gathered sample, the coarse weights / cdf while
// resampling, and one scratch area shared by the resampling sort and the merge order.  Colours are NOT staged: they
// are read straight from the network output (coalesced in the per-layer pass, gathered through L1/L2 in the merged pass),
// which keeps the footprint at 8-10 bytes per sample and ~32 warps resident per SM.
struct PassSmem {
  int per_warp_floats, off_sig, off_w, off_cdf, off_sort, sort_floats;
};

__host__ __device__ inline int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

static PassSmem pass_layout(int l, int S, int n2, bool regs) {
  PassSmem L;
  const int tot = l * S;
  L.off_sig = tot;
  L.off_w = 2 * tot;
  L.off_cdf = L.off_w + ((n2 > 0 && !regs) ? S : 0);      // the register-resident path keeps the weights in registers ...
  L.off_sort = L.off_cdf + (n2 > 0 ? S : 0);
  int sf = (tot + 1) / 2;                     // merge order: one uint16 per sample
  if (!regs) {                                // ... and sorts / merges there too: no sort area beyond the merge order
    if (n2 > 0 && next_pow2(S + n2) > sf) sf = next_pow2(S + n2);
    if (n2 > 0 && S + next_pow2(n2) > sf) sf = S + next_pow2(n2);
  }
  L.sort_floats = sf;
  L.per_warp_floats = (L.off_sort + sf + 3) & ~3;
  return L;
}

constexpr int ORDER_K_BITS = 9;               // STNERF_MAX_S = 512 samples per list, STNERF_MAX_LAYERS = 8 lists
static_assert(STNERF_MAX_S <= (1 << ORDER_K_BITS) && STNERF_MAX_LAYERS <= (1 << (16 - ORDER_K_BITS)), "merge order code is 16 bits");

// NT, NZ > 0: the coarse pass' per-layer composite + resampling runs register-resident (resample.cuh: NT = ceil(n1/32) depth slots
// and NZ = pow2 >= ceil(n2/32) new-depth slots per lane); NT == 0: generic shared-memory path (fine pass, unusual sample counts).
template <int NT, int NZ>
__global__ void __launch_bounds__(256, 3) composite_pass_kernel(const CompositeArgs a, const DevScene scene, int n_layers, const PassSmem L) {
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float* base = smem + (size_t)warp * L.per_warp_floats;
  float* s_t = base;
  float* s_sig = base + L.off_sig;
  float* s_w = base + L.off_w;
  float* s_cdf = base + L.off_cdf;
  float* s_sortf = base + L.off_sort;
  uint16_t* order = reinterpret_cast<uint16_t*>(s_sortf);

  const int S = a.S, n2 = a.n2;
  const bool fine = a.fine != 0;
  const float near_p = scene.near_plane, boarder = scene.boarder;
  const PassMask pm = pass_mask(scene);
  const long long plane = 5 * a.n_total;
  const bool pixels = a.pixel_layout != 0;
  unsigned shown_mask = 1u;
  for (int i = 1; i < n_layers; ++i) shown_mask |= (scene.shown[i] != 0 ? 1u : 0u) << i;

  for (long long r = (long long)blockIdx.x * wpb + warp; r < a.n; r += (long long)gridDim.x * wpb) {
    const long long rg = a.ray_base + r;
    int n_m = 0;                                  // entries gathered for the merged composite
    unsigned slot_layers = 0;                     // 4 bits per gathered list: which layer it is
    bool all_asc = true;                          // every gathered list is non-decreasing (always true for fine passes)
    float single[5] = {0.f, 0.f, 0.f, 0.f, 0.f};  // pixel of the background layer's own composite (reused when it is the only list)
    bool have_single = false;
    for (int i = 0; i < n_layers; ++i) {
      float* oimg = a.out ? a.out + (size_t)(1 + i) * plane : nullptr;
      const bool hit = (i == 0) || (a.mask[i * a.mask_layer_stride + r] != 0);
      if (!hit) {                                 // all samples at t=-1000 with sigma 0: inert (SURVEY A.10)
        const float z5[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        write_pixel(oimg, rg, a.n_total, pixels, z5, lane);
        continue;
      }
      const bool shown = (shown_mask >> i) & 1u;
      const int off = n_m;
      slot_layers |= (unsigned)i << (4 * (n_m / S));
      const float* tp = a.t + i * a.t_layer_stride + r * S;
      const float4* rp = reinterpret_cast<const float4*>(a.raw + i * a.raw_layer_stride) + r * S;
      for (int k = lane; k < S; k += 32) {
        const float tk = tp[k];
        float sg = 0.f, factor;
        if (shown) sg = pass_sigma(pm, i, fine, tk, rp[k].w, factor);
        s_t[off + k] = tk;
        s_sig[off + k] = sg;
      }
      __syncwarp();
      const bool done_elsewhere = (a.skip_layers >> i) & 1u;       // per-layer image + resampling produced by the fused SpaceNet kernel
      if (done_elsewhere) {
        all_asc = all_asc && warp_is_ascending(s_t + off, S, lane);
        n_m += S;
        continue;
      }
      const bool want_w = (!fine) && n2 > 0;
      if (NT > 0 && !fine) {
        // register-resident per-layer composite + hierarchical resampling of this layer (layered_rfrender.py:435-463)
        constexpr int NTr = NT > 0 ? NT : 1, NZr = NZ > 0 ? NZ : 1;
        float tr[NTr], sr[NTr];
#pragma unroll
        for (int q = 0; q < NTr; ++q) {
          const int k = q * 32 + lane;
          tr[q] = k < S ? s_t[off + k] : 0.f;
          sr[q] = k < S ? s_sig[off + k] : 0.f;
        }
        const float* up = a.u ? a.u + i * a.u_layer_stride + r * n2 : nullptr;
        const uint64_t seed = a.seed;
        const unsigned long long gid = a.idmap(rg);
        rs::LayerOut lo;
        rs::composite_resample_ray<NTr, NZr>(
            tr, sr, S, want_w ? n2 : 0, boarder,
            [rp, shown, lane](int q) {
              if (!shown) return make_float3(0.5f, 0.5f, 0.5f);
              const float4 v = __ldg(rp + q * 32 + lane);
              return make_float3(sigmoidf_ref(v.x), sigmoidf_ref(v.y), sigmoidf_ref(v.z));
            },
            [up, seed, i, gid](int j) { return up ? up[j] : philox_uniform(seed, 64u + (uint32_t)i, gid, (uint32_t)j); },
            s_cdf, want_w ? a.t_fine + i * a.tf_layer_stride + r * (S + n2) : nullptr, lane, lo,
            (want_w && a.z_new) ? a.z_new + i * a.zn_layer_stride + r * n2 : nullptr,
            (want_w && a.z_new) ? a.src_map + i * a.sm_layer_stride + r * (S + n2) : nullptr);
        write_pixel(oimg, rg, a.n_total, pixels, lo.pix, lane);
        if (i == 0) {
#pragma unroll
          for (int q = 0; q < 5; ++q) single[q] = lo.pix[q];
          have_single = true;
        }
        all_asc = all_asc && warp_is_ascending(s_t + off, S, lane);
        n_m += S;
        continue;
      }
      const bool asc = warp_is_ascending(s_t + off, S, lane);
      all_asc = all_asc && asc;
      float o5[5];
      // a hidden layer contributes sigmoid(0) colours with zero weight (its network output is never read)
      composite_run(S, [off](int j) { return off + j; },
                    [rp, shown](int j) {
                      if (!shown) return make_float3(0.5f, 0.5f, 0.5f);
                      const float4 v = __ldg(rp + j);
                      return make_float3(sigmoidf_ref(v.x), sigmoidf_ref(v.y), sigmoidf_ref(v.z));
                    },
                    s_t, s_sig, boarder, 0.f, false, want_w ? s_w : nullptr, lane, o5);
      write_pixel(oimg, rg, a.n_total, pixels, o5, lane);
      if (i == 0) {
#pragma unroll
        for (int q = 0; q < 5; ++q) single[q] = o5[q];
        have_single = true;
      }
      __syncwarp();
      if (want_w) {
        // hierarchical resampling of this layer (layered_rfrender.py:459-463)
        const float* up = a.u ? a.u + i * a.u_layer_stride + r * n2 : nullptr;
        const uint64_t seed = a.seed;
        const unsigned long long gid = a.idmap(rg);
        sample_pdf_ray(s_t + off, s_w, S, n2,
                       [up, seed, i, gid](int j) {
                         return up ? up[j] : philox_uniform(seed, 64u + (uint32_t)i, gid, (uint32_t)j);
                       },
                       s_cdf, s_sortf + S, lane);
        const int S2 = S + n2;
        float* tf = a.t_fine + i * a.tf_layer_stride + r * S2;
        if (asc) {
          // torch.sort(cat(t, z)) (:462) = sort the n2 new depths, then rank-merge with the ascending coarse depths
          float* zs = s_sortf + S;
          const int P2 = next_pow2(n2);
          for (int k = n2 + lane; k < P2; k += 32) zs[k] = CUDART_INF_F;
          __syncwarp();
          warp_bitonic_sort(zs, P2, lane);
          for (int k = lane; k < S; k += 32) {
            const float v = s_t[off + k];
            tf[k + lower_bound_s(zs, n2, v)] = v;
          }
          for (int k = lane; k < n2; k += 32) {
            const float v = zs[k];
            tf[k + upper_bound_s(s_t + off, S, v)] = v;
          }
        } else {
          const int P = next_pow2(S2);
          for (int k = lane; k < S; k += 32) s_sortf[k] = s_t[off + k];
          for (int k = S2 + lane; k < P; k += 32) s_sortf[k] = CUDART_INF_F;
          __syncwarp();
          warp_bitonic_sort(s_sortf, P, lane);
          for (int k = lane; k < S2; k += 32) tf[k] = s_sortf[k];
        }
        __syncwarp();
      }
      n_m += S;
    }
    // ---- merged composite over every hit layer's samples, ordered by (t, cat index)  (:425-448 / :587-606)
    if (a.out != nullptr) {
      const int n_lists = n_m / S;
      // One list only (the ray hits nothing but the background) and no sample in front of the near plane: the merged composite is
      // the per-layer composite of that list, operation for operation -- its pixel was just computed (kept in `single`).
      if (n_lists == 1 && have_single && !(fine && s_t[0] < near_p) && all_asc) {
        write_pixel(a.out, rg, a.n_total, pixels, single, lane);
        __syncwarp();
        continue;
      }
      if (all_asc) {
        // every list is sorted: the stable (t, cat index) order is a rank computation -- position of sample (h,k) =
        // k + #(samples of earlier lists with t' <= t) + #(samples of later lists with t' < t)
        for (int e = lane; e < n_m; e += 32) {
          const int h = e / S, k = e - h * S;
          const float key = s_t[e];
          int pos = k;
          for (int h2 = 0; h2 < n_lists; ++h2) {
            if (h2 == h) continue;
            pos += (h2 < h) ? upper_bound_s(s_t + h2 * S, S, key) : lower_bound_s(s_t + h2 * S, S, key);
          }
          order[pos] = (uint16_t)((h << ORDER_K_BITS) | k);
        }
      } else {
        // some list is out of order (degenerate boxes, NaNs): brute-force stable rank under the total order of float_key.
        // O(n^2), never taken by well-formed rays.
        for (int e = lane; e < n_m; e += 32) {
          const int h = e / S, k = e - h * S;
          const uint32_t key = float_key(s_t[e]);
          int pos = 0;
          for (int e2 = 0; e2 < n_m; ++e2) {
            const uint32_t k2 = float_key(s_t[e2]);
            pos += (k2 < key || (k2 == key && e2 < e)) ? 1 : 0;
          }
          order[pos] = (uint16_t)((h << ORDER_K_BITS) | k);
        }
      }
      __syncwarp();
      float o5[5];
      const float* raw = a.raw;
      const long long rls = a.raw_layer_stride;
      composite_run(n_m,
                    [order, S](int j) { const int c = order[j]; return (c >> ORDER_K_BITS) * S + (c & ((1 << ORDER_K_BITS) - 1)); },
                    [order, S, raw, rls, r, slot_layers, shown_mask](int j) {
                      const int c = order[j];
                      const int layer = (slot_layers >> (4 * (c >> ORDER_K_BITS))) & 15u;
                      if (!((shown_mask >> layer) & 1u)) return make_float3(0.5f, 0.5f, 0.5f);
                      const float4 v = __ldg(reinterpret_cast<const float4*>(raw + layer * rls) + r * S + (c & ((1 << ORDER_K_BITS) - 1)));
                      return make_float3(sigmoidf_ref(v.x), sigmoidf_ref(v.y), sigmoidf_ref(v.z));
                    },
                    s_t, s_sig, boarder, near_p, fine, nullptr, lane, o5);
      write_pixel(a.out, rg, a.n_total, pixels, o5, lane);
      __syncwarp();
    }
  }
}

// SMs of the current device: the grids below are capped at a few waves of resident blocks
static int device_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) {
    cudaGetLastError();
    return 1;
  }
  return n;
}

template <int NT, int NZ>
static int launch_pass_t(const CompositeArgs& a, const DevScene& scene, int n_layers, const PassSmem& L, cudaStream_t st) {
  const size_t per_warp = (size_t)L.per_warp_floats * sizeof(float);
  // blocks of up to 8 warps, as many blocks per SM as shared memory allows (228 KB per SM, 1 KB reserved per block)
  int wpb = 8;
  while (wpb > 1 && per_warp * wpb > 100 * 1024) wpb >>= 1;
  if (per_warp * wpb > 200 * 1024) return STNERF_EINVAL;
  const size_t smem = per_warp * wpb;
  auto kern = composite_pass_kernel<NT, NZ>;
  STNERF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // three blocks of 8 warps per SM (85 registers per thread): ask for the largest shared-memory carve-out so that shared memory
  // does not cap the residency below that
  STNERF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  int per_sm = (int)((227 * 1024) / (smem + 1024));
  if (per_sm * wpb > 64) per_sm = 64 / wpb;
  if (per_sm < 1) per_sm = 1;
  long long blocks = (a.n + wpb - 1) / wpb;
  const long long cap = (long long)device_sms() * per_sm * 4;
  if (blocks > cap) blocks = cap;
  kern<<<(int)blocks, wpb * 32, smem, st>>>(a, scene, n_layers, L);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

bool composite_pass_in_registers(int S, int n2, int fine) { return !fine && S <= 128 && n2 <= 256; }

int launch_composite_pass(const CompositeArgs& a, const DevScene& scene, int n_layers, cudaStream_t st, bool force_generic) {
  if (a.n <= 0) return STNERF_OK;
  if (a.S > STNERF_MAX_S || n_layers > STNERF_MAX_LAYERS) return STNERF_EINVAL;
  const bool regs = composite_pass_in_registers(a.S, a.n2, a.fine) && !force_generic;
  const PassSmem L = pass_layout(n_layers, a.S, a.fine ? 0 : a.n2, regs);
  if (regs) {
    // coarse pass: register-resident per-layer composite + resampling, instantiated for the slot counts in use
    const int nt = (a.S + 31) / 32, nzr = (std::max(a.n2, 1) + 31) / 32;
    const int nz = nzr <= 1 ? 1 : nzr <= 2 ? 2 : nzr <= 4 ? 4 : 8;
#define STNERF_PASS_CASE(T_, Z_) if (nt == T_ && nz == Z_) return launch_pass_t<T_, Z_>(a, scene, n_layers, L, st);
    STNERF_PASS_CASE(1, 1) STNERF_PASS_CASE(1, 2) STNERF_PASS_CASE(1, 4) STNERF_PASS_CASE(1, 8)
    STNERF_PASS_CASE(2, 1) STNERF_PASS_CASE(2, 2) STNERF_PASS_CASE(2, 4) STNERF_PASS_CASE(2, 8)
    STNERF_PASS_CASE(3, 1) STNERF_PASS_CASE(3, 2) STNERF_PASS_CASE(3, 4) STNERF_PASS_CASE(3, 8)
    STNERF_PASS_CASE(4, 1) STNERF_PASS_CASE(4, 2) STNERF_PASS_CASE(4, 4) STNERF_PASS_CASE(4, 8)
#undef STNERF_PASS_CASE
  }
  return launch_pass_t<0, 0>(a, scene, n_layers, L, st);
}

// ---------------------------------------------------------------------------------------------------------
// Unit entry point a10: VolumeRenderer.forward on explicit (t, rgb, sigma) arrays.  Warp per ray, streaming:
// 20 B/sample in, 4 B/sample out (weights) -- the HBM-roofline kernel of the compositing stage.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) composite_simple_kernel(const float* __restrict__ t, const float* __restrict__ rgb,
                                                              const float* __restrict__ sigma, long long n, int S, float boarder,
                                                              float* __restrict__ color, float* __restrict__ depth,
                                                              float* __restrict__ acc, float* __restrict__ w) {
  constexpr int RB = 6;                      // rows of 32 samples whose loads are issued together (memory-level parallelism)
  const int lane = threadIdx.x & 31;
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = wid; r < n; r += nw) {
    const float* tp = t + r * S;
    const float* sp = sigma + r * S;
    const float* cp = rgb + r * S * 3;
    float carry = 1.0f, cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f, ca = 0.f;
    for (int base = 0; base < S; base += 32 * RB) {
      float tv[RB + 1], sv[RB], c0[RB], c1[RB], c2[RB];
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        const int j = base + q * 32 + lane;
        const bool valid = j < S;
        tv[q] = valid ? __ldg(tp + j) : 0.0f;
        sv[q] = valid ? __ldg(sp + j) : 0.0f;
        c0[q] = valid ? __ldg(cp + 3 * j) : 0.0f;
        c1[q] = valid ? __ldg(cp + 3 * j + 1) : 0.0f;
        c2[q] = valid ? __ldg(cp + 3 * j + 2) : 0.0f;
      }
      {                                      // first depth of the next batch (delta of this batch's last sample)
        const int jn = base + RB * 32;
        tv[RB] = (lane == 0 && jn < S) ? __ldg(tp + jn) : 0.0f;
      }
#pragma unroll
      for (int q = 0; q < RB; ++q) {
        const int j = base + q * 32 + lane;
        if (base + q * 32 >= S) break;       // warp-uniform
        const bool valid = j < S;
        const float tj = tv[q];
        float tn = __shfl_down_sync(FULL, tj, 1);
        const float tfirst_next = __shfl_sync(FULL, tv[q + 1], 0);
        if (lane == 31) tn = tfirst_next;
        float f = 1.0f, alpha = 0.0f;
        if (valid) {
          const float delta = (j == S - 1) ? boarder : (tn - tj);
          const float e = expf(-fmaxf(sv[q], 0.0f) * delta);
          alpha = 1.0f - e;
          f = (1.0f - alpha) + 1e-10f;
        }
        const float incl = warp_incl_mul(f, lane);
        float excl = __shfl_up_sync(FULL, incl, 1);
        if (lane == 0) excl = 1.0f;
        const float T = carry * excl;
        carry = carry * __shfl_sync(FULL, incl, 31);
        if (valid) {
          const float ww = alpha * T;
          if (w) w[r * S + j] = ww;
          cr += sigmoidf_ref(c0[q]) * ww;
          cg += sigmoidf_ref(c1[q]) * ww;
          cb += sigmoidf_ref(c2[q]) * ww;
          cd += ww * tj;
          ca += ww;
        }
      }
    }
    cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb); cd = warp_sum(cd); ca = warp_sum(ca);
    if (lane == 0) {
      color[3 * r] = cr; color[3 * r + 1] = cg; color[3 * r + 2] = cb;
      depth[r] = cd;
      acc[r] = ca;
    }
  }
}

int launch_composite_simple(const float* t, const float* rgb, const float* sigma, long long n, int S, float boarder,
                            float* color, float* depth, float* acc, float* w, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  const int block = 256;
  long long blocks = (n * 32 + block - 1) / block;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  composite_simple_kernel<<<(int)blocks, block, 0, st>>>(t, rgb, sigma, n, S, boarder, color, depth, acc, w);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Gradient of composite_simple_kernel's outputs (color, depth, acc, w) with respect to rgb and sigma.  Warp per ray.
//   w_k = alpha_k T_k,  T_k = prod_{j<k} f_j,  f_j = 1 - alpha_j + 1e-10,  alpha = 1 - exp(-relu(sigma) delta)
//   g_k = d_color . sigmoid(rgb_k) + d_depth t_k + d_acc + d_w_k                      (dL/dw_k)
//   d_alpha_k = T_k g_k - (sum_{m>k} w_m g_m) / f_k                                    (f_k >= 1e-10: never 0)
//   d_sigma_k = d_alpha_k (delta_k exp(-relu(sigma_k) delta_k)) [sigma_k > 0],   d_rgb_k = d_color w_k y (1 - y)
// Nothing is saved by the forward: pass 1 recomputes the transmittance at the start of every 32-sample row with the
// forward's arithmetic (same rows, same scan, so T and w are the forward's bits) into shared memory; pass 2 walks the rows
// from the last to the first, carrying the suffix sum of w g down with a reverse warp scan.  Every output element is
// written once by one lane: no atomics, and a ray's gradients do not depend on the rest of the batch.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_incl_add_rev(float v, int lane) {      // sum over lanes >= lane
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float n = __shfl_down_sync(FULL, v, d);
    if (lane + d < 32) v = v + n;
  }
  return v;
}

// delta, exp(-relu(sigma) delta), alpha and f of sample j < S of one ray, as composite_simple_kernel computes them
__device__ __forceinline__ void backward_sample(const float* tp, const float* sp, int S, int j, float boarder, float& tj,
                                                float& sg, float& delta, float& e, float& alpha, float& f) {
  tj = __ldg(tp + j);
  sg = __ldg(sp + j);
  delta = (j == S - 1) ? boarder : (__ldg(tp + j + 1) - tj);
  e = expf(-fmaxf(sg, 0.0f) * delta);
  alpha = 1.0f - e;
  f = (1.0f - alpha) + 1e-10f;
}

__global__ void __launch_bounds__(256) composite_backward_kernel(
    const float* __restrict__ t, const float* __restrict__ rgb, const float* __restrict__ sigma, long long n, int S,
    float boarder, const float* __restrict__ d_color, const float* __restrict__ d_depth, const float* __restrict__ d_acc,
    const float* __restrict__ d_w, float* __restrict__ d_rgb, float* __restrict__ d_sigma) {
  extern __shared__ float s_rows[];
  const int lane = threadIdx.x & 31;
  const int rows = (S + 31) >> 5;
  float* s_carry = s_rows + (size_t)(threadIdx.x >> 5) * rows;      // T at the first sample of every row
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = wid; r < n; r += nw) {
    const float* tp = t + r * S;
    const float* sp = sigma + r * S;
    const float* cp = rgb + r * S * 3;
    float carry = 1.0f;
    for (int row = 0; row < rows; ++row) {
      const int j = row * 32 + lane;
      float f = 1.0f;
      if (j < S) {
        float tj, sg, delta, e, alpha;
        backward_sample(tp, sp, S, j, boarder, tj, sg, delta, e, alpha, f);
      }
      const float incl = warp_incl_mul(f, lane);
      if (lane == 0) s_carry[row] = carry;
      carry = carry * __shfl_sync(FULL, incl, 31);
    }
    __syncwarp();
    const float dcr = d_color ? __ldg(d_color + 3 * r) : 0.0f;
    const float dcg = d_color ? __ldg(d_color + 3 * r + 1) : 0.0f;
    const float dcb = d_color ? __ldg(d_color + 3 * r + 2) : 0.0f;
    const float dd = d_depth ? __ldg(d_depth + r) : 0.0f;
    const float da = d_acc ? __ldg(d_acc + r) : 0.0f;
    float later_rows = 0.0f;                 // sum of w_m g_m over the rows after this one
    for (int row = rows - 1; row >= 0; --row) {
      const int j = row * 32 + lane;
      const bool valid = j < S;
      float tj = 0.f, sg = 0.f, delta = 0.f, e = 1.f, alpha = 0.f, f = 1.f;
      float y0 = 0.f, y1 = 0.f, y2 = 0.f, g = 0.f;
      if (valid) {
        backward_sample(tp, sp, S, j, boarder, tj, sg, delta, e, alpha, f);
        if (d_color) {
          y0 = sigmoidf_ref(__ldg(cp + 3 * j));
          y1 = sigmoidf_ref(__ldg(cp + 3 * j + 1));
          y2 = sigmoidf_ref(__ldg(cp + 3 * j + 2));
          g = dcr * y0 + dcg * y1 + dcb * y2;
        }
        if (d_depth) g = g + dd * tj;       // NULL upstreams add nothing (not 0 * t: t may be huge)
        if (d_acc) g = g + da;
        if (d_w) g = g + __ldg(d_w + r * S + j);
      }
      const float incl = warp_incl_mul(f, lane);
      float excl = __shfl_up_sync(FULL, incl, 1);
      if (lane == 0) excl = 1.0f;
      const float T = s_carry[row] * excl;
      const float w = alpha * T;
      const float sfx = warp_incl_add_rev(valid ? w * g : 0.0f, lane);
      float after = __shfl_down_sync(FULL, sfx, 1);
      if (lane == 31) after = 0.0f;
      const float later = later_rows + after;
      later_rows = later_rows + __shfl_sync(FULL, sfx, 0);
      if (valid) {
        const float dalpha = T * g - later / f;
        d_sigma[r * S + j] = sg > 0.0f ? dalpha * (delta * e) : 0.0f;     // torch's relu: no gradient at exactly 0
        float* o = d_rgb + (r * S + j) * 3;
        o[0] = dcr * w * (1.0f - y0) * y0;
        o[1] = dcg * w * (1.0f - y1) * y1;
        o[2] = dcb * w * (1.0f - y2) * y2;
      }
    }
    __syncwarp();
  }
}

int launch_composite_backward(const float* t, const float* rgb, const float* sigma, long long n, int S, float boarder,
                              const float* d_color, const float* d_depth, const float* d_acc, const float* d_w, float* d_rgb,
                              float* d_sigma, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  const size_t per_warp = (size_t)((S + 31) / 32) * sizeof(float);
  int wpb = 8;
  while (wpb > 1 && per_warp * wpb > 48 * 1024) wpb >>= 1;
  const size_t smem = per_warp * wpb;
  if (smem > 200 * 1024) return STNERF_EINVAL;                  // more than 1.6 M samples per ray
  if (smem > 48 * 1024)
    STNERF_CUDA(cudaFuncSetAttribute(composite_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  long long blocks = (n + wpb - 1) / wpb;
  if (blocks > (long long)device_sms() * 64 / wpb) blocks = (long long)device_sms() * 64 / wpb;
  composite_backward_kernel<<<(int)blocks, wpb * 32, smem, st>>>(t, rgb, sigma, n, S, boarder, d_color, d_depth, d_acc, d_w,
                                                                 d_rgb, d_sigma);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Unit entry point a11: sample_pdf (+ optional sort-merge with the coarse depths).
// ---------------------------------------------------------------------------------------------------------
__global__ void sample_pdf_kernel(const float* __restrict__ t, const float* __restrict__ w, const float* __restrict__ u,
                                  long long n, int n1, int n2, float* __restrict__ z, float* __restrict__ t_fine,
                                  int per_warp_floats) {
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float* s_t = smem + (size_t)warp * per_warp_floats;
  float* s_w = s_t + n1;
  float* s_cdf = s_w + n1;
  float* s_sort = s_cdf + n1;
  const int S2 = n1 + n2, P = next_pow2(S2);
  for (long long r = (long long)blockIdx.x * wpb + warp; r < n; r += (long long)gridDim.x * wpb) {
    for (int k = lane; k < n1; k += 32) { s_t[k] = t[r * n1 + k]; s_w[k] = w[r * n1 + k]; }
    __syncwarp();
    const float* up = u + r * n2;
    sample_pdf_ray(s_t, s_w, n1, n2, [up](int j) { return up[j]; }, s_cdf, s_sort + n1, lane);
    if (z) for (int j = lane; j < n2; j += 32) z[r * n2 + j] = s_sort[n1 + j];
    if (t_fine) {
      for (int k = lane; k < n1; k += 32) s_sort[k] = s_t[k];
      for (int k = S2 + lane; k < P; k += 32) s_sort[k] = CUDART_INF_F;
      __syncwarp();
      warp_bitonic_sort(s_sort, P, lane);
      for (int k = lane; k < S2; k += 32) t_fine[r * S2 + k] = s_sort[k];
    }
    __syncwarp();
  }
}

int launch_sample_pdf(const float* t, const float* w, const float* u, long long n, int n1, int n2, float* z,
                      float* t_fine, cudaStream_t st) {
  if (n <= 0) return STNERF_OK;
  if (n1 < 3 || n2 < 1) return STNERF_EINVAL;
  const int per_warp = ((3 * n1 + next_pow2(n1 + n2)) + 3) & ~3;
  const int wpb = 4;
  const size_t smem = (size_t)per_warp * wpb * sizeof(float);
  if (smem > 48 * 1024)
    STNERF_CUDA(cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  long long blocks = (n + wpb - 1) / wpb;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  sample_pdf_kernel<<<(int)blocks, wpb * 32, smem, st>>>(t, w, u, n, n1, n2, z, t_fine, per_warp);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // namespace stnerf
