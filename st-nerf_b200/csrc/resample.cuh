// Register-resident warp-per-ray compositing + hierarchical resampling of ONE layer's coarse samples.
//
// Restates layers/render_layer.py:8-58 (gen_weight / VolumeRenderer), utils/sample_pdf.py:18-63 and the
// `torch.sort(torch.cat([t, z]))` of modeling/layered_rfrender.py:459-463 for one (ray, layer) handled by one warp.
// Everything a lane needs lives in registers (sample k of the ray sits in lane k % 32, slot k / 32); the only scratch is
// `n1` floats of shared memory per warp (the cdf, later the coarse depths for the merge).  That is what lets the same
// code run (a) in the stand-alone compositing kernel (composite.cu) and (b) inside the SpaceNet tensor-core kernel's spare
// warps (mlp_tc.cu), where a tile of 128 points = whole rays and the coarse rgb / sigma never leave the SM.
//
// Arithmetic is written with explicit round-to-nearest intrinsics (no FMA contraction), so both translation units -- one
// compiled with -fmad=false, one without -- produce the same bits, and every product / sum rounds like the separate ATen
// ops of the reference.  Scans use warp shuffles (tree order): results agree with torch.cumprod / cumsum to a few ulp.
#pragma once
#include <math_constants.h>
#include <stdint.h>

namespace stnerf {
namespace rs {

constexpr unsigned FULLMASK = 0xffffffffu;

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = __fadd_rn(v, __shfl_xor_sync(FULLMASK, v, d));
  return v;
}
__device__ __forceinline__ float wscan_mul(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float n = __shfl_up_sync(FULLMASK, v, d);
    if (lane >= d) v = __fmul_rn(v, n);
  }
  return v;
}
__device__ __forceinline__ float wscan_add(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float n = __shfl_up_sync(FULLMASK, v, d);
    if (lane >= d) v = __fadd_rn(v, n);
  }
  return v;
}

// first index with a[idx] >= key / > key in an ascending array (torch.searchsorted, right=False / True)
__device__ __forceinline__ int lower_bound_s(const float* a, int n, float key) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
  return lo;
}
__device__ __forceinline__ int upper_bound_s(const float* a, int n, float key) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] <= key) lo = mid + 1; else hi = mid; }
  return lo;
}

// One image pixel (rgb, depth, acc) of ray `rg`: plane layout rgb (N,3) | depth (N) | acc (N), or 5 interleaved floats.
__device__ __forceinline__ void write_pixel(float* img, long long rg, long long n_total, bool pixels, const float o5[5], int lane) {
  if (img == nullptr || lane >= 5) return;
  const float v = lane == 0 ? o5[0] : lane == 1 ? o5[1] : lane == 2 ? o5[2] : lane == 3 ? o5[3] : o5[4];
  if (pixels) img[rg * 5 + lane] = v;
  else if (lane < 3) img[rg * 3 + lane] = v;
  else img[(long long)lane * n_total + rg] = v;
}

// value of striped element `idx` (lane idx % 32, slot idx / 32) of a register array; every lane must call it
template <int N>
__device__ __forceinline__ float gather(const float (&v)[N], int idx) {
  float out = 0.f;
#pragma unroll
  for (int s = 0; s < N; ++s) {
    const float x = __shfl_sync(FULLMASK, v[s], idx & 31);
    if ((idx >> 5) == s) out = x;
  }
  return out;
}

// Bitonic sort (ascending) of the 32*NR striped elements of a warp: element e = slot*32 + lane.
template <int NR>
__device__ __forceinline__ void bitonic_regs(float (&v)[NR], int lane) {
#pragma unroll
  for (int k = 2; k <= 32 * NR; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= 32) {                       // partner in another slot of the same lane
        const int js = j >> 5, ks = k >> 5;
#pragma unroll
        for (int s = 0; s < NR; ++s) {
          if ((s & js) == 0) {
            const int p = s | js;
            const bool up = (ks >= NR) ? true : ((s & ks) == 0);
            const float a = v[s], b = v[p];
            const float lo = fminf(a, b), hi = fmaxf(a, b);
            v[s] = up ? lo : hi;
            v[p] = up ? hi : lo;
          }
        }
      } else {                             // partner in another lane, same slot
#pragma unroll
        for (int s = 0; s < NR; ++s) {
          const float o = __shfl_xor_sync(FULLMASK, v[s], j);
          const bool up = (k >= 32) ? (k >= 32 * NR ? true : ((s & (k >> 5)) == 0)) : ((lane & k) == 0);
          const bool lower = (lane & j) == 0;
          v[s] = (lower == up) ? fminf(v[s], o) : fmaxf(v[s], o);
        }
      }
    }
  }
}

// What one warp produces for one (ray, layer).
struct LayerOut {
  float pix[5];        // colour (3), depth, accumulated opacity of the per-layer coarse image
};

// t[s], sg[s]: depth and (already masked) density of sample s*32+lane (any value where s*32+lane >= n1).
// rgb_at(s): sigmoid colour of that sample -- only called where the weight is non-zero.
// get_u(j): uniform j of this (ray, layer).   cdf: >= n1 floats of shared memory owned by this warp.
// tf: global, n1+n2 floats: receives sort(cat(t, z)) (nullptr: no resampling, image only).
// zs / src (optional, both or neither; n1+n2 <= 256): the n2 new depths in ascending order, and for every position of `tf`
// where its depth came from -- k < n1: coarse sample k, n1 + e: new depth e.  Lets the fine pass evaluate the MotionNet on the
// new depths only and take the flow of the coarse depths from the coarse pass (same network, same points).
template <int NT, int NZ, typename RgbAt, typename GetU>
__device__ __forceinline__ void composite_resample_ray(const float (&t)[NT], const float (&sg)[NT], int n1, int n2, float boarder,
                                                       RgbAt rgb_at, GetU get_u, float* cdf, float* __restrict__ tf, int lane,
                                                       LayerOut& out, float* __restrict__ zs = nullptr,
                                                       uint8_t* __restrict__ src = nullptr) {
  // ---- gen_weight + VolumeRenderer.forward (render_layer.py:8-58) -----------------------------------------------------
  float w[NT];
  float carry = 1.0f;
  float cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f, ca = 0.f;
  bool asc = true;
#pragma unroll
  for (int s = 0; s < NT; ++s) {
    const int j = s * 32 + lane;
    const bool valid = j < n1;
    const float tj = t[s];
    float tn = __shfl_down_sync(FULLMASK, tj, 1);
    const float first_next = __shfl_sync(FULLMASK, (s + 1 < NT) ? t[(s + 1 < NT) ? s + 1 : s] : 0.f, 0);
    if (lane == 31) tn = first_next;
    float f = 1.0f, alpha = 0.0f;
    if (valid) {
      const float delta = (j == n1 - 1) ? boarder : __fsub_rn(tn, tj);                  // render_layer.py:37-40
      if (j < n1 - 1 && !(tj <= tn)) asc = false;
      const float e = expf(-__fmul_rn(fmaxf(sg[s], 0.0f), delta));                       // :11
      alpha = __fsub_rn(1.0f, e);
      f = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);                                     // :12
    }
    const float incl = wscan_mul(f, lane);
    float excl = __shfl_up_sync(FULLMASK, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float T = __fmul_rn(carry, excl);
    carry = __fmul_rn(carry, __shfl_sync(FULLMASK, incl, 31));
    w[s] = 0.f;
    if (valid) {
      const float ww = __fmul_rn(alpha, T);
      w[s] = ww;
      if (ww != 0.0f) {                    // a zero weight adds exactly +0 to every sum: its colour is neither read nor squashed
        const float3 c = rgb_at(s);
        cr = __fadd_rn(cr, __fmul_rn(c.x, ww));                                          // :45
        cg = __fadd_rn(cg, __fmul_rn(c.y, ww));
        cb = __fadd_rn(cb, __fmul_rn(c.z, ww));
        cd = __fadd_rn(cd, __fmul_rn(ww, tj));                                           // :46
        ca = __fadd_rn(ca, ww);                                                          // :47
      }
    }
  }
  out.pix[0] = wsum(cr); out.pix[1] = wsum(cg); out.pix[2] = wsum(cb); out.pix[3] = wsum(cd); out.pix[4] = wsum(ca);
  if (tf == nullptr || n2 <= 0) return;
  asc = __all_sync(FULLMASK, asc);

  // ---- sample_pdf (utils/sample_pdf.py:18-63) ----------------------------------------------------------------------------
  const int nb = n1 - 2, nc = n1 - 1;                        // weights[..., 1:-1]; len(cdf) == len(bins)
  float wn[NT];                                              // wn[s] = w of sample s*32+lane+1
  float part = 0.f;
#pragma unroll
  for (int s = 0; s < NT; ++s) {
    float x = __shfl_down_sync(FULLMASK, w[s], 1);
    const float first_next = __shfl_sync(FULLMASK, (s + 1 < NT) ? w[(s + 1 < NT) ? s + 1 : s] : 0.f, 0);
    if (lane == 31) x = first_next;
    wn[s] = x;
    if (s * 32 + lane < nb) part = __fadd_rn(part, __fadd_rn(x, 1e-5f));                 // :21
  }
  const float tot = wsum(part);
  float acc = 0.f;
  if (lane == 0) cdf[0] = 0.0f;                                                          // :24
#pragma unroll
  for (int s = 0; s < NT; ++s) {
    const int m = s * 32 + lane;
    const float pdf = (m < nb) ? __fdiv_rn(__fadd_rn(wn[s], 1e-5f), tot) : 0.0f;         // :22
    const float incl = wscan_add(pdf, lane);
    if (m < nb) cdf[m + 1] = __fadd_rn(acc, incl);                                       // :23
    acc = __fadd_rn(acc, __shfl_sync(FULLMASK, incl, 31));
  }
  float bins[NT];                                                                        // :20
#pragma unroll
  for (int s = 0; s < NT; ++s) {
    float tn = __shfl_down_sync(FULLMASK, t[s], 1);
    const float first_next = __shfl_sync(FULLMASK, (s + 1 < NT) ? t[(s + 1 < NT) ? s + 1 : s] : 0.f, 0);
    if (lane == 31) tn = first_next;
    bins[s] = __fmul_rn(0.5f, __fadd_rn(tn, t[s]));
  }
  __syncwarp();
  float z[NZ];
#pragma unroll
  for (int q = 0; q < NZ; ++q) {
    const int j = q * 32 + lane;
    const float uu = (j < n2) ? get_u(j) : 0.f;
    const int lo = upper_bound_s(cdf, nc, uu);                                           // :47
    const int below = max(lo - 1, 0);                                                    // :48
    const int above = min(lo, nc - 1);                                                   // :49
    const float cbv = cdf[below], cav = cdf[above];
    const float bb = gather<NT>(bins, below), ba = gather<NT>(bins, above);
    float den = __fsub_rn(cav, cbv);
    if (den < 1e-5f) den = 1.0f;                                                         // :59
    const float tt = __fdiv_rn(__fsub_rn(uu, cbv), den);
    z[q] = (j < n2) ? __fadd_rn(bb, __fmul_rn(tt, __fsub_rn(ba, bb))) : CUDART_INF_F;    // :61
  }
  __syncwarp();

  // ---- sort(cat(t, z)) (layered_rfrender.py:462) ---------------------------------------------------------------------------
  const int S2 = n1 + n2;
  if (asc) {
    // sort the n2 new depths, then merge with the ascending coarse depths by rank:
    //   position of z_e = e + #{k : t_k <= z_e};  the coarse depths fill the remaining positions in order
    bitonic_regs<NZ>(z, lane);
#pragma unroll
    for (int s = 0; s < NT; ++s)
      if (s * 32 + lane < n1) cdf[s * 32 + lane] = t[s];        // the scratch now holds the coarse depths
    __syncwarp();
    constexpr int NW = NT + NZ;                                  // 32-bit words covering the n1 + n2 output positions
    unsigned occ[NW];
#pragma unroll
    for (int wd = 0; wd < NW; ++wd) occ[wd] = 0u;
#pragma unroll
    for (int q = 0; q < NZ; ++q) {
      const int e = q * 32 + lane;
      if (e < n2) {
        const float key = z[q];
        const int pos = e + upper_bound_s(cdf, n1, key);
        tf[pos] = key;
        if (zs != nullptr) { zs[e] = key; src[pos] = (uint8_t)(n1 + e); }
#pragma unroll
        for (int wd = 0; wd < NW; ++wd)
          if ((pos >> 5) == wd) occ[wd] |= 1u << (pos & 31);
      }
    }
#pragma unroll
    for (int wd = 0; wd < NW; ++wd) {
      occ[wd] = __reduce_or_sync(FULLMASK, occ[wd]);
      const int base = wd * 32;                                  // positions >= S2 do not exist: mark them taken
      if (base + 32 > S2) occ[wd] |= (S2 <= base) ? 0xffffffffu : (0xffffffffu << (S2 - base));
    }
#pragma unroll
    for (int s = 0; s < NT; ++s) {
      int k = s * 32 + lane;
      if (k < n1) {
        int pos = -1;
#pragma unroll
        for (int wd = 0; wd < NW; ++wd) {
          if (pos < 0) {
            const unsigned freeb = ~occ[wd];
            const int nfree = __popc(freeb);
            if (k < nfree) pos = wd * 32 + (int)__fns(freeb, 0, k + 1);
            else k -= nfree;
          }
        }
        tf[pos] = t[s];
        if (src != nullptr) src[pos] = (uint8_t)(s * 32 + lane);
      }
    }
  } else {
    // a list that is not ascending (degenerate boxes, NaNs): full sort of the concatenation, like the reference
    constexpr int NR0 = NT + NZ;
    constexpr int NR = NR0 <= 1 ? 1 : NR0 <= 2 ? 2 : NR0 <= 4 ? 4 : NR0 <= 8 ? 8 : 16;
    float v[NR];
#pragma unroll
    for (int s = 0; s < NR; ++s) v[s] = CUDART_INF_F;
    // cat(t, z) packed densely through the scratch is not needed: padding (+inf) may sit anywhere before the sort
#pragma unroll
    for (int s = 0; s < NT; ++s) v[s] = (s * 32 + lane < n1) ? t[s] : CUDART_INF_F;
#pragma unroll
    for (int q = 0; q < NZ; ++q) v[NT + q] = z[q];
    bitonic_regs<NR>(v, lane);
#pragma unroll
    for (int s = 0; s < NR; ++s)
      if (s * 32 + lane < S2) tf[s * 32 + lane] = v[s];
    // no source map for such a ray (it cannot arise for a performer box: its depths ascend unless a coordinate is NaN); keep the
    // consumers inside their buffers
    if (zs != nullptr) {
#pragma unroll
      for (int q = 0; q < NZ; ++q)
        if (q * 32 + lane < n2) zs[q * 32 + lane] = z[q];
      for (int k = lane; k < S2; k += 32) src[k] = (uint8_t)min(k, n1 + n2 - 1);
    }
  }
  __syncwarp();
}

}  // namespace rs
}  // namespace stnerf
