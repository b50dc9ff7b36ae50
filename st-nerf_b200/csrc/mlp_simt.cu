// fp32 CUDA-core (FFMA) evaluation of SpaceNet and MotionNet: precision mode STNERF_PREC_FP32_SIMT.
//
// This is the bit-closest mode (plain fp32 products, fp32 accumulation) and the on-device cross-check for the
// tensor-core kernels in mlp_tc.cu.  One persistent CTA per SM walks tiles of 64 points; activations live in
// shared memory feature-major ([feature][point], padded) so the A operand of every layer is a broadcast
// LDS.128 and the weights ([k][n], n contiguous) stream through L1 with fully coalesced 128 B rows.
//
// Restates modeling/spacenet.py:101-160, modeling/motion_net.py:34-71, utils/dimension_kernel.py:24-33 and the
// point construction + inverse edit of modeling/layered_rfrender.py:293-303 / :465-475.
#include "common.cuh"

namespace stnerf {

namespace {
constexpr int BM = 64;         // points per tile
constexpr int BMP = 68;        // padded row pitch (floats): 16B-aligned rows, conflict-free 128-bit column stores
constexpr int NT = 256;        // threads per CTA
constexpr int P_ROWS = 96;     // encoding buffer rows (>= 84 for MotionNet)
constexpr int SMEM_FLOATS = (HID + HID + P_ROWS) * BMP + 16 * BM;
}  // namespace

size_t simt_smem_bytes() { return (size_t)SMEM_FLOATS * sizeof(float); }

// out[n][row] = act(bias[n] + sum_k in[k][row] * Wt[k][n])   for a 64-row tile.
// warp w owns rows 8w..8w+7, lane owns columns lane + 32 j.
template <int NOUT>
__device__ __forceinline__ void dense_layer(const float* __restrict__ in1, int K1, const float* __restrict__ in2, int K2,
                                            const float* __restrict__ Wt, const float* __restrict__ bias,
                                            float* __restrict__ out, bool relu) {
  constexpr int NJ = NOUT / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[8][NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const float b = __ldg(bias + lane + 32 * j);
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r][j] = b;
  }
  const float* w = Wt + lane;
  for (int seg = 0; seg < 2; ++seg) {
    const float* in = seg == 0 ? in1 : in2;
    const int K = seg == 0 ? K1 : K2;
    if (K == 0) continue;
    const float* a = in + 8 * warp;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(a + k * BMP);
      const float4 a1 = *reinterpret_cast<const float4*>(a + k * BMP + 4);
      float wv[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) wv[j] = __ldg(w + 32 * j);
      w += NOUT;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        acc[0][j] = fmaf(a0.x, wv[j], acc[0][j]);
        acc[1][j] = fmaf(a0.y, wv[j], acc[1][j]);
        acc[2][j] = fmaf(a0.z, wv[j], acc[2][j]);
        acc[3][j] = fmaf(a0.w, wv[j], acc[3][j]);
        acc[4][j] = fmaf(a1.x, wv[j], acc[4][j]);
        acc[5][j] = fmaf(a1.y, wv[j], acc[5][j]);
        acc[6][j] = fmaf(a1.z, wv[j], acc[6][j]);
        acc[7][j] = fmaf(a1.w, wv[j], acc[7][j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    float4 v0, v1;
    v0.x = acc[0][j]; v0.y = acc[1][j]; v0.z = acc[2][j]; v0.w = acc[3][j];
    v1.x = acc[4][j]; v1.y = acc[5][j]; v1.z = acc[6][j]; v1.w = acc[7][j];
    if (relu) {
      v0.x = fmaxf(v0.x, 0.f); v0.y = fmaxf(v0.y, 0.f); v0.z = fmaxf(v0.z, 0.f); v0.w = fmaxf(v0.w, 0.f);
      v1.x = fmaxf(v1.x, 0.f); v1.y = fmaxf(v1.y, 0.f); v1.z = fmaxf(v1.z, 0.f); v1.w = fmaxf(v1.w, 0.f);
    }
    float* o = out + (lane + 32 * j) * BMP + 8 * warp;
    *reinterpret_cast<float4*>(o) = v0;
    *reinterpret_cast<float4*>(o + 4) = v1;
  }
}

// Per-tile point set-up shared by both nets.  meta rows: 0-2 xyz, 3-5 dir, 6 time, 7 valid, 9-11 rgb, 12 sigma,
// 14-15 output index (int64)
struct TilePoint {
  float x, y, z, dx, dy, dz, tm;
  long long out_index;   // raw-buffer sample index (ray*S + k) or p
  bool valid;
};

__device__ __forceinline__ TilePoint fetch_point(const PointSrc& s, long long p, long long n_points) {
  TilePoint q;
  q.valid = p < n_points;
  q.x = q.y = q.z = q.dx = q.dy = q.dz = q.tm = 0.f;
  q.out_index = p;
  if (!q.valid) return q;
  if (s.mode == SRC_EXPLICIT) {
    const float* pp = s.pos + p * s.pos_stride;
    q.x = pp[0]; q.y = pp[1]; q.z = pp[2];
    if (s.dirs) { q.dx = s.dirs[3 * p]; q.dy = s.dirs[3 * p + 1]; q.dz = s.dirs[3 * p + 2]; }
    if (s.times) q.tm = s.times[p * s.time_stride];
    return q;
  }
  const long long slot = p / s.S;
  const int k = (int)(p - slot * s.S);
  const long long ray = s.hit ? (long long)s.hit[slot] : slot;
  const float* rp = s.rays + ray * s.ray_stride;
  q.dx = rp[3]; q.dy = rp[4]; q.dz = rp[5];
  q.tm = rp[6 + s.layer];
  q.out_index = ray * s.S + k;
  if (s.mode == SRC_XYZ) {
    q.x = s.pos[3 * p]; q.y = s.pos[3 * p + 1]; q.z = s.pos[3 * p + 2];
    return q;
  }
  const float tt = s.t[ray * s.S + k];
  float v[3];
  march_point(s, rp, tt, q.dx, q.dy, q.dz, v);      // common.cuh (also the training point assembly, train_march.cu)
  q.x = v[0]; q.y = v[1]; q.z = v[2];
  return q;
}

// ---------------------------------------------------------------------------------------------------------
// SpaceNet
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT, 1)
spacenet_simt_kernel(PointSrc src, SpaceNetW W, float* __restrict__ raw, float* __restrict__ rgb_out,
                     float* __restrict__ sigma_out) {
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem;
  float* bufB = bufA + HID * BMP;
  float* bufP = bufB + HID * BMP;
  float* meta = bufP + P_ROWS * BMP;          // [16][BM]
  const int tid = threadIdx.x;
  const int pt = tid & (BM - 1), part = tid >> 6;
  const long long n_points = src_num_points(src);
  const long long n_tiles = (n_points + BM - 1) / BM;

  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    __syncthreads();
    if (tid < BM) {
      const TilePoint q = fetch_point(src, tile * BM + tid, n_points);
      meta[0 * BM + tid] = q.x; meta[1 * BM + tid] = q.y; meta[2 * BM + tid] = q.z;
      meta[3 * BM + tid] = q.dx; meta[4 * BM + tid] = q.dy; meta[5 * BM + tid] = q.dz;
      meta[6 * BM + tid] = q.tm;
      meta[7 * BM + tid] = q.valid ? 1.f : 0.f;
      reinterpret_cast<long long*>(meta + 14 * BM)[tid] = q.out_index;   // rows 14-15
    }
    __syncthreads();
    // positional encoding of the position, 63 rows (utils/dimension_kernel.py:24-33)
    if (part == 0) {
#pragma unroll
      for (int d = 0; d < 3; ++d) bufP[d * BMP + pt] = meta[d * BM + pt];
    }
    for (int q = part; q < 30; q += 4) {
      const int f = q / 3, d = q - 3 * f;
      float s, c;
      sincosf(meta[d * BM + pt] * (float)(1 << f), &s, &c);
      bufP[(3 + 6 * f + d) * BMP + pt] = s;
      bufP[(6 + 6 * f + d) * BMP + pt] = c;
    }
    __syncthreads();
    dense_layer<HID>(bufP, PE_POS, nullptr, 0, W.w[0], W.b[0], bufA, true);  __syncthreads();
    dense_layer<HID>(bufA, HID, nullptr, 0, W.w[1], W.b[1], bufB, true);     __syncthreads();
    dense_layer<HID>(bufB, HID, nullptr, 0, W.w[2], W.b[2], bufA, true);     __syncthreads();
    dense_layer<HID>(bufA, HID, nullptr, 0, W.w[3], W.b[3], bufB, true);     __syncthreads();
    dense_layer<HID>(bufB, HID, bufP, PE_POS, W.w[4], W.b[4], bufA, true);   __syncthreads();   // skip concat :137
    dense_layer<HID>(bufA, HID, nullptr, 0, W.w[5], W.b[5], bufB, true);     __syncthreads();
    dense_layer<HID>(bufB, HID, nullptr, 0, W.w[6], W.b[6], bufA, true);     __syncthreads();
    // x = bufA.  density head (:139) + relu'd direction/time encodings for the rgb head (:141-149, :82)
    if (tid < BM) {
      float s = W.b_sigma;
      for (int k = 0; k < HID; ++k) s = fmaf(bufA[k * BMP + tid], __ldg(W.w_sigma + k), s);
      meta[12 * BM + tid] = s;
    }
    if (part == 0) {
#pragma unroll
      for (int d = 0; d < 3; ++d) bufP[d * BMP + pt] = fmaxf(meta[(3 + d) * BM + pt], 0.f);
      if (W.use_time) bufP[PE_DIR * BMP + pt] = fmaxf(meta[6 * BM + pt], 0.f);
    }
    for (int q = part; q < 12 + (W.use_time ? 10 : 0); q += 4) {
      float s, c;
      if (q < 12) {
        const int f = q / 3, d = q - 3 * f;
        sincosf(meta[(3 + d) * BM + pt] * (float)(1 << f), &s, &c);
        bufP[(3 + 6 * f + d) * BMP + pt] = fmaxf(s, 0.f);
        bufP[(6 + 6 * f + d) * BMP + pt] = fmaxf(c, 0.f);
      } else {
        const int f = q - 12;
        sincosf(meta[6 * BM + pt] * (float)(1 << f), &s, &c);
        bufP[(PE_DIR + 1 + 2 * f) * BMP + pt] = fmaxf(s, 0.f);
        bufP[(PE_DIR + 2 + 2 * f) * BMP + pt] = fmaxf(c, 0.f);
      }
    }
    __syncthreads();
    dense_layer<HEAD>(bufA, HID, bufP, PE_DIR + (W.use_time ? PE_TIME : 0), W.w_rgbh, W.b_rgbh, bufB, true);
    __syncthreads();
    if (tid < 3 * BM) {
      const float* wr = W.w_rgbo + part * HEAD;
      float v = W.b_rgbo[part];
      for (int k = 0; k < HEAD; ++k) v = fmaf(bufB[k * BMP + pt], __ldg(wr + k), v);
      meta[(9 + part) * BM + pt] = v;
    }
    __syncthreads();
    if (tid < BM && meta[7 * BM + tid] != 0.f) {
      const long long oi = reinterpret_cast<const long long*>(meta + 14 * BM)[tid];
      const float r = meta[9 * BM + tid], g = meta[10 * BM + tid], b = meta[11 * BM + tid], s = meta[12 * BM + tid];
      if (raw) reinterpret_cast<float4*>(raw)[oi] = make_float4(r, g, b, s);
      if (rgb_out) { rgb_out[3 * oi] = r; rgb_out[3 * oi + 1] = g; rgb_out[3 * oi + 2] = b; }
      if (sigma_out) sigma_out[oi] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// MotionNet
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT, 1)
motionnet_simt_kernel(PointSrc src, MotionNetW W, const int* __restrict__ lerp_flag, int lerp_force,
                      float* __restrict__ xyz_out, float* __restrict__ flow_out) {
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem;
  float* bufB = bufA + HID * BMP;
  float* bufP = bufB + HID * BMP;
  float* meta = bufP + P_ROWS * BMP;
  const int tid = threadIdx.x;
  const int pt = tid & (BM - 1), part = tid >> 6;
  const long long n_points = src_num_points(src);
  const long long n_tiles = (n_points + BM - 1) / BM;
  const bool lerp = lerp_force >= 0 ? (lerp_force != 0) : (lerp_flag && *lerp_flag != 0);

  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    __syncthreads();
    if (tid < BM) {
      const TilePoint q = fetch_point(src, tile * BM + tid, n_points);
      meta[0 * BM + tid] = q.x; meta[1 * BM + tid] = q.y; meta[2 * BM + tid] = q.z;
      meta[3 * BM + tid] = q.tm;
      meta[7 * BM + tid] = q.valid ? 1.f : 0.f;
    }
    __syncthreads();
    // PE([x,y,z,t], L=10): rows [0..3] raw, 4+8f+d sin, 8+8f+d cos  (modeling/motion_net.py:14,48-65)
    {
      const float tm = meta[3 * BM + pt];
      const float lo = floorf(tm), wgt = tm - lo, omw = 1.0f - wgt;
      for (int q = part; q < 44; q += 4) {          // q = 0..3 raw columns, then 40 (freq, dim) pairs
        if (q < 4) {
          float v;
          if (!lerp) v = meta[q * BM + pt];
          else {
            const float a = (q < 3) ? meta[q * BM + pt] : lo, b = (q < 3) ? meta[q * BM + pt] : lo + 1.0f;
            v = __fadd_rn(__fmul_rn(omw, a), __fmul_rn(wgt, b));                       // :63
          }
          bufP[q * BMP + pt] = v;
        } else {
          const int f = (q - 4) >> 2, d = (q - 4) & 3;
          const float fr = (float)(1 << f);
          float s, c;
          if (!lerp) {
            sincosf(meta[d * BM + pt] * fr, &s, &c);
          } else {
            const float a = (d < 3) ? meta[d * BM + pt] : lo, b = (d < 3) ? a : lo + 1.0f;
            float s0, c0, s1, c1;
            sincosf(a * fr, &s0, &c0);
            sincosf(b * fr, &s1, &c1);
            s = __fadd_rn(__fmul_rn(omw, s0), __fmul_rn(wgt, s1));
            c = __fadd_rn(__fmul_rn(omw, c0), __fmul_rn(wgt, c1));
          }
          bufP[(4 + 8 * f + d) * BMP + pt] = s;
          bufP[(8 + 8 * f + d) * BMP + pt] = c;
        }
      }
    }
    __syncthreads();
    dense_layer<HEAD>(bufP, PE_MOTION, nullptr, 0, W.w[0], W.b[0], bufA, true);  __syncthreads();
    dense_layer<HEAD>(bufA, HEAD, nullptr, 0, W.w[1], W.b[1], bufB, true);       __syncthreads();
    dense_layer<HEAD>(bufB, HEAD, nullptr, 0, W.w[2], W.b[2], bufA, true);       __syncthreads();
    dense_layer<HEAD>(bufA, HEAD, nullptr, 0, W.w[3], W.b[3], bufB, true);       __syncthreads();
    dense_layer<HEAD>(bufB, HEAD, nullptr, 0, W.w[4], W.b[4], bufA, true);       __syncthreads();
    if (tid < 3 * BM && meta[7 * BM + pt] != 0.f) {
      const float* wr = W.w_out + part * HEAD;
      float v = W.b_out[part];
      for (int k = 0; k < HEAD; ++k) v = fmaf(bufA[k * BMP + pt], __ldg(wr + k), v);
      const long long p = tile * BM + pt;
      if (flow_out) flow_out[3 * p + part] = v;
      if (xyz_out) xyz_out[3 * p + part] = __fadd_rn(meta[part * BM + pt], v);         // layered_rfrender.py:356 / :510
    }
  }
}

int launch_spacenet_simt(const PointSrc& src, const SpaceNetW& w, float* raw, long long /*raw_slot_stride*/,
                         float* rgb_out, float* sigma_out, int num_sms, cudaStream_t st) {
  // set on every launch: the attribute is per device, and one process may drive several (cost: microseconds)
  STNERF_CUDA(cudaFuncSetAttribute(spacenet_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)simt_smem_bytes()));
  spacenet_simt_kernel<<<num_sms, NT, simt_smem_bytes(), st>>>(src, w, raw, rgb_out, sigma_out);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

int launch_motionnet_simt(const PointSrc& src, const MotionNetW& w, const int* lerp_flag_dev, int lerp_force,
                          float* xyz_out, float* flow_out, int num_sms, cudaStream_t st) {
  STNERF_CUDA(cudaFuncSetAttribute(motionnet_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)simt_smem_bytes()));
  motionnet_simt_kernel<<<num_sms, NT, simt_smem_bytes(), st>>>(src, w, lerp_flag_dev, lerp_force, xyz_out, flow_out);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

}  // namespace stnerf
