// What the two training GEMMs share: the fp32 SIMT GEMM of mlp_train.cu and the 3xTF32 warpgroup-MMA GEMM of
// mlp_train_tc.cu run the same three roles (forward, input delta, weight-gradient partials) with the same epilogue functors.
#pragma once
#include "common.cuh"

namespace stnerf {

namespace {
// A view of a matrix: element (r, c) at p[r*sr + c*sc]
struct Mat {
  const float* p;
  long long sr, sc;
  __device__ __forceinline__ float at(long long r, long long c) const { return p[r * sr + c * sc]; }
};

struct ZeroInit {
  __device__ __forceinline__ float operator()(int) const { return 0.f; }
};
struct BiasInit {
  const float* b;
  __device__ __forceinline__ float operator()(int m) const { return __ldg(b + m); }
};

// forward: output (m, n) -> p[m*sm + n*sn], optionally ReLU'd
struct Store {
  float* p;
  long long sm, sn;
  int relu;
  __device__ __forceinline__ void operator()(int m, long long n, float v) const { p[m * sm + n * sn] = relu ? fmaxf(v, 0.f) : v; }
};

// delta of a layer's input.  Rows m < split are a ReLU output h (saved, pitch P): out = (v [+ ws[m] ds[n]]) where h > 0,
// else 0.  Rows m >= split belong to PE(pos), which has no ReLU: written to (acc = 0) or added to (acc = 1) enc.
struct DeltaEpi {
  float* out;
  const float* h;
  long long P;
  const float* ws;
  const float* ds;
  int split;
  float* enc;
  int acc;
  __device__ __forceinline__ void operator()(int m, long long n, float v) const {
    if (m < split) {
      if (ws) v = fmaf(__ldg(ws + m), ds[n], v);
      out[m * P + n] = h[m * P + n] > 0.f ? v : 0.f;
    } else {
      float* e = enc + (m - split) * P + n;
      *e = acc ? *e + v : v;
    }
  }
};

// weight gradient: the partial tile of point chunk blockIdx.z
struct PartialStore {
  float* part;
  int N;
  long long MN;
  __device__ __forceinline__ void operator()(int m, long long n, float v) const {
    part[blockIdx.z * MN + (long long)m * N + n] = v;
  }
};
}  // namespace

// mlp_train_tc.cu: the three roles on wgmma with 3xTF32 products (STNERF_TRAIN_TC_3XTF32).  Feature-major operands of pitch P,
// nn.Linear weights W (M_out x k, row-major).
//   forward  out(M x P)        = relu(W . in + b), in = k rows
//   delta    DeltaEpi(W^T . d), W of nout rows and kin columns; rows 0..M-1 of W^T (M <= kin)
//   weights  part[z](M x N)    = d . h^T over points [z*chunk, (z+1)*chunk), for the chunk reduction of mlp_train.cu
int tc_train_forward(const float* W, int K, const float* bias, const float* in, int M, long long P, float* out, cudaStream_t st);
int tc_train_delta(const float* W, int kin, int nout, const float* d_out, int M, long long P, float* out, const float* h,
                   const float* ws, const float* ds, int split, float* enc, int acc, cudaStream_t st);
int tc_train_wgrad(const float* d, const float* h, int M, int N, long long P, long long chunk, float* part, cudaStream_t st);

}  // namespace stnerf
