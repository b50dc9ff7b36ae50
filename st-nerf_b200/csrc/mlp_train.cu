// fp32 CUDA-core training path of SpaceNet and MotionNet: a forward that keeps what the backward needs, and the backward
// (input deltas, weight and bias gradients, d_pos).
//
// Restates modeling/spacenet.py:101-160, modeling/motion_net.py:34-71 and utils/dimension_kernel.py:24-33, and
// differentiates them the way torch.autograd differentiates the reference: ReLU passes the gradient where its OUTPUT is > 0,
// directions, times and MotionNet's xyzt get no gradient (modeling/layered_rfrender.py:272,314-315 detach them).
//
// Every layer is one launch of a single smem-tiled fp32 SIMT GEMM (gemm_kernel) with an epilogue functor.  Activations are
// kept feature-major in the caller's `saved` buffer: row r of a batch of P points is saved[r*P .. r*P + P-1].
//   forward   out(n_out x P) = W(n_out x k) . in(k x P)          + bias, ReLU           ("NN")
//   delta     d_in(k x P)    = W^T . d_out(n_out x P), masked by in > 0                  ("NT" in the points-major view)
//   weights   dW(n_out x k)  = d_out . in^T, summed over points                          ("TN")
// Weight and bias gradients are sums over the batch.  They are formed deterministically: the points are cut into chunks that
// depend on P only, every CTA of a chunk writes its partial tile, and a second pass adds the partials in chunk order (weights)
// or in a fixed tree (biases, rowsum_chunks_kernel).  There are no floating-point atomics, so two identical calls give
// identical bits.
//
// The forward GEMM starts every output at its bias and adds the k terms in ascending order with one fmaf each, exactly like
// dense_layer in mlp_simt.cu, and the encodings use the same sincosf arguments: the training forward is bit-identical to
// STNERF_PREC_FP32_SIMT.
//
// STNERF_TRAIN_TC_3XTF32 routes the GEMMs of every layer with 128 or more outputs to the 3xTF32 tensor-core GEMM of
// mlp_train_tc.cu (same roles, epilogue functors and point chunks; mlp_train.cuh); the 1- and 3-wide heads, the encodings, d_pos,
// the bias row sums and the chunk reduction run here in both precisions.
//
// Weights are the stnerf_load_* blob (state_dict order, nn.Linear (out, in) row-major), read in place; the gradients come
// back as one blob in the same order.
#include "mlp_train.cuh"

namespace stnerf {

namespace {
constexpr int TB = 64;            // output tile: TB x TB
constexpr int TK = 16;            // k step
constexpr int TT = 256;           // threads: 16 x 16, each 4 x 4 outputs
constexpr int TBP = TB + 4;       // smem row pitch (floats): 16 B-aligned rows
constexpr int MAX_SPLIT = 128;    // point chunks of a weight-gradient sum
constexpr int MIN_CHUNK = 256;    // points per chunk, at least

// saved rows of a SpaceNet: h1 h2 h3 h4 PE(pos) h5 h6 h7 ENC h8, so that both concatenated inputs are contiguous rows:
// stage2.0 reads [h4; PE(pos)] (spacenet.py:137), rgb_net.1 reads [h7; ENC] with ENC = relu([PE(dir), PE(t)]) (:143-149, :82)
constexpr int S_H1 = 0, S_H4 = 3 * HID, S_PE = 4 * HID, S_H5 = S_PE + PE_POS, S_H7 = S_H5 + 2 * HID, S_ENC = S_H7 + HID;
constexpr int S_IN[7] = {S_PE, S_H1, S_H1 + HID, S_H1 + 2 * HID, S_H4, S_H5, S_H5 + HID};   // input row of trunk layer l
constexpr int S_OUT[7] = {S_H1, S_H1 + HID, S_H1 + 2 * HID, S_H4, S_H5, S_H5 + HID, S_H7};
// saved rows of a MotionNet: PE(xyzt) h1 .. h5
constexpr int M_PE = 0;
__host__ __device__ constexpr int m_h(int i) { return PE_MOTION + HEAD * (i - 1); }

int enc_rows(int use_time) { return PE_DIR + (use_time ? PE_TIME : 0); }
int s_h8(int use_time) { return S_ENC + enc_rows(use_time); }

// C(m, n) = init(m) + sum over k in chunk blockIdx.z of A(m, k) B(k, n), k ascending, one fmaf per term; epi(m, n, C).
// A_KC / B_KC: the operand is contiguous along k (else along m / n), which picks the coalesced tile-load order.
// BLOCKED: each k step of TK terms is summed on its own and then added to C, so that the rounding error of a K-term sum grows
// with TK + K / TK terms instead of K (the backward's sums); else every term goes straight into C (the forward, whose order
// is dense_layer's).
template <bool A_KC, bool B_KC, bool BLOCKED, class Init, class Epi>
__global__ void __launch_bounds__(TT) gemm_kernel(Mat A, Mat B, int M, long long N, long long K, long long kchunk, Init init,
                                                  Epi epi) {
  __shared__ __align__(16) float As[TK][TBP];
  __shared__ __align__(16) float Bs[TK][TBP];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * TB;
  const long long n0 = (long long)blockIdx.x * TB;
  const long long kb = (long long)blockIdx.z * kchunk, ke = min(K, kb + kchunk);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + 4 * ty + i;
    const float b = m < M ? init(m) : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = b;
  }
  for (long long k0 = kb; k0 < ke; k0 += TK) {
    const int kn = (int)min((long long)TK, ke - k0);
#pragma unroll
    for (int e = 0; e < TB * TK / TT; ++e) {
      const int idx = tid + e * TT;
      const int ar = A_KC ? idx / TK : idx % TB, ac = A_KC ? idx % TK : idx / TB;
      As[ac][ar] = (m0 + ar < M && ac < kn) ? A.at(m0 + ar, k0 + ac) : 0.f;
      const int bk = B_KC ? idx % TK : idx / TB, bn = B_KC ? idx / TK : idx % TB;
      Bs[bk][bn] = (n0 + bn < N && bk < kn) ? B.at(k0 + bk, n0 + bn) : 0.f;
    }
    __syncthreads();
    float sum[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) sum[i][j] = BLOCKED ? 0.f : acc[i][j];
    auto step = [&](int kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][4 * ty]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][4 * tx]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sum[i][j] = fmaf(av[i], bv[j], sum[i][j]);
    };
    if (kn == TK) {
#pragma unroll
      for (int kk = 0; kk < TK; ++kk) step(kk);
    } else {
      for (int kk = 0; kk < kn; ++kk) step(kk);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = BLOCKED ? acc[i][j] + sum[i][j] : sum[i][j];
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + 4 * ty + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long n = n0 + 4 * tx + j;
      if (m < M && n < N) epi(m, n, acc[i][j]);
    }
  }
}

template <bool A_KC, bool B_KC, bool BLOCKED = false, class Init, class Epi>
int gemm(Mat A, Mat B, int M, long long N, long long K, long long kchunk, Init init, Epi epi, cudaStream_t st) {
  if (M <= 0 || N <= 0) return STNERF_OK;
  const long long nz = K > 0 ? (K + kchunk - 1) / kchunk : 1;
  const dim3 grid((unsigned)((N + TB - 1) / TB), (unsigned)((M + TB - 1) / TB), (unsigned)nz);
  gemm_kernel<A_KC, B_KC, BLOCKED, Init, Epi><<<grid, TT, 0, st>>>(A, B, M, N, K, kchunk, init, epi);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// points per chunk of a weight-gradient sum: a function of P alone, so the summation order is too
long long grad_chunk(long long P) {
  const long long c = (P + MAX_SPLIT - 1) / MAX_SPLIT;
  return c < MIN_CHUNK ? MIN_CHUNK : (c + TK - 1) / TK * TK;
}

__global__ void reduce_partials_kernel(const float* __restrict__ part, int nz, long long MN, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= MN) return;
  float s = 0.f;
  for (int z = 0; z < nz; ++z) s += part[z * MN + i];
  out[i] = s;
}

// Bias gradients, out[m] = sum_p D(m, p), in two fixed trees: CTA (z, m) sums row m over point chunk z of grad_chunk(P) (each
// thread at most chunk / TT points in sequence, then a tree over the threads) into part[z*M + m]; then one CTA per row adds
// the chunk partials in a tree.  A single thread summing P / TT points in sequence (P = 2^20: 4096 fp32 adds) lost to
// torch's own fp32 sum by 39x at P = 1 190 007; a run is now ceil(grad_chunk(P) / TT): 33 up to P = 1 081 344, 37 there.
__global__ void __launch_bounds__(TT) rowsum_chunks_kernel(Mat D, long long P, long long chunk, float* __restrict__ part) {
  __shared__ float red[TT];
  const int z = blockIdx.x, m = blockIdx.y, tid = threadIdx.x;
  const long long pe = min(P, (z + 1) * chunk);
  float s = 0.f;
  for (long long p = z * chunk + tid; p < pe; p += TT) s += D.at(m, p);
  red[tid] = s;
  __syncthreads();
  for (int w = TT / 2; w > 0; w >>= 1) {
    if (tid < w) red[tid] += red[tid + w];
    __syncthreads();
  }
  if (tid == 0) part[(long long)z * gridDim.y + m] = red[0];
}

__global__ void __launch_bounds__(MAX_SPLIT) rowsum_tree_kernel(const float* __restrict__ part, int nz, int M,
                                                                float* __restrict__ out) {
  __shared__ float red[MAX_SPLIT];
  const int m = blockIdx.x, tid = threadIdx.x;
  red[tid] = tid < nz ? part[tid * M + m] : 0.f;
  __syncthreads();
  for (int w = MAX_SPLIT / 2; w > 0; w >>= 1) {
    if (tid < w) red[tid] += red[tid + w];
    __syncthreads();
  }
  if (tid == 0) out[m] = red[0];
}

// The wide layers (128 or more outputs) run on the 3xTF32 tensor-core GEMM in STNERF_TRAIN_TC_3XTF32; the 1- and 3-wide heads
// always run on the SIMT GEMM.
bool on_tc(int prec, int M) { return prec == STNERF_TRAIN_TC_3XTF32 && M >= HEAD; }

// dW (M x N, row-major at dw) = sum_p D(m, p) H(n, p) and db (M) = sum_p D(m, p), for H = saved rows starting at `h`
template <bool D_KC>
int weight_grad(Mat D, const float* h, int M, int N, long long P, float* dw, float* db, float* part, cudaStream_t st,
                int prec = STNERF_TRAIN_FP32) {
  const long long ch = grad_chunk(P), nz = (P + ch - 1) / ch, MN = (long long)M * N;
  int rc = (D_KC && on_tc(prec, M)) ? tc_train_wgrad(D.p, h, M, N, P, ch, part, st)
                                    : gemm<D_KC, true, true>(D, Mat{h, 1, P}, M, N, P, ch, ZeroInit{}, PartialStore{part, N, MN}, st);
  if (rc) return rc;
  reduce_partials_kernel<<<(unsigned)((MN + 255) / 256), 256, 0, st>>>(part, (int)nz, MN, dw);
  STNERF_LAUNCH_CHECK();
  // part is free again once the weight partials are reduced; nz <= MAX_SPLIT for every P (grad_chunk)
  if (nz > 0) {
    rowsum_chunks_kernel<<<dim3((unsigned)nz, (unsigned)M), TT, 0, st>>>(D, P, ch, part);
    STNERF_LAUNCH_CHECK();
  }
  rowsum_tree_kernel<<<M, MAX_SPLIT, 0, st>>>(part, (int)nz, M, db);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

// offsets of every layer's weight and bias in a stnerf_load_* blob
struct Layout {
  int n;
  int kin[10], nout[10];
  long long w[10], b[10];
};
Layout make_layout(int n, const int* kin, const int* nout) {
  Layout L;
  L.n = n;
  long long off = 0;
  for (int i = 0; i < n; ++i) {
    L.kin[i] = kin[i]; L.nout[i] = nout[i];
    L.w[i] = off; L.b[i] = off + (long long)kin[i] * nout[i];
    off = L.b[i] + nout[i];
  }
  return L;
}
Layout spacenet_layout(int use_time) {          // modeling/spacenet.py:45-86
  const int kin[10] = {PE_POS, HID, HID, HID, HID + PE_POS, HID, HID, HID, HID + enc_rows(use_time), HEAD};
  const int nout[10] = {HID, HID, HID, HID, HID, HID, HID, 1, HEAD, 3};
  return make_layout(10, kin, nout);
}
Layout motionnet_layout() {                     // modeling/motion_net.py:18-30
  const int kin[6] = {PE_MOTION, HEAD, HEAD, HEAD, HEAD, HEAD};
  const int nout[6] = {HEAD, HEAD, HEAD, HEAD, HEAD, 3};
  return make_layout(6, kin, nout);
}

// ---------------------------------------------------------------------------------------------------------
// encodings (one thread per point; the same sincosf arguments as mlp_simt.cu)
// ---------------------------------------------------------------------------------------------------------
// PE(pos) (utils/dimension_kernel.py:24-33) and ENC = relu([PE(dir), PE(t)]) (spacenet.py:128-131, 143-149, rgb_net[0] :82)
__global__ void spacenet_encode_kernel(const float* __restrict__ pos, const float* __restrict__ dirs,
                                       const float* __restrict__ times, int use_time, long long P, float* __restrict__ saved) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float* pe = saved + S_PE * P + p;
  float* enc = saved + S_ENC * P + p;
  float s, c;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float x = pos[3 * p + d], v = dirs[3 * p + d];
    pe[d * P] = x;
    for (int f = 0; f < 10; ++f) {
      sincosf(x * (float)(1 << f), &s, &c);
      pe[(3 + 6 * f + d) * P] = s;
      pe[(6 + 6 * f + d) * P] = c;
    }
    enc[d * P] = fmaxf(v, 0.f);
    for (int f = 0; f < 4; ++f) {
      sincosf(v * (float)(1 << f), &s, &c);
      enc[(3 + 6 * f + d) * P] = fmaxf(s, 0.f);
      enc[(6 + 6 * f + d) * P] = fmaxf(c, 0.f);
    }
  }
  if (use_time) {
    const float t = times[p];
    enc[PE_DIR * P] = fmaxf(t, 0.f);
    for (int f = 0; f < 10; ++f) {
      sincosf(t * (float)(1 << f), &s, &c);
      enc[(PE_DIR + 1 + 2 * f) * P] = fmaxf(s, 0.f);
      enc[(PE_DIR + 2 + 2 * f) * P] = fmaxf(c, 0.f);
    }
  }
}

// PE(x, y, z, t), or the encoding lerped between floor(t) and floor(t) + 1 (motion_net.py:48-65); rows 0-3 raw,
// 4+8f+d sin, 8+8f+d cos.  The lerp is decided for the whole batch (:53) or forced.
__global__ void motionnet_encode_kernel(const float* __restrict__ xyzt, long long P, const int* __restrict__ lerp_flag,
                                        int lerp_force, float* __restrict__ saved) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const bool lerp = lerp_force >= 0 ? (lerp_force != 0) : (lerp_flag && *lerp_flag != 0);
  float* pe = saved + M_PE * P + p;
  float x[4];
#pragma unroll
  for (int d = 0; d < 4; ++d) x[d] = xyzt[4 * p + d];
  const float lo = floorf(x[3]), wgt = x[3] - lo, omw = 1.0f - wgt;
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    if (!lerp) {
      pe[d * P] = x[d];
    } else {
      const float a = d < 3 ? x[d] : lo, b = d < 3 ? x[d] : lo + 1.0f;
      pe[d * P] = __fadd_rn(__fmul_rn(omw, a), __fmul_rn(wgt, b));                     // :63
    }
    for (int f = 0; f < 10; ++f) {
      const float fr = (float)(1 << f);
      float s, c;
      if (!lerp) {
        sincosf(x[d] * fr, &s, &c);
      } else {
        const float a = d < 3 ? x[d] : lo, b = d < 3 ? a : lo + 1.0f;
        float s0, c0, s1, c1;
        sincosf(a * fr, &s0, &c0);
        sincosf(b * fr, &s1, &c1);
        s = __fadd_rn(__fmul_rn(omw, s0), __fmul_rn(wgt, s1));
        c = __fadd_rn(__fmul_rn(omw, c0), __fmul_rn(wgt, c1));
      }
      pe[(4 + 8 * f + d) * P] = s;
      pe[(8 + 8 * f + d) * P] = c;
    }
  }
}

// d_pos = dPE/dpos . dPE: the raw term plus 2^f cos(2^f x) for sin rows and -2^f sin(2^f x) for cos rows
__global__ void spacenet_dpos_kernel(const float* __restrict__ saved, const float* __restrict__ dpe, long long P,
                                     float* __restrict__ d_pos) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float x = saved[(S_PE + d) * P + p];
    float g = dpe[d * P + p];
    for (int f = 0; f < 10; ++f) {
      const float fr = (float)(1 << f);
      float s, c;
      sincosf(x * fr, &s, &c);
      g = fmaf(fr, fmaf(c, dpe[(3 + 6 * f + d) * P + p], -s * dpe[(6 + 6 * f + d) * P + p]), g);
    }
    d_pos[3 * p + d] = g;
  }
}

unsigned pt_blocks(long long P) { return (unsigned)((P + 255) / 256); }

// forward of one hidden / output layer: out rows = act(W . in rows + b)
int fwd_layer(const float* W, const Layout& L, int l, const float* in, long long P, Store out, cudaStream_t st,
              int prec = STNERF_TRAIN_FP32) {
  if (on_tc(prec, L.nout[l]))      // every wide layer is a ReLU'd hidden layer stored feature-major
    return tc_train_forward(W + L.w[l], L.kin[l], W + L.b[l], in, L.nout[l], P, out.p, st);
  return gemm<true, false>(Mat{W + L.w[l], L.kin[l], 1}, Mat{in, P, 1}, L.nout[l], P, L.kin[l], L.kin[l],
                           BiasInit{W + L.b[l]}, out, st);
}
// delta of layer l's input rows 0..M-1 from the layer's output delta d_out (nout[l] x P, feature-major)
int delta_layer(const float* W, const Layout& L, int l, const float* d_out, int M, long long P, DeltaEpi epi, cudaStream_t st,
                int prec = STNERF_TRAIN_FP32) {
  if (on_tc(prec, L.nout[l]))
    return tc_train_delta(W + L.w[l], L.kin[l], L.nout[l], d_out, M, P, epi.out, epi.h, epi.ws, epi.ds, epi.split, epi.enc, epi.acc,
                          st);
  return gemm<false, false, true>(Mat{W + L.w[l], 1, L.kin[l]}, Mat{d_out, P, 1}, M, P, L.nout[l], L.nout[l], ZeroInit{}, epi,
                                  st);
}
}  // namespace

size_t train_saved_floats(int kind, int use_time) {
  return kind == 0 ? (size_t)(s_h8(use_time) + HEAD) : (size_t)m_h(6);
}

size_t train_scratch_bytes(int kind, int /*use_time*/, long long P) {
  const size_t part = (size_t)MAX_SPLIT * (kind == 0 ? HID * (HID + PE_POS) : HEAD * HEAD);
  const size_t rows = kind == 0 ? 2 * HID + PE_POS : 2 * HEAD;
  return (part + rows * (size_t)P) * sizeof(float);
}

int launch_spacenet_train_forward(const float* W, int use_time, const float* pos, const float* dirs, const float* times,
                                  long long P, float* rgb, float* sigma, float* saved, cudaStream_t st, int prec) {
  const Layout L = spacenet_layout(use_time);
  spacenet_encode_kernel<<<pt_blocks(P), 256, 0, st>>>(pos, dirs, times, use_time, P, saved);
  STNERF_LAUNCH_CHECK();
  int rc = 0;
  for (int l = 0; l < 7 && !rc; ++l)                                                       // stage1, stage2 :135-137
    rc = fwd_layer(W, L, l, saved + S_IN[l] * P, P, Store{saved + S_OUT[l] * P, P, 1, 1}, st, prec);
  const int h8 = s_h8(use_time);
  if (!rc) rc = fwd_layer(W, L, 7, saved + S_H7 * P, P, Store{sigma, 0, 1, 0}, st);          // density_net :139
  if (!rc) rc = fwd_layer(W, L, 8, saved + S_H7 * P, P, Store{saved + h8 * P, P, 1, 1}, st, prec); // rgb_net.1 :143-149
  if (!rc) rc = fwd_layer(W, L, 9, saved + h8 * P, P, Store{rgb, 1, 3, 0}, st);             // rgb_net.3
  return rc;
}

int launch_spacenet_backward(const float* W, int use_time, long long P, const float* saved, const float* d_rgb,
                             const float* d_sigma, float* dW, float* d_pos, void* scratch, cudaStream_t st, int prec) {
  const Layout L = spacenet_layout(use_time);
  float* D0 = (float*)scratch;
  float* D1 = D0 + HID * P;
  float* dpe = D1 + HID * P;
  float* part = dpe + PE_POS * P;
  const float* h8 = saved + s_h8(use_time) * P;
  const float* h7 = saved + S_H7 * P;
  int rc;
  // rgb_net.3: weights, then delta of h8
  if ((rc = weight_grad<false>(Mat{d_rgb, 1, 3}, h8, 3, HEAD, P, dW + L.w[9], dW + L.b[9], part, st))) return rc;
  if ((rc = gemm<false, true>(Mat{W + L.w[9], 1, HEAD}, Mat{d_rgb, 1, 3}, HEAD, P, 3, 3, ZeroInit{},
                              DeltaEpi{D1, h8, P, nullptr, nullptr, HEAD, nullptr, 0}, st))) return rc;
  // density_net.0 and rgb_net.1: weights, then delta of h7 from both heads (the direction / time rows get none)
  if ((rc = weight_grad<true>(Mat{d_sigma, 0, 1}, h7, 1, HID, P, dW + L.w[7], dW + L.b[7], part, st))) return rc;
  if ((rc = weight_grad<true>(Mat{D1, P, 1}, h7, HEAD, L.kin[8], P, dW + L.w[8], dW + L.b[8], part, st, prec))) return rc;
  if ((rc = delta_layer(W, L, 8, D1, HID, P, DeltaEpi{D0, h7, P, W + L.w[7], d_sigma, HID, nullptr, 0}, st, prec))) return rc;
  // trunk, top down.  stage2.0's input delta splits at the skip concatenation (:137): rows 0-255 reach h4, rows 256-318
  // reach PE(pos), as does stage1.0's.
  float *cur = D0, *nxt = D1;
  for (int l = 6; l >= 0; --l) {
    if ((rc = weight_grad<true>(Mat{cur, P, 1}, saved + S_IN[l] * P, HID, L.kin[l], P, dW + L.w[l], dW + L.b[l], part, st,
                                prec)))
      return rc;
    if (l > 0) {
      const int M = (l == 4 && d_pos) ? HID + PE_POS : HID;
      if ((rc = delta_layer(W, L, l, cur, M, P, DeltaEpi{nxt, saved + S_IN[l] * P, P, nullptr, nullptr, HID, dpe, 0}, st,
                            prec)))
        return rc;
      float* t = cur; cur = nxt; nxt = t;
    } else if (d_pos) {
      if ((rc = delta_layer(W, L, 0, cur, PE_POS, P, DeltaEpi{nullptr, nullptr, P, nullptr, nullptr, 0, dpe, 1}, st, prec)))
        return rc;
    }
  }
  if (d_pos) {
    spacenet_dpos_kernel<<<pt_blocks(P), 256, 0, st>>>(saved, dpe, P, d_pos);
    STNERF_LAUNCH_CHECK();
  }
  return STNERF_OK;
}

int launch_motionnet_train_forward(const float* W, const float* xyzt, long long P, const int* lerp_flag, int lerp_force,
                                   float* flow, float* saved, cudaStream_t st, int prec) {
  const Layout L = motionnet_layout();
  motionnet_encode_kernel<<<pt_blocks(P), 256, 0, st>>>(xyzt, P, lerp_flag, lerp_force, saved);
  STNERF_LAUNCH_CHECK();
  int rc = 0;
  for (int l = 0; l < 5 && !rc; ++l)                                                        // motion_net.0 .. .8
    rc = fwd_layer(W, L, l, saved + (l == 0 ? M_PE : m_h(l)) * P, P, Store{saved + m_h(l + 1) * P, P, 1, 1}, st, prec);
  if (!rc) rc = fwd_layer(W, L, 5, saved + m_h(5) * P, P, Store{flow, 1, 3, 0}, st);         // motion_net.10
  return rc;
}

int launch_motionnet_backward(const float* W, long long P, const float* saved, const float* d_flow, float* dW, void* scratch,
                              cudaStream_t st, int prec) {
  const Layout L = motionnet_layout();
  float* D0 = (float*)scratch;
  float* D1 = D0 + HEAD * P;
  float* part = D1 + HEAD * P;
  const float* h5 = saved + m_h(5) * P;
  int rc;
  if ((rc = weight_grad<false>(Mat{d_flow, 1, 3}, h5, 3, HEAD, P, dW + L.w[5], dW + L.b[5], part, st))) return rc;
  if ((rc = gemm<false, true>(Mat{W + L.w[5], 1, HEAD}, Mat{d_flow, 1, 3}, HEAD, P, 3, 3, ZeroInit{},
                              DeltaEpi{D0, h5, P, nullptr, nullptr, HEAD, nullptr, 0}, st))) return rc;
  float *cur = D0, *nxt = D1;
  for (int l = 4; l >= 0; --l) {
    const float* in = saved + (l == 0 ? M_PE : m_h(l)) * P;
    if ((rc = weight_grad<true>(Mat{cur, P, 1}, in, HEAD, L.kin[l], P, dW + L.w[l], dW + L.b[l], part, st, prec))) return rc;
    if (l > 0) {                                            // the encoding of xyzt gets no gradient
      if ((rc = delta_layer(W, L, l, cur, HEAD, P, DeltaEpi{nxt, in, P, nullptr, nullptr, HEAD, nullptr, 0}, st, prec)))
        return rc;
      float* t = cur; cur = nxt; nxt = t;
    }
  }
  return STNERF_OK;
}

}  // namespace stnerf
