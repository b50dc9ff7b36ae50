// 3xTF32 warpgroup-MMA (sm_90a wgmma) GEMM of the training path: STNERF_TRAIN_TC_3XTF32.
//
// The same three roles as the fp32 SIMT GEMM of mlp_train.cu, with its epilogue functors (mlp_train.cuh) and its point chunks:
//   forward   out(n_out x P) = relu(W . in + b)                      (BiasInit, Store)
//   delta     d_in(k x P)    = W^T . d_out, masked by in > 0         (DeltaEpi: skip / PE(pos) row split, ws . ds of the density head)
//   weights   partial tile of chunk z = d_out . in^T over its points (PartialStore; mlp_train.cu adds the partials in chunk order)
// mlp_train.cu routes every layer with 128 or more outputs here (the 7 SpaceNet trunk layers, rgb_net.1, motion_net.0 - .8); the
// 1- and 3-wide heads stay on the SIMT GEMM.
//
// Precision.  Every operand x is split as hi = tf32_rna(x), lo = tf32_rna(x - hi) (x - hi is exact in fp32), and every product is
// Alo.Bhi + Ahi.Blo + Ahi.Bhi on wgmma m64n128k8 .tf32 with fp32 accumulation: about 22 significant bits per product.  Unlike the
// render's fp16 split, tf32 keeps fp32's 8-bit exponent, so deltas and gradient terms of any magnitude fp32 can hold keep their
// relative precision without scaling (lo underflows only where x is within 2^22 of the smallest normal).
// Order: within one k-stage of 32 the two correction products of all four k8 steps go first, then Ahi.Bhi, into an accumulator
// that starts from zero (scale-d = 0) at every stage; after the stage the accumulator is added into a separate fp32 register
// total with an ordinary round-to-nearest add (PROMOTE_STAGES).  So no wgmma accumulator runs over more than 32 k-terms -- the
// tensor core's fp32 accumulation truncates (DESIGN.md section 4) -- and the small products are added while the accumulator is
// small.  The forward starts the total at the bias.
//
// Shape.  A CTA of two warpgroups computes a 128 (M) x 128 (N) tile; warpgroup w owns rows 64 w .. 64 w + 63 and holds their
// 64 x 128 accumulator and total in registers.  Both operands go through registers: all 256 threads load the next [128 x 32]
// fp32 tile of A and of B from global memory (coalesced along whichever of rows or k is contiguous), split it and write the hi /
// lo halves into the 128B-swizzled K-major shared-memory layout that tf32 wgmma requires for both operands -- this is where the
// feature-major (point-contiguous) activations are transposed.  Two stages of 64 KB: stage s + 1 is loaded before the twelve
// MMAs of stage s are issued and split and stored while they execute.  Rows beyond M / N and k beyond the chunk are zero in shared
// memory and masked in the epilogue, so K = 63, 84, 283, 304, 319 and the 63-row PE(pos) deltas need no special case.
//
// Determinism: no atomics; a point's outputs are a function of its own column only (every column of a tile sees the same k
// order), and the weight-gradient chunks are fixed by P alone, so identical calls give identical bits.  The forward is not
// bit-identical to any render precision mode.
#include "mlp_train.cuh"

namespace stnerf {

namespace {

constexpr int TM = 128, TN = 128;                 // CTA tile
constexpr int TKS = 32;                           // k per stage: one 128-byte swizzle row of fp32
constexpr int NT = 256;                           // two math warpgroups
constexpr int OP_BYTES = TM * TKS * 4;            // one [128 rows x 32 k] fp32 operand tile, 128B-swizzled K-major: 16 KB
constexpr int STAGE_BYTES = 4 * OP_BYTES;         // A hi | A lo | B hi | B lo
constexpr int SMEM_BYTES = 2 * STAGE_BYTES + 1024;   // two stages + alignment of the 1024-byte swizzle atoms
constexpr int PER_T = TM * TKS / NT;              // elements of one operand tile each thread loads and splits per stage
constexpr int PROMOTE_STAGES = 1;                 // k-stages per wgmma accumulator block (DESIGN.md section 3.8)
static_assert(TM == TN, "one element mapping serves both operand tiles");

// Operand view: element (r, k) at p[r*sr + k*sk], rows r < rows
struct Op {
  const float* p;
  long long sr, sk, rows;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// K-major SWIZZLE_128B descriptor (mode 1): 8-row groups 1024 B apart; one k8 step of tf32 is +32 bytes on the start address
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// byte offset of element (r, k) of a [rows x 32] fp32 tile, 128B-swizzled K-major
__device__ __forceinline__ uint32_t sw128_f32(int r, int k) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 2) ^ r) & 7) << 4) + ((k & 3) << 2));
}

#define TF_D "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define TF_OPS(d) \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (+)= A[64 x 8] . B[128 x 8]^T, both tf32 K-major in shared memory, fp32 accumulate; scale_d = 0 ignores D's input
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {" TF_D "}, %64, %65, p, 1, 1;\n\t}"
      : TF_OPS(d)
      : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Element e of this thread's share of a [128 x 32] tile.  KC (operand contiguous along k in global memory): a warp reads one
// row's 32 k (128 B).  Else (contiguous along rows): a warp reads 8 consecutive rows at 4 consecutive k (4 x 32 B), which also
// makes its shared-memory stores hit 32 different banks.
template <bool KC>
__device__ __forceinline__ void elem(int tid, int e, int& r, int& k) {
  const int lane = tid & 31, w = (tid >> 5) + (NT / 32) * e;
  if (KC) {
    r = w;
    k = lane;
  } else {
    r = ((w & 15) << 3) | (lane >> 2);
    k = ((w >> 4) << 2) | (lane & 3);
  }
}

// This thread's share of loading one operand tile per stage: the address of its element 0 and pointer steps to the others
// (pointer bumps rather than 16 precomputed 64-bit addresses, which would not fit beside the accumulators).
template <bool KC>
struct Loader {
  const float* q;              // element 0 at the current stage
  long long step_r, step_k;    // KC: element e + 1 is 8 rows further; else odd elements are 64 rows further, pairs 4 k further
  long long step_s;            // one stage further along k
  int r, k, rows_left;         // element 0's (row, k) in the tile; rows of the operand from the tile's first row on
  __device__ __forceinline__ Loader(const Op& X, long long r0, long long k0, int tid) {
    elem<KC>(tid, 0, r, k);
    q = X.p + (r0 + r) * X.sr + (k0 + k) * X.sk;
    step_r = (KC ? 8 : 64) * X.sr;
    step_k = 4 * X.sk;
    step_s = TKS * X.sk;
    rows_left = (int)min(X.rows - r0, (long long)(1 << 30));
  }
  __device__ __forceinline__ void load(float (&v)[PER_T], int k_left) const {
    const float* p = q;
    if (KC) {
      const bool kok = k < k_left;
#pragma unroll
      for (int e = 0; e < PER_T; ++e, p += step_r) v[e] = (kok && r + 8 * e < rows_left) ? __ldg(p) : 0.f;
    } else {
      const bool r0ok = r < rows_left, r1ok = r + 64 < rows_left;
#pragma unroll
      for (int e = 0; e < PER_T; e += 2, p += step_k) {
        const bool kok = k + 2 * e < k_left;
        v[e] = (kok && r0ok) ? __ldg(p) : 0.f;
        v[e + 1] = (kok && r1ok) ? __ldg(p + step_r) : 0.f;
      }
    }
  }
  __device__ __forceinline__ void next() { q += step_s; }
};

// hi tile at `hi`, lo tile OP_BYTES after it
template <bool KC>
__device__ __forceinline__ void store_op(uint8_t* hi, const float (&v)[PER_T], int tid) {
#pragma unroll
  for (int e = 0; e < PER_T; ++e) {
    int r, k;
    elem<KC>(tid, e, r, k);
    const uint32_t off = sw128_f32(r, k);
    const float h = tf32_rna(v[e]);
    *reinterpret_cast<float*>(hi + off) = h;
    *reinterpret_cast<float*>(hi + OP_BYTES + off) = tf32_rna(v[e] - h);
  }
}

// C(m, n) = init(m) + sum over k in chunk blockIdx.z of A(m, k) B(n, k); epi(m, n, C) for m < A.rows, n < B.rows
template <bool A_KC, bool B_KC, class Init, class Epi>
__global__ void __launch_bounds__(NT, 1) tc_gemm_kernel(const Op A, const Op B, long long K, long long kchunk, Init init, Epi epi) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw), base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
  const long long m0 = (long long)blockIdx.y * TM, n0 = (long long)blockIdx.x * TN;
  const long long kb = (long long)blockIdx.z * kchunk, ke = min(K, kb + kchunk);
  const int ns = ke > kb ? (int)((ke - kb + TKS - 1) / TKS) : 0;
  // accumulator fragment: acc[i] is tile row r_frag + 8 ((i >> 1) & 1), column c_frag + 8 (i >> 2) + (i & 1)
  const int r_frag = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2), c_frag = 2 * (t & 3);
  float acc[64], tot[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const long long m = m0 + r_frag + 8 * ((i >> 1) & 1);
    tot[i] = m < A.rows ? init((int)m) : 0.f;
    acc[i] = 0.f;
  }
  float va[PER_T], vb[PER_T];
  Loader<A_KC> la(A, m0, kb, tid);
  Loader<B_KC> lb(B, n0, kb, tid);
  if (ns > 0) {
    la.load(va, (int)min(ke - kb, (long long)TKS));
    lb.load(vb, (int)min(ke - kb, (long long)TKS));
    store_op<A_KC>(smem, va, tid);
    store_op<B_KC>(smem + 2 * OP_BYTES, vb, tid);
  }
  fence_proxy_async();
  __syncthreads();
  for (int s = 0; s < ns; ++s) {
    const bool more = s + 1 < ns;
    if (more) {
      const int k_left = (int)min(ke - kb - (long long)(s + 1) * TKS, (long long)TKS);
      la.next();
      lb.next();
      la.load(va, k_left);
      lb.load(vb, k_left);
    }
    const uint32_t a_hi = base + (s & 1) * STAGE_BYTES + wg * (64 * 128), a_lo = a_hi + OP_BYTES;
    const uint32_t b_hi = base + (s & 1) * STAGE_BYTES + 2 * OP_BYTES, b_lo = b_hi + OP_BYTES;
    const uint32_t fresh = (s % PROMOTE_STAGES) == 0;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < TKS / 8; ++j) {
      wgmma_tf32(acc, desc_sw128(a_lo + 32 * j), desc_sw128(b_hi + 32 * j), (j > 0 || !fresh) ? 1u : 0u);
      wgmma_tf32(acc, desc_sw128(a_hi + 32 * j), desc_sw128(b_lo + 32 * j), 1u);
    }
#pragma unroll
    for (int j = 0; j < TKS / 8; ++j) wgmma_tf32(acc, desc_sw128(a_hi + 32 * j), desc_sw128(b_hi + 32 * j), 1u);
    wgmma_commit();
    if (more) {      // the other stage was last read by the MMAs of stage s - 1, which have retired
      uint8_t* nb = smem + ((s + 1) & 1) * STAGE_BYTES;
      store_op<A_KC>(nb, va, tid);
      store_op<B_KC>(nb + 2 * OP_BYTES, vb, tid);
    }
    wgmma_wait0();
    if ((s + 1) % PROMOTE_STAGES == 0 || !more) {
#pragma unroll
      for (int i = 0; i < 64; ++i) tot[i] += acc[i];
    }
    fence_proxy_async();
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const long long m = m0 + r_frag + 8 * ((i >> 1) & 1), n = n0 + c_frag + 8 * (i >> 2) + (i & 1);
    if (m < A.rows && n < B.rows) epi((int)m, n, tot[i]);
  }
}

template <bool A_KC, bool B_KC, class Init, class Epi>
int tc_gemm(Op A, Op B, long long K, long long kchunk, Init init, Epi epi, cudaStream_t st) {
  if (A.rows <= 0 || B.rows <= 0) return STNERF_OK;
  auto kern = tc_gemm_kernel<A_KC, B_KC, Init, Epi>;
  STNERF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  const long long nz = K > 0 ? (K + kchunk - 1) / kchunk : 1;
  const dim3 grid((unsigned)((B.rows + TN - 1) / TN), (unsigned)((A.rows + TM - 1) / TM), (unsigned)nz);
  kern<<<grid, NT, SMEM_BYTES, st>>>(A, B, K, kchunk, init, epi);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}
}  // namespace

int tc_train_forward(const float* W, int K, const float* bias, const float* in, int M, long long P, float* out, cudaStream_t st) {
  return tc_gemm<true, false>(Op{W, K, 1, M}, Op{in, 1, P, P}, K, K, BiasInit{bias}, Store{out, P, 1, 1}, st);
}

int tc_train_delta(const float* W, int kin, int nout, const float* d_out, int M, long long P, float* out, const float* h,
                   const float* ws, const float* ds, int split, float* enc, int acc, cudaStream_t st) {
  return tc_gemm<false, false>(Op{W, 1, kin, M}, Op{d_out, 1, P, P}, nout, nout, ZeroInit{},
                               DeltaEpi{out, h, P, ws, ds, split, enc, acc}, st);
}

int tc_train_wgrad(const float* d, const float* h, int M, int N, long long P, long long chunk, float* part, cudaStream_t st) {
  return tc_gemm<true, true>(Op{d, P, 1, M}, Op{h, P, 1, N}, P, chunk, ZeroInit{}, PartialStore{part, N, (long long)M * N}, st);
}

}  // namespace stnerf
