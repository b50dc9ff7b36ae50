// Hopper (sm_90a) tensor-core evaluation of SpaceNet and MotionNet with warpgroup MMAs (wgmma): precision modes TC_3XF16 "exact",
// TC_3XF16_CF "exact_cf", TC_MIXED "mixed", TC_F16 "fast".
//
// Persistent CTAs (one per SM) walk tiles of 128 points.  Per tile the whole network runs on-chip:
//   * CTA = three warpgroups.  Warpgroup 0: warp 0 streams the weights, warps 2..3 are the coarse-pass compositing warps
//     (FuseCoarse, below).  Warpgroups 1 and 2 are the math warpgroups: warpgroup 1 + w owns rows 64 w .. 64 w + 63 of the tile,
//     issues their MMAs (wgmma m64 x N x k16, N = 256 or 128, accumulators in registers) and runs their epilogues.  The two
//     math warpgroups share nothing but the weight ring, so while one runs its epilogue the other keeps the tensor cores busy;
//   * activations (A operand) are fp16 hi/lo pairs.  The hi halves (and the whole encoding) live in shared memory in the
//     canonical 128B-swizzled K-major layout ([128 rows x 64 k] blocks); a layer's epilogue overwrites the rows its own MMAs
//     have just finished reading.  In the SpaceNet kernel the lo halves of the hidden activations stay in the math threads'
//     registers, in the wgmma A-fragment layout the accumulator already has (epi_hidden), and Alo*Whi is the register-A form
//     of wgmma; that frees 64 KB of shared memory for a 7-deep weight ring, and setmaxnreg moves registers from warpgroup 0
//     to the math warpgroups to hold them;
//   * weights (B operand) are pre-packed on the host into [N out-rows x 32 k] fp16 blocks that are already the 64B-swizzled
//     shared-memory image -- per layer the hi and then the lo stage of every 32-k sub-chunk, in the layer's K order, each
//     stored once -- and stream through a ring of stages with 1-D bulk async copies (cp.async.bulk + mbarrier complete_tx) from
//     L2, in the order of the layer's steps (WSched); a slot is refilled once every math warp has seen the MMAs that read it
//     retire (wgmma.wait_group);
//   * exact mode issues three fp16 MMAs per product, D += Ahi*Whi + Alo*Whi + Ahi*Wlo (fp32 accumulate), which reproduces fp32
//     products to ~2^-22 (SURVEY App. C.3: the only tensor-core formulation inside the 1e-3 gate); mixed mode keeps that
//     everywhere the density depends on and runs the colour-only layer rgb_net.1 in one pass;
//   * order of the three products (template parameter LOFIRST): interleaved per 32-k sub-chunk (default: every weight stage is
//     streamed once), or -- TC_3XF16_CF "exact_cf", coarse pass + MotionNets -- the two correction products FIRST over the whole K
//     range, then Ahi*Whi, so the accumulator is small while the corrections are added (stnerf_selftest_umma_accum measures how
//     the tensor core rounds its fp32 accumulation); the hi weight stages are then streamed twice (stored once);
//   * relu(PE(dir) | PE(time)) enters rgb_net.1 as a per-ray fp32 bias computed by head_bias_kernel
//     (b1 + W1[:,256:] . relu(enc)), so the last GEMM is a clean K=256;
//   * the 1-wide density head, the 3-wide rgb / flow heads and all biases are fp32 FFMA work in the epilogue;
//   * in the coarse pass (n1 = 64: a tile = two whole rays of one layer) the two compositing warps composite the tile's rgb / sigma
//     rows and draw + merge the fine depths (FuseCoarse, resample.cuh): the coarse samples never leave the SM.
//
// Restates modeling/spacenet.py:101-160, modeling/motion_net.py:34-71, utils/dimension_kernel.py:24-33.
#include <cuda_fp16.h>
#include <string.h>
#include <type_traits>
#include <vector>
#include "mlp_tc.cuh"
#include "resample.cuh"

namespace stnerf {

namespace {

constexpr int TILE_M = 128;
constexpr int ABLOCK = 16384;                // activation block [128 rows x 64 k] fp16, SWIZZLE_128B
constexpr int STAGE_BYTES = 16384;           // weight stage   [256 rows x 32 k] fp16, SWIZZLE_64B (N=128 layers use half)
constexpr int NTHREADS = 384;                // warpgroup 0: producer + compositing warps; warpgroups 1, 2: math
constexpr int MATH_WG0 = 1, N_MATH_WARPS = 8;
constexpr int MAX_STAGE = 8;
// registers per thread after setmaxnreg (SpaceNet kernel): warpgroup 0 (producer, compositing warps) and the math warpgroups;
// 128 REGS_WG0 + 256 REGS_MATH must not exceed the 384 x 168 the launch allocates
constexpr int REGS_WG0 = 56, REGS_MATH = 224;
static_assert(128 * REGS_WG0 + 256 * REGS_MATH <= 384 * 168, "register file");
constexpr int BAR_WFULL = 0, BAR_WEMPTY = 8, BAR_RAWFULL = 16, BAR_RAWEMPTY = 18;          // 20 barriers
// misc region: barriers | per-row point info of the current tile | final rows for the compositing warps | their scratch
constexpr int MISC_ROWS = 256;               // Pt[128]
constexpr int MISC_PART = MISC_ROWS + 128 * 24;   // float4[128]: the tile's final (rgb logits, sigma) rows (coarse-pass fusion)
constexpr int MISC_CDF = MISC_PART + 2048;   // fused compositing warps: cdf / depth scratch, 2 x 64 floats
constexpr int MISC_TOTAL = MISC_CDF + 512;

// ---------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar), "r"((uint32_t)pred)
               : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug traps (the kernel aborts with an error) instead of hanging the GPU.  The loop lives inside one asm
// block so that the compiler sees no divergent branch in front of the warpgroup MMAs that follow a wait.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 c;\n\t"
      "mov.u32 c, 0;\n"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni DONE_%=;\n\t"
      "add.u32 c, c, 1;\n\t"
      "setp.gt.u32 p, c, 67108864;\n\t"
      "@p trap;\n\t"
      "bra.uni WAIT_%=;\n"
      "DONE_%=:\n\t}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// per-thread register budget of the whole warpgroup (sm_90a); every thread of the warpgroup executes the same one
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier of one math warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// Weight-stage load by one elected lane of the converged producer warp: announce the bytes on `bar`, then the bulk copy.
__device__ __forceinline__ void load_stage_elect(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%3], %2;\n\t"
      "@pe cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// ---- warpgroup MMA ----------------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptors (sm_90 layout), K-major operands: start address >> 4 in bits 0-13, leading byte offset
// (unused by swizzled K-major operands) in 16-29, stride byte offset (8-row groups) >> 4 in 32-45, swizzle mode in 62-63.
//   A: SWIZZLE_128B (mode 1), 8-row groups 1024 B apart;  B: SWIZZLE_64B (mode 2), 8-row groups 512 B apart.
// One K=16 step further along K is +32 bytes on the start address (the swizzle is applied to the absolute address).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint64_t desc_sw64(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across a wgmma.wait_group
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// fp32 accumulator operands of an m64nNk16 wgmma: %0 .. %63 (N = 128), then %64 .. %127 (N = 256), and their constraints
#define WGMMA_D_LO "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define WGMMA_D_HI "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define WGMMA_OPS_LO(d) \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define WGMMA_OPS_HI(d) \
    "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
    "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
    "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
    "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
    "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
    "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
    "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
    "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])

// D[64 x 256] += A[64 x 16] * B[256 x 16]^T, both K-major in shared memory; fp16 in, fp32 accumulate in registers
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{" WGMMA_D_LO ", " WGMMA_D_HI "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : WGMMA_OPS_LO(d), WGMMA_OPS_HI(d)
      : "l"(da), "l"(db), "r"(1));
}
// D[64 x 128] += A[64 x 16] * B[128 x 16]^T, both K-major in shared memory; fp16 in, fp32 accumulate in registers
__device__ __forceinline__ void wgmma_n128(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{" WGMMA_D_LO "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : WGMMA_OPS_LO(d)
      : "l"(da), "l"(db), "r"(1));
}
// The same with A in registers: a[0..3] is this thread's fragment of the 64 x 16 A slice (f16x2 each: rows r, r + 8 at columns
// c, c + 1, then the same rows at columns c + 8, c + 9, with r and c as in the accumulator fragment -- see epi_hidden).
// wgmma reads the registers asynchronously: they must not change before the MMA has retired (wgmma.wait_group).
__device__ __forceinline__ void wgmma_n256_rs(float (&d)[128], const uint32_t* a, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{" WGMMA_D_LO ", " WGMMA_D_HI "}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
      : WGMMA_OPS_LO(d), WGMMA_OPS_HI(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_n128_rs(float (&d)[128], const uint32_t* a, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{" WGMMA_D_LO "}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : WGMMA_OPS_LO(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}

template <int N>
__device__ __forceinline__ void wgmma_k16(float (&d)[128], uint64_t da, uint64_t db) {
  if (N == 256) wgmma_n256(d, da, db);
  else wgmma_n128(d, da, db);
}
template <int N>
__device__ __forceinline__ void wgmma_k16_rs(float (&d)[128], const uint32_t* a, uint64_t db) {
  if (N == 256) wgmma_n256_rs(d, a, db);
  else wgmma_n128_rs(d, a, db);
}

// {lo16 = fp16(a), hi16 = fp16(b)}, saturating to +-65504 (fp16 range guard of the split)
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t p) {
  return __half22float2(*reinterpret_cast<const __half2*>(&p));
}

// byte offset of element (row, col) of a [rows x 64] fp16 block, 128B-swizzled K-major (activations)
__host__ __device__ inline uint32_t sw128_offset(int row, int col) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((col >> 3) ^ (row & 7)) & 7) << 4) + ((col & 7) << 1));
}
// byte offset of element (row, col) of a [rows x 32] fp16 block, 64B-swizzled K-major (weights)
__host__ __device__ inline uint32_t sw64_offset(int row, int col) {
  return (uint32_t)((row >> 3) * 512 + (row & 7) * 64 + ((((col >> 3) ^ ((row >> 1) & 3)) & 3) << 4) + ((col & 7) << 1));
}

// ---------------------------------------------------------------------------------------------------------
// network schedules (compile-time)
// ---------------------------------------------------------------------------------------------------------
enum { NET_SPACE = 0, NET_MOTION = 1 };

template <int NET> struct Sched;
template <> struct Sched<NET_SPACE> {
  static constexpr int N_LAYERS = 8;
  // shared memory: activations (4 hi blocks), encoding (hi, lo), a 7-deep ring of 16 KB weight stages, misc.  The lo halves of
  // the activations never reach shared memory: each math thread keeps its fragment of them in registers (lo_in_regs, epi_hidden)
  static constexpr bool lo_in_regs = true;
  static constexpr int act_base = 0, enc_base = 4 * ABLOCK;
  static constexpr int ENC_LO_STRIDE = ABLOCK;
  static constexpr int n_stage = 7, stage_bytes = STAGE_BYTES;
  static constexpr int ring_base = 6 * ABLOCK, misc_base = ring_base + n_stage * stage_bytes, smem_total = misc_base + MISC_TOTAL;
  static_assert(smem_total <= 232448, "shared memory budget (227 KB per CTA)");
  __host__ __device__ static constexpr int n_out(int l) { return l == 7 ? 128 : 256; }
  __host__ __device__ static constexpr int act_chunks(int l) { return l == 0 ? 0 : 4; }
  __host__ __device__ static constexpr int enc_chunks(int l) { return (l == 0 || l == 4) ? 1 : 0; }
  // the skip layer consumes its encoding chunk FIRST (the weight stream is packed in the same order)
  __host__ __device__ static constexpr bool enc_first(int l) { return l == 4; }
};
template <> struct Sched<NET_MOTION> {
  static constexpr int N_LAYERS = 5;
  // the encoding (read by layer 0 only) shares the activation blocks: layer 0's epilogue overwrites it after its MMAs retired
  static constexpr bool lo_in_regs = false;
  static constexpr int act_base = 0, enc_base = 0;
  static constexpr int LO_STRIDE = 2 * ABLOCK;
  static constexpr int ENC_LO_STRIDE = 2 * ABLOCK;
  static constexpr int n_stage = 8, stage_bytes = 8192;
  static constexpr int ring_base = 4 * ABLOCK, misc_base = ring_base + n_stage * stage_bytes, smem_total = misc_base + MISC_TOTAL;
  __host__ __device__ static constexpr int n_out(int) { return 128; }
  __host__ __device__ static constexpr int act_chunks(int l) { return l == 0 ? 0 : 2; }
  __host__ __device__ static constexpr int enc_chunks(int l) { return l == 0 ? 2 : 0; }
  __host__ __device__ static constexpr bool enc_first(int) { return false; }
};
static_assert(Sched<NET_SPACE>::n_stage <= MAX_STAGE && Sched<NET_MOTION>::n_stage <= MAX_STAGE, "barrier slots");

// Weight schedule of a layer: the one definition of the order in which the producer streams the weight stages and the math
// warpgroups consume them.  A layer's section of the stream holds, per 32-k sub-chunk in the layer's K order, the hi stage and
// then the lo stage ([n_out rows x 32 k] fp16 each).  Each step loads one stage and multiplies it with the A slice of one
// sub-chunk:
//   * interleaved split (exact, mixed): per sub-chunk the lo stage (Ahi*Wlo), then the hi stage (Ahi*Whi, then Alo*Whi);
//   * corrections first (LOFIRST, exact_cf): per sub-chunk the lo stage (Ahi*Wlo) and the hi stage (Alo*Whi) over the whole
//     K range, then every hi stage again (Ahi*Whi);
//   * single pass (fast, and the last layer in mixed): the hi stages only (Ahi*Whi).
enum { A_HI = 0, A_LO = 1, A_HI_LO = 2 };     // A operand of a step: Ahi, Alo, or Ahi then Alo (two MMA pairs off one stage)
template <int A>
struct WStep {
  static constexpr int a = A;
  uint32_t offset;                            // byte offset of the step's weight stage inside the layer's section
  uint32_t sub;                               // 32-k sub-chunk of the A chunk
};
template <int NET>
struct WSched {
  using S = Sched<NET>;
  __host__ __device__ static constexpr int n_chunks(int l) { return S::act_chunks(l) + S::enc_chunks(l); }
  __host__ __device__ static constexpr uint32_t stage_bytes(int l) { return (uint32_t)S::n_out(l) * 64; }
  __host__ __device__ static constexpr size_t layer_bytes(int l) { return (size_t)n_chunks(l) * 2 /*sub-chunks*/ * 2 /*hi, lo*/ * stage_bytes(l); }
  // chunk id (activation chunks 0 .. act_chunks-1, then the encoding chunks) at position c of the layer's K order: the skip
  // layer takes its encoding chunk first
  __host__ __device__ static constexpr int chunk_at(int l, int c) {
    return S::enc_first(l) ? (c == 0 ? S::act_chunks(l) : c - 1) : c;
  }
  static constexpr bool enc_first_valid() {
    for (int l = 0; l < S::N_LAYERS; ++l)
      if (S::enc_first(l) && (S::act_chunks(l) == 0 || S::enc_chunks(l) == 0)) return false;
    return true;
  }
  static_assert(enc_first_valid(), "enc_first(l) needs activation chunks and an encoding chunk to reorder");
  // The steps of layer l, in order: per A chunk, a = chunk(chunk id) once, then f(a, WStep<A>) for every step on that chunk.
  // The operand is a compile-time constant, so every kind of step is a separate, straight-line copy of f.
  template <bool LOFIRST, class C, class F>
  __device__ __forceinline__ static void for_each_step(int l, bool split, C&& chunk, F&& f) {
    // written out rather than n_chunks(l): with the call, nvcc fully unrolls the MotionNet correction pass, and that kernel spills
    const int nact = S::act_chunks(l), nch = nact + S::enc_chunks(l);
    const uint32_t bytes = stage_bytes(l);
    auto at = [&](const auto& a, int c, uint32_t sub, uint32_t lo_stage, auto op) {
      f(a, WStep<decltype(op)::value>{(2 * (2 * (uint32_t)c + sub) + lo_stage) * bytes, sub});
    };
    using HI = std::integral_constant<int, A_HI>;
    using LO = std::integral_constant<int, A_LO>;
    using HI_LO = std::integral_constant<int, A_HI_LO>;
    if (!LOFIRST || !split) {
      for (int c = 0; c < nch; ++c) {
        const auto a = chunk(chunk_at(l, c));
        for (uint32_t sub = 0; sub < 2; ++sub) {
          if (split) { at(a, c, sub, 1u, HI()); at(a, c, sub, 0u, HI_LO()); }
          else at(a, c, sub, 0u, HI());
        }
      }
    } else {
      for (int c = 0; c < nch; ++c) {
        const auto a = chunk(chunk_at(l, c));
        for (uint32_t sub = 0; sub < 2; ++sub) { at(a, c, sub, 1u, HI()); at(a, c, sub, 0u, LO()); }
      }
      for (int c = 0; c < nch; ++c) {
        const auto a = chunk(chunk_at(l, c));
        for (uint32_t sub = 0; sub < 2; ++sub) at(a, c, sub, 0u, HI());
      }
    }
  }
};

template <int NET>
__host__ __device__ constexpr size_t stream_bytes_per_tile() {
  size_t n = 0;
  for (int l = 0; l < Sched<NET>::N_LAYERS; ++l) n += WSched<NET>::layer_bytes(l);
  return n;
}

struct TcParams {
  FuseCoarse fuse;            // SpaceNet, coarse pass: per-layer compositing + resampling in the compositing warps
  PointSrc src;
  const uint8_t* wstream;     // packed weight stream (per layer: hi, lo stage per 32-k sub-chunk; see WSched)
  const float* aux;           // fp32: biases [8][256] | w_sigma[256] | b_sigma | w_out[3][128] | b_out[3]
  const float* cbuf;          // SpaceNet: per-slot rgb_net.1 bias (b1 + W1[:,256:].relu(enc(dir,time))), [slots][128]
  int exact;                  // 1: 3-term split, 0: single fp16 pass
  int single_last;            // with exact: the LAST GEMM layer (SpaceNet rgb_net.1, colour branch only) runs a single pass
  int lo_first;               // split layers (selects the kernel instantiation): 0 = interleaved per 32-k sub-chunk (hi stages
                              // streamed once); 1 = correction products first over the whole K range, then Ahi*Whi (WSched)
  // outputs
  float* raw;                 // float4 per sample (pipeline mode)
  float* rgb_out;             // explicit mode
  float* sigma_out;
  float* xyz_out;             // MotionNet: deformed position (pipeline) ...
  float* flow_out;            // ... or flow (explicit)
  const int* lerp_flag;
  int lerp_force;
};

constexpr int AUX_BIAS = 0, AUX_WSIG = 8 * 256, AUX_BSIG = AUX_WSIG + 256, AUX_WOUT = AUX_BSIG + 4,
              AUX_BOUT = AUX_WOUT + 3 * 128, AUX_FLOATS = AUX_BOUT + 4;


// ---------------------------------------------------------------------------------------------------------
// point fetch
// ---------------------------------------------------------------------------------------------------------
struct Pt { float x, y, z, tm; int out_index; int cidx; };

__device__ __forceinline__ Pt fetch_pt(const PointSrc& s, long long p, long long n_points) {
  Pt q;
  q.x = q.y = q.z = q.tm = 0.f;
  q.out_index = -1;
  q.cidx = 0;
  if (p >= n_points) return q;
  if (s.mode == SRC_EXPLICIT) {
    const float* pp = s.pos + p * s.pos_stride;
    q.x = pp[0]; q.y = pp[1]; q.z = pp[2];
    if (s.times) q.tm = s.times[p * s.time_stride];
    q.out_index = (int)p;
    q.cidx = (int)p;
    return q;
  }
  const long long slot = p / s.S;
  const int k = (int)(p - slot * s.S);
  const long long ray = s.hit ? (long long)s.hit[slot] : slot;
  const float* rp = s.rays + ray * s.ray_stride;
  q.tm = rp[6 + s.layer];
  q.out_index = (int)(ray * s.S + k);
  q.cidx = (int)slot;
  if (s.mode == SRC_XYZ) {
    q.x = s.pos[3 * p]; q.y = s.pos[3 * p + 1]; q.z = s.pos[3 * p + 2];
    return q;
  }
  if (s.mode == SRC_XYZ_MAP) {           // fine pass with flow reuse: where did depth k of this ray come from?
    const int m = s.src_map[ray * s.S + k];
    const float* pp = (m < s.n_first) ? s.pos + 3 * (slot * s.n_first + m) : s.pos2 + 3 * (slot * (s.S - s.n_first) + (m - s.n_first));
    q.x = pp[0]; q.y = pp[1]; q.z = pp[2];
    return q;
  }
  float v[3];
  march_point(s, rp, s.t[ray * s.S + k], rp[3], rp[4], rp[5], v);
  q.x = v[0]; q.y = v[1]; q.z = v[2];
  return q;
}

// Full-range sin/cos (Cody-Waite + Payne-Hanek slow path) out of line: inlining it at every encoding site made the
// kernels 150-400 KB of SASS, far beyond the instruction cache.  Three / four independent angles per call, so the
// dependent reduction + polynomial chains of the copies interleave (the epilogue warps are latency-bound here: two warps
// per scheduler).
struct SinCos3 { float s0, s1, s2, c0, c1, c2; };
struct SinCos4 { float s0, s1, s2, s3, c0, c1, c2, c3; };
__device__ __noinline__ SinCos3 sincos_full3(float x0, float x1, float x2) {
  SinCos3 r;
  sincosf(x0, &r.s0, &r.c0); sincosf(x1, &r.s1, &r.c1); sincosf(x2, &r.s2, &r.c2);
  return r;
}
__device__ __noinline__ SinCos4 sincos_full4(float x0, float x1, float x2, float x3) {
  SinCos4 r;
  sincosf(x0, &r.s0, &r.c0); sincosf(x1, &r.s1, &r.c1); sincosf(x2, &r.s2, &r.c2); sincosf(x3, &r.s3, &r.c3);
  return r;
}

// Write NV fp32 values of one row as fp16 hi (+lo) 16-byte chunks: columns col0 .. col0+NV-1 of an activation block
// (col0 and NV multiples of 8).
template <int NV>
__device__ __forceinline__ void store_row_split(uint8_t* hi_blk, int lo_stride, int row, int col0, const float (&v)[NV],
                                                bool exact) {
#pragma unroll
  for (int g = 0; g < NV / 8; ++g) {
    uint32_t hp[4], lp[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a = v[g * 8 + 2 * e], b = v[g * 8 + 2 * e + 1];
      hp[e] = pack_f16x2(a, b);
      const float2 hf = unpack_f16x2(hp[e]);
      lp[e] = pack_f16x2(a - hf.x, b - hf.y);
    }
    const uint32_t off = sw128_offset(row, col0 + g * 8);
    *reinterpret_cast<uint4*>(hi_blk + off) = make_uint4(hp[0], hp[1], hp[2], hp[3]);
    if (exact) *reinterpret_cast<uint4*>(hi_blk + lo_stride + off) = make_uint4(lp[0], lp[1], lp[2], lp[3]);
  }
}

// Input encoding of one row, written by the two threads (half = 0/1) that own the row, in PIECES that are spread over
// the idle time the epilogue warps have between layers (each piece = whole 16-byte chunks of the swizzled block).
// Column order is a permutation of the reference's (utils/dimension_kernel.py:24-33); the weight packer applies the
// same permutation (enc_perm_* below).  With f_k = [sin(2^k x), sin(2^k y), sin(2^k z), cos ...] (6 values, SpaceNet)
// or the 8-value xyzt analogue (MotionNet):
//   SpaceNet, 64 cols : half 0 -> [f0 f1 f2 | f3 f4 x y]      half 1 -> [f5 f6 f7 | f8 f9 z 0]        (2 pieces of 16 cols)
//   MotionNet, 2 x 64 : half h -> block h: chunk c<5 = f_(5h+c), chunk 5 = [x y z t 0 0 0 0] (h=0) / 0, chunks 6,7 = 0
//                       pieces: {f_(5h), f_(5h+1)}, {f_(5h+2), f_(5h+3)}, {f_(5h+4), raw}
template <int half, int piece>
__device__ __forceinline__ void encode_space_piece(uint8_t* smem, const Pt& pt, int row, bool exact, float (&carry)[2]) {
  using S = Sched<NET_SPACE>;
  uint8_t* enc = smem + S::enc_base;
  const float xs[3] = {pt.x, pt.y, pt.z};
  float v[16];
  auto trig = [&](int f, float* dst) {
    const float fr = (float)(1 << f);
    const SinCos3 q = sincos_full3(xs[0] * fr, xs[1] * fr, xs[2] * fr);
    dst[0] = q.s0; dst[1] = q.s1; dst[2] = q.s2; dst[3] = q.c0; dst[4] = q.c1; dst[5] = q.c2;
  };
  if (piece == 0) {
    float t3[6];
    trig(5 * half + 0, v); trig(5 * half + 1, v + 6); trig(5 * half + 2, t3);
    v[12] = t3[0]; v[13] = t3[1]; v[14] = t3[2]; v[15] = t3[3];
    carry[0] = t3[4]; carry[1] = t3[5];
  } else {
    v[0] = carry[0]; v[1] = carry[1];
    trig(5 * half + 3, v + 2); trig(5 * half + 4, v + 8);
    v[14] = half == 0 ? xs[0] : xs[2];
    v[15] = half == 0 ? xs[1] : 0.f;
  }
  store_row_split<16>(enc, S::ENC_LO_STRIDE, row, half * 32 + piece * 16, v, exact);
}

template <int half, int piece>
__device__ __forceinline__ void encode_motion_piece(uint8_t* smem, const Pt& pt, int row, bool exact, bool lerp) {
  using S = Sched<NET_MOTION>;
  uint8_t* enc = smem + S::enc_base + half * ABLOCK;
  const float lo_t = floorf(pt.tm), wgt = pt.tm - lo_t, omw = 1.0f - wgt;
  const float in4[4] = {pt.x, pt.y, pt.z, pt.tm};
  auto trig = [&](int f, float* dst) {
    const float fr = (float)(1 << f);
    if (!lerp) {
      const SinCos4 q = sincos_full4(in4[0] * fr, in4[1] * fr, in4[2] * fr, in4[3] * fr);
      dst[0] = q.s0; dst[1] = q.s1; dst[2] = q.s2; dst[3] = q.s3; dst[4] = q.c0; dst[5] = q.c1; dst[6] = q.c2; dst[7] = q.c3;
    } else {     // (1-w)*PE([xyz, floor t]) + w*PE([xyz, floor t + 1]) column by column (motion_net.py:63)
      const SinCos4 q = sincos_full4(in4[0] * fr, in4[1] * fr, in4[2] * fr, lo_t * fr);
      const SinCos3 q1 = sincos_full3((lo_t + 1.0f) * fr, 0.f, 0.f);
      const float s0[4] = {q.s0, q.s1, q.s2, q.s3}, c0[4] = {q.c0, q.c1, q.c2, q.c3};
      const float s1[4] = {q.s0, q.s1, q.s2, q1.s0}, c1[4] = {q.c0, q.c1, q.c2, q1.c0};
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        dst[d] = __fadd_rn(__fmul_rn(omw, s0[d]), __fmul_rn(wgt, s1[d]));
        dst[4 + d] = __fadd_rn(__fmul_rn(omw, c0[d]), __fmul_rn(wgt, c1[d]));
      }
    }
  };
  float v[16];
  trig(5 * half + 2 * piece, v);
  if (piece < 2) {
    trig(5 * half + 2 * piece + 1, v + 8);
  } else {
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      float a = 0.f;
      if (half == 0) {
        a = in4[d];
        if (lerp) {
          const float lo = d < 3 ? in4[d] : lo_t, hi = d < 3 ? in4[d] : lo_t + 1.0f;
          a = __fadd_rn(__fmul_rn(omw, lo), __fmul_rn(wgt, hi));
        }
      }
      v[8 + d] = a; v[12 + d] = 0.f;
    }
  }
  store_row_split<16>(enc, S::ENC_LO_STRIDE, row, piece * 16, v, exact);
}

// piece dispatcher (half is warp-uniform)
template <int NET, int piece>
__device__ __forceinline__ void encode_piece(uint8_t* smem, const Pt& pt, int row, int half, bool exact, bool lerp,
                                             float (&carry)[2]) {
  if (NET == NET_SPACE) {
    if (half == 0) encode_space_piece<0, piece < 2 ? piece : 1>(smem, pt, row, exact, carry);
    else encode_space_piece<1, piece < 2 ? piece : 1>(smem, pt, row, exact, carry);
  } else {
    if (half == 0) encode_motion_piece<0, piece>(smem, pt, row, exact, lerp);
    else encode_motion_piece<1, piece>(smem, pt, row, exact, lerp);
  }
}

// ---------------------------------------------------------------------------------------------------------
// coarse-pass fusion: what the two spare warps of the SpaceNet kernel run (see FuseCoarse in mlp_tc.cuh)
// ---------------------------------------------------------------------------------------------------------
// Tile `tile` holds slots 2*tile and 2*tile+1 (a slot = one hit ray of this layer, 64 coarse samples = rows 64*j .. 64*j+63);
// warp `j` composites slot 2*tile+j from the rows the epilogue warps left in `rows` (float4 per row: rgb logits, sigma).
template <int NZ>
__device__ __noinline__ void fused_composite_loop(const TcParams& P, const float* rows, float* cdf, uint32_t bar_full, uint32_t bar_empty,
                                                  long long n_tiles, int j, int lane) {
  const FuseCoarse& F = P.fuse;
  const PointSrc& src = P.src;
  const long long n_slots = src.count ? (long long)(*src.count) : src.n_slots;
  const int n1 = 64, n2 = F.n2;
  uint32_t n = 0;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++n) {
    mbar_wait(bar_full, n & 1);
    const long long slot = tile * 2 + j;
    if (slot < n_slots) {
      const long long ray = src.hit ? (long long)src.hit[slot] : slot;
      const float* tp = src.t + ray * n1;
      const float4* rp = reinterpret_cast<const float4*>(rows) + j * 64;
      float t[2], sg[2];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int k = s * 32 + lane;
        float factor;
        t[s] = __ldg(tp + k);
        sg[s] = pass_sigma(F.mask, F.layer, false, t[s], rp[k].w, factor);
      }
      const float* up = F.u ? F.u + ray * n2 : nullptr;
      const uint64_t seed = F.seed;
      const uint32_t stream = 64u + (uint32_t)F.layer;
      const unsigned long long gid = F.idmap(F.ray_base + ray);
      rs::LayerOut lo;
      rs::composite_resample_ray<2, NZ>(
          t, sg, n1, n2, F.boarder,
          [rp, lane](int s) {
            const float4 v = rp[s * 32 + lane];
            return make_float3(__fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v.x))), __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v.y))),
                               __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v.z))));
          },
          [up, seed, stream, gid](int jj) { return up ? up[jj] : philox_uniform(seed, stream, gid, (uint32_t)jj); },
          cdf, F.t_fine + ray * (n1 + n2), lane, lo, F.z_new ? F.z_new + ray * n2 : nullptr,
          F.z_new ? F.src_map + ray * (n1 + n2) : nullptr);
      rs::write_pixel(F.img, F.ray_base + ray, F.n_total, F.pixels, lo.pix, lane);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty);
  }
}

// ---------------------------------------------------------------------------------------------------------
// the kernel: one layer of a math warpgroup
// ---------------------------------------------------------------------------------------------------------
// MMAs of layer l for this warpgroup's 64 rows (A rows at byte offset a_row of every activation / encoding block), one weight
// stage per step of WSched.  A stage is handed back (one arrival per math warp on w_empty) once the MMAs that read it have
// retired: wgmma.wait_group 1 after the next stage's MMAs are issued keeps one stage of MMAs in flight.
// S::lo_in_regs: the lo halves of the activation chunks are the register fragments alo (written by epi_hidden); the encoding
// chunks keep both halves in shared memory.
template <int NET, int N, bool LOFIRST>
__device__ __forceinline__ void mma_layer(float (&acc)[128], const uint32_t (&alo)[64], int l, bool sp, uint32_t sbase,
                                          uint32_t a_row, uint32_t bars, uint32_t& cnt, int lane) {
  using S = Sched<NET>;
  using W = WSched<NET>;
  constexpr uint32_t NST = S::n_stage;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  acc_fence<N / 2>(acc);
  wgmma_fence();
  const int nact = S::act_chunks(l);
  int pend = -1;
  auto release = [&](int s) {
    __syncwarp();
    mbar_arrive_if(bars + 8u * (uint32_t)(BAR_WEMPTY + s), lane == 0);
  };
  // hi / lo halves of A chunk ch (64 k): activation chunks 0..nact-1, then the encoding chunks.  z = the activation chunk whose
  // lo half is in registers, or -1 (lo in shared memory)
  auto a_block = [&](int ch) {
    uint32_t hi, lo = 0;
    int z = -1;
    if (ch < nact) {
      hi = sbase + S::act_base + ch * ABLOCK + a_row;
      if constexpr (S::lo_in_regs) z = ch;
      else lo = hi + S::LO_STRIDE;
    } else {
      hi = sbase + S::enc_base + (ch - nact) * ABLOCK + a_row;
      lo = hi + S::ENC_LO_STRIDE;
    }
    return make_int3((int)hi, (int)lo, z);
  };
  W::template for_each_step<LOFIRST>(l, sp, a_block, [&](const int3& a, auto st) {
    const uint32_t hi = (uint32_t)a.x + 64u * st.sub, lo = (uint32_t)a.y + 64u * st.sub;
    const uint32_t s = cnt % NST, n = cnt / NST;
    mbar_wait(bars + 8u * (BAR_WFULL + s), n & 1);
    const uint32_t w = sbase + S::ring_base + s * S::stage_bytes;
    // the two k16 MMAs of this stage with A = the lo half of the sub-chunk
    auto mma_lo = [&]() {
      if (S::lo_in_regs && a.z >= 0) {
        // register fragments of 32-k sub-chunk q = 2 z + sub of the 256 activation columns: alo[8 q .. 8 q + 7].  The
        // branches are warpgroup-uniform (z and sub come from the step loop); registers are indexed by constants only.
        const int q = 2 * a.z + (int)st.sub;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (q == i) {
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) wgmma_k16_rs<N>(acc, &alo[8 * i + 4 * ks], desc_sw64(w + ks * 32));
          }
      } else {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) wgmma_k16<N>(acc, desc_sw128(lo + ks * 32), desc_sw64(w + ks * 32));
      }
    };
    if constexpr (decltype(st)::a == A_LO) {
      mma_lo();
    } else {
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) wgmma_k16<N>(acc, desc_sw128(hi + ks * 32), desc_sw64(w + ks * 32));
      if constexpr (decltype(st)::a == A_HI_LO) mma_lo();
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (pend >= 0) release(pend);
    pend = (int)s;
    ++cnt;
  });
  wgmma_wait<0>();
  acc_fence<N / 2>(acc);
  release(pend);
}

// Hidden-layer epilogue from the accumulator fragment: bias, ReLU, fp16 hi (+ lo) split into the activation blocks (rows r0 and
// r0 + 8, columns 8 j + cq, +1 for j < N / 8); SIGMA: the density head's partial dot products of the two rows.
// S::lo_in_regs: lo goes to alo[2 j] (row r0) and alo[2 j + 1] (row r0 + 8) instead.  Column groups 2 k and 2 k + 1 of the
// accumulator fragment are exactly the register A fragment of k16-slice k of the next layer, so alo[4 k .. 4 k + 3] is that
// slice's A operand as it is (wgmma_n256_rs).
template <int NET, int N, bool SIGMA>
__device__ __forceinline__ void epi_hidden(const float (&acc)[128], const float* __restrict__ bias, const float* __restrict__ wsig,
                                           uint8_t* smem, int r0, int cq, bool lo_too, float& sig0, float& sig1,
                                           uint32_t (&alo)[64]) {
  using S = Sched<NET>;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = 8 * j + cq;
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
    const float v00 = fmaxf(acc[4 * j] + b.x, 0.f), v01 = fmaxf(acc[4 * j + 1] + b.y, 0.f);
    const float v10 = fmaxf(acc[4 * j + 2] + b.x, 0.f), v11 = fmaxf(acc[4 * j + 3] + b.y, 0.f);
    if (SIGMA) {
      const float2 w = __ldg(reinterpret_cast<const float2*>(wsig + col));
      sig0 = fmaf(v00, w.x, sig0); sig0 = fmaf(v01, w.y, sig0);
      sig1 = fmaf(v10, w.x, sig1); sig1 = fmaf(v11, w.y, sig1);
    }
    uint8_t* blk = smem + S::act_base + (col >> 6) * ABLOCK;
    const uint32_t o0 = sw128_offset(r0, col & 63), o1 = sw128_offset(r0 + 8, col & 63);
    const uint32_t h0 = pack_f16x2(v00, v01), h1 = pack_f16x2(v10, v11);
    *reinterpret_cast<uint32_t*>(blk + o0) = h0;
    *reinterpret_cast<uint32_t*>(blk + o1) = h1;
    const float2 f0 = unpack_f16x2(h0), f1 = unpack_f16x2(h1);
    const uint32_t l0 = pack_f16x2(v00 - f0.x, v01 - f0.y), l1 = pack_f16x2(v10 - f1.x, v11 - f1.y);
    if constexpr (S::lo_in_regs) {
      // written whether the next layer reads them or not: a conditional write would keep the previous layer's fragments
      // alive through the epilogue next to the accumulator
      alo[2 * j] = l0;
      alo[2 * j + 1] = l1;
    } else if (lo_too) {
      *reinterpret_cast<uint32_t*>(blk + S::LO_STRIDE + o0) = l0;
      *reinterpret_cast<uint32_t*>(blk + S::LO_STRIDE + o1) = l1;
    }
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

template <int NET, bool LOFIRST>
__global__ void __launch_bounds__(NTHREADS, 1) mlp_tc_kernel(const __grid_constant__ TcParams P) {
  using S = Sched<NET>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  if ((sbase & 1023u) != 0) {                    // swizzled operands need a 1024-byte aligned base
    if (threadIdx.x == 0) printf("stnerf mlp_tc: dynamic shared memory base %u is not 1024-byte aligned\n", sbase);
    __trap();
  }
  const uint32_t bars = sbase + S::misc_base;
  auto BAR = [bars](int i) { return bars + 8u * (uint32_t)i; };
  Pt* s_rows = reinterpret_cast<Pt*>(smem + S::misc_base + MISC_ROWS);          // the current tile's points (per math warpgroup rows)
  float* s_part = reinterpret_cast<float*>(smem + S::misc_base + MISC_PART);    // [128][4]

  const int tid = threadIdx.x, lane = tid & 31;
  // warp and warpgroup indices broadcast from lane 0: the compiler then knows every role branch below is warp-uniform, and the
  // warpgroup MMAs inside them are not serialized as if they sat on a divergent path
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wgi = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const bool exact = P.exact != 0;
  // 3-term split for layer l?  (mixed mode: everything the density depends on is split, the colour-only layer is not)
  const bool single_last = P.single_last != 0;
  auto split = [&](int l) { return exact && !(single_last && l == S::N_LAYERS - 1); };
  const long long n_points = src_num_points(P.src);
  const long long n_tiles = (n_points + TILE_M - 1) / TILE_M;
  constexpr uint32_t NST = S::n_stage;
  if (tid == 0) {
    for (int i = 0; i < MAX_STAGE; ++i) { mbar_init(BAR(BAR_WFULL + i), 1); mbar_init(BAR(BAR_WEMPTY + i), N_MATH_WARPS); }
    for (int j = 0; j < 2; ++j) {
      mbar_init(BAR(BAR_RAWFULL + j), 4);          // the four warps of math warpgroup j (its 64 rows = one ray)
      mbar_init(BAR(BAR_RAWEMPTY + j), 1);         // compositing warp j
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // SpaceNet (S::lo_in_regs): the math threads hold the accumulator (128 registers) and the lo activation fragments (64), so
  // warpgroup 0 hands registers over to them.  Each role's setmaxnreg sits inside its branch, where ptxas can tell which
  // budget the code after it runs under.
  if (wgi < MATH_WG0) {
    if constexpr (S::lo_in_regs) setmaxnreg_dec<REGS_WG0>();
    if (warp == 0) {
      // =============================== weight producer: the whole warp runs the loop, one elected lane issues ===============================
      using W = WSched<NET>;
      uint32_t cnt = 0;
      for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint8_t* layer = P.wstream;
        for (int l = 0; l < S::N_LAYERS; ++l) {
          W::template for_each_step<LOFIRST>(l, split(l), [](int) { return 0; }, [&](int, auto st) {
            const uint32_t s = cnt % NST, n = cnt / NST;
            mbar_wait(BAR(BAR_WEMPTY + s), (n & 1) ^ 1);
            load_stage_elect(sbase + S::ring_base + s * S::stage_bytes, layer + st.offset, W::stage_bytes(l), BAR(BAR_WFULL + s));
            ++cnt;
          });
          layer += W::layer_bytes(l);
        }
      }
    } else if (NET == NET_SPACE && (warp == 2 || warp == 3)) {
      // =============================== compositing warps (coarse-pass fusion) ===============================
      if (P.fuse.on) {
        const int j = warp - 2;
        float* cdf = reinterpret_cast<float*>(smem + S::misc_base + MISC_CDF) + j * 64;
        if (P.fuse.n2 <= 128)
          fused_composite_loop<4>(P, s_part, cdf, BAR(BAR_RAWFULL + j), BAR(BAR_RAWEMPTY + j), n_tiles, j, lane);
        else
          fused_composite_loop<8>(P, s_part, cdf, BAR(BAR_RAWFULL + j), BAR(BAR_RAWEMPTY + j), n_tiles, j, lane);
      }
    }
  } else {
    if constexpr (S::lo_in_regs) setmaxnreg_inc<REGS_MATH>();
    // =============================== math warpgroups: encoding, MMAs, epilogues ===============================
    const int wg = wgi - MATH_WG0;                    // 0, 1: rows 64 wg .. 64 wg + 63 of every tile
    const int wt = tid & 127;
    const int erow = wg * 64 + (wt & 63), ehalf = wt >> 6;    // encoding: two threads per row, one per half of the frequencies
    const int r0 = wg * 64 + (wt >> 5) * 16 + (lane >> 2);    // accumulator fragment: rows r0, r0 + 8, columns 8 j + cq, +1
    const int cq = 2 * (lane & 3);
    const uint32_t a_row = (uint32_t)wg * 8u * 1024u;         // byte offset of the warpgroup's rows in a swizzled block
    const float* bias_all = P.aux + AUX_BIAS;
    const bool lerp = (NET == NET_MOTION) && (P.lerp_force >= 0 ? (P.lerp_force != 0) : (P.lerp_flag && *P.lerp_flag != 0));
    const bool fused = (NET == NET_SPACE) && P.fuse.on;
    uint32_t cnt = 0, tile_no = 0;
    float acc[128];
    uint32_t alo[64];                                  // S::lo_in_regs: lo activations of the last hidden layer (epi_hidden)
#pragma unroll
    for (int i = 0; i < 64; ++i) alo[i] = 0u;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_no) {
      // the previous tile's MMAs have retired in every warp of the warpgroup and its rows are written out: its blocks are free
      wg_bar_sync(wg);
      const Pt cur = fetch_pt(P.src, tile * TILE_M + erow, n_points);
      if (ehalf == 0) s_rows[erow] = cur;
      float carry[2] = {0.f, 0.f};
      if (NET == NET_MOTION) {
        // zero padding of the MotionNet encoding blocks (chunks 6.. of block 0, 5.. of block 1): the activations overwrite them
        uint8_t* enc = smem + S::enc_base + ehalf * ABLOCK;
        for (int c = (ehalf == 0 ? 48 : 40); c < 64; c += 8) {
          const uint32_t off = sw128_offset(erow, c);
          *reinterpret_cast<uint4*>(enc + off) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(enc + S::ENC_LO_STRIDE + off) = make_uint4(0, 0, 0, 0);
        }
      }
      encode_piece<NET, 0>(smem, cur, erow, ehalf, exact, lerp, carry);
      encode_piece<NET, 1>(smem, cur, erow, ehalf, exact, lerp, carry);
      if (NET == NET_MOTION) encode_piece<NET, 2>(smem, cur, erow, ehalf, exact, lerp, carry);
      float sig0 = 0.f, sig1 = 0.f;
      for (int l = 0; l < S::N_LAYERS; ++l) {
        // the A operand of this layer (encoding / previous epilogue) is written by every thread of the warpgroup
        fence_proxy_async();
        wg_bar_sync(wg);
        const bool last = (l == S::N_LAYERS - 1);
        if (!last) {
          mma_layer<NET, (NET == NET_SPACE ? 256 : 128), LOFIRST>(acc, alo, l, split(l), sbase, a_row, bars, cnt, lane);
          if (NET == NET_SPACE && l == 6)
            epi_hidden<NET, 256, true>(acc, bias_all + l * 256, P.aux + AUX_WSIG, smem, r0, cq, split(l + 1), sig0, sig1, alo);
          else
            epi_hidden<NET, (NET == NET_SPACE ? 256 : 128), false>(acc, bias_all + l * 256, nullptr, smem, r0, cq, split(l + 1), sig0,
                                                                  sig1, alo);
          continue;
        }
        // last layer: 128 features -> 3-wide head in fp32 (rgb_net.3 / motion_net.10).
        // SpaceNet: the bias is the per-ray vector of head_bias_kernel (dir/time part of rgb_net.1 + b1).
        mma_layer<NET, 128, LOFIRST>(acc, alo, l, split(l), sbase, a_row, bars, cnt, lane);
        const Pt p0 = s_rows[r0], p1 = s_rows[r0 + 8];
        const float* b0 = (NET == NET_SPACE) ? (P.cbuf + (size_t)p0.cidx * 128) : bias_all + l * 256;
        const float* b1 = (NET == NET_SPACE) ? (P.cbuf + (size_t)p1.cidx * 128) : bias_all + l * 256;
        float d0[3] = {0.f, 0.f, 0.f}, d1[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = 8 * j + cq;
          const float2 ba = __ldg(reinterpret_cast<const float2*>(b0 + col));
          const float2 bb = __ldg(reinterpret_cast<const float2*>(b1 + col));
          const float v00 = fmaxf(acc[4 * j] + ba.x, 0.f), v01 = fmaxf(acc[4 * j + 1] + ba.y, 0.f);
          const float v10 = fmaxf(acc[4 * j + 2] + bb.x, 0.f), v11 = fmaxf(acc[4 * j + 3] + bb.y, 0.f);
#pragma unroll
          for (int o = 0; o < 3; ++o) {
            const float2 w = __ldg(reinterpret_cast<const float2*>(P.aux + AUX_WOUT + o * 128 + col));
            d0[o] = fmaf(v00, w.x, d0[o]); d0[o] = fmaf(v01, w.y, d0[o]);
            d1[o] = fmaf(v10, w.x, d1[o]); d1[o] = fmaf(v11, w.y, d1[o]);
          }
        }
#pragma unroll
        for (int o = 0; o < 3; ++o) { d0[o] = quad_sum(d0[o]) + P.aux[AUX_BOUT + o]; d1[o] = quad_sum(d1[o]) + P.aux[AUX_BOUT + o]; }
        if (NET == NET_SPACE) { sig0 = quad_sum(sig0) + P.aux[AUX_BSIG]; sig1 = quad_sum(sig1) + P.aux[AUX_BSIG]; }
        if (fused) {
          // the compositing warp of these rows must be done with the previous tile's (it has had a whole tile period)
          if (tile_no > 0) mbar_wait(BAR(BAR_RAWEMPTY + wg), (tile_no - 1) & 1);
          if ((lane & 3) == 0) {
            reinterpret_cast<float4*>(s_part)[r0] = make_float4(d0[0], d0[1], d0[2], sig0);
            reinterpret_cast<float4*>(s_part)[r0 + 8] = make_float4(d1[0], d1[1], d1[2], sig1);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(BAR(BAR_RAWFULL + wg));
        }
        if ((lane & 3) == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const Pt& p = h ? p1 : p0;
            const float* o = h ? d1 : d0;
            const float sg = h ? sig1 : sig0;
            if (p.out_index < 0) continue;
            const int oi = p.out_index;
            if (NET == NET_SPACE) {
              if (P.raw) reinterpret_cast<float4*>(P.raw)[oi] = make_float4(o[0], o[1], o[2], sg);
              if (P.rgb_out) { P.rgb_out[3 * (size_t)oi] = o[0]; P.rgb_out[3 * (size_t)oi + 1] = o[1]; P.rgb_out[3 * (size_t)oi + 2] = o[2]; }
              if (P.sigma_out) P.sigma_out[oi] = sg;
            } else {
              const long long pidx = tile * TILE_M + r0 + 8 * h;     // compact point index
              if (P.flow_out) { P.flow_out[3 * pidx] = o[0]; P.flow_out[3 * pidx + 1] = o[1]; P.flow_out[3 * pidx + 2] = o[2]; }
              if (P.xyz_out) {                                       // layered_rfrender.py:356 / :510
                P.xyz_out[3 * pidx] = __fadd_rn(p.x, o[0]);
                P.xyz_out[3 * pidx + 1] = __fadd_rn(p.y, o[1]);
                P.xyz_out[3 * pidx + 2] = __fadd_rn(p.z, o[2]);
              }
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// per-slot bias of rgb_net.1: c[slot][n] = b1[n] + sum_k W1[n][256+k] * relu(enc_k(dir, time))   (fp32)
// (modeling/spacenet.py:141-152 with the leading ReLU of rgb_net, :82; enc = [PE(dir, L=4) (27) | PE(time, L=10) (21)])
// ---------------------------------------------------------------------------------------------------------
constexpr int HB_SLOTS = 8;
__global__ void __launch_bounds__(128) head_bias_kernel(PointSrc src, const float* __restrict__ w_tail /*[48][128]*/,
                                                        const float* __restrict__ b1, int use_time,
                                                        float* __restrict__ cbuf) {
  __shared__ float s_enc[HB_SLOTS][48];
  const long long n_slots = src.count ? (long long)(*src.count) : src.n_slots;
  const int nk = PE_DIR + (use_time ? PE_TIME : 0);
  const int tid = threadIdx.x;
  float w[48];
#pragma unroll
  for (int k = 0; k < 48; ++k) w[k] = (k < nk) ? __ldg(w_tail + k * 128 + tid) : 0.f;
  const float bias = __ldg(b1 + tid);
  for (long long s0 = (long long)blockIdx.x * HB_SLOTS; s0 < n_slots; s0 += (long long)gridDim.x * HB_SLOTS) {
    __syncthreads();
    // thread (sl, j): encoding entry j of slot s0+sl
    for (int e = tid; e < HB_SLOTS * 48; e += 128) {
      const int sl = e / 48, j = e - sl * 48;
      const long long slot = s0 + sl;
      float v = 0.f;
      if (slot < n_slots && j < nk) {
        float d[3], tm;
        if (src.mode == SRC_EXPLICIT) {
          d[0] = src.dirs[3 * slot]; d[1] = src.dirs[3 * slot + 1]; d[2] = src.dirs[3 * slot + 2];
          tm = src.times ? src.times[slot * src.time_stride] : 0.f;
        } else {
          const long long ray = src.hit ? (long long)src.hit[slot] : slot;
          const float* rp = src.rays + ray * src.ray_stride;
          d[0] = rp[3]; d[1] = rp[4]; d[2] = rp[5];
          tm = rp[6 + src.layer];
        }
        if (j < PE_DIR) {
          if (j < 3) v = d[j];
          else {
            const int r = j - 3, f = r / 6, m = r - 6 * f;        // [sin xyz | cos xyz] per frequency
            const float a = d[m % 3] * (float)(1 << f);
            v = (m < 3) ? sinf(a) : cosf(a);
          }
        } else {
          const int r = j - PE_DIR;
          if (r == 0) v = tm;
          else {
            const int f = (r - 1) >> 1;
            const float a = tm * (float)(1 << f);
            v = ((r - 1) & 1) ? cosf(a) : sinf(a);
          }
        }
        v = fmaxf(v, 0.f);
      }
      s_enc[sl][j] = v;
    }
    __syncthreads();
#pragma unroll
    for (int sl = 0; sl < HB_SLOTS; ++sl) {
      const long long slot = s0 + sl;
      if (slot >= n_slots) break;
      float acc = bias;
#pragma unroll
      for (int k = 0; k < 48; ++k) acc = fmaf(w[k], s_enc[sl][k], acc);
      cbuf[slot * 128 + tid] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// self-test: D (128 x 256) = A (128 x 64) * B^T (256 x 64) in fp16 through exactly the descriptors / swizzles / bulk copy /
// accumulator fragment of the kernel above (two math warpgroups of 64 rows each)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 1) wgmma_selftest_kernel(const float* __restrict__ A, const uint8_t* __restrict__ Bstages,
                                                               float* __restrict__ D, int reps) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar = sbase + ABLOCK + 2 * STAGE_BYTES;
  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, lane = tid & 31;
  if ((sbase & 1023u) != 0) __trap();
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < 128) {                               // A: row `tid`, 64 columns, written with the encoder's store path (hi only)
    for (int c0 = 0; c0 < 64; c0 += 32) {
      float v[32];
      for (int i = 0; i < 32; ++i) v[i] = A[tid * 64 + c0 + i];
      store_row_split<32>(smem, 0, tid, c0, v, false);
    }
  }
  fence_proxy_async();
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar, 2 * STAGE_BYTES);        // two 32-wide k sub-chunks
    bulk_g2s(sbase + ABLOCK, Bstages, 2 * STAGE_BYTES, bar);
  }
  mbar_wait(bar, 0);
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  acc_fence<128>(acc);
  wgmma_fence();
  for (int rep = 0; rep < reps; ++rep) {         // reps > 1: the same product accumulated again and again (accumulation probe)
#pragma unroll
    for (int sub = 0; sub < 2; ++sub)
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
        wgmma_n256(acc, desc_sw128(sbase + (uint32_t)wg * 8192u + sub * 64 + ks * 32),
                   desc_sw64(sbase + ABLOCK + sub * STAGE_BYTES + ks * 32));
    wgmma_commit();
    wgmma_wait<0>();
  }
  acc_fence<128>(acc);
  const int r0 = wg * 64 + (wt >> 5) * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int col = 8 * j + cq;
    D[r0 * 256 + col] = acc[4 * j];
    D[r0 * 256 + col + 1] = acc[4 * j + 1];
    D[(r0 + 8) * 256 + col] = acc[4 * j + 2];
    D[(r0 + 8) * 256 + col + 1] = acc[4 * j + 3];
  }
}

// ---------------------------------------------------------------------------------------------------------
// host: weight packing
// ---------------------------------------------------------------------------------------------------------
// One layer of the stream.  W is (N, K_total) row-major.  A 64-wide k-chunk is described by the 64 source columns it
// multiplies (-1 = zero padding), in the column order the device writes its A operand; `chunks` is indexed by chunk id
// (activation chunks, then encoding chunks), the stream takes them in WSched::chunk_at order.
struct LayerSpec { const float* W; int N, K_total; std::vector<std::vector<int>> chunks; };

std::vector<int> iota_chunk(int k0, int kend) {
  std::vector<int> c(64, -1);
  for (int i = 0; i < 64 && k0 + i < kend; ++i) c[i] = k0 + i;
  return c;
}
// encoding-buffer column -> reference PE column (see encode_space_piece / encode_motion_piece).
// Reference order (utils/dimension_kernel.py:24-33): raw (d), then per frequency f: sin (d values), cos (d values).
std::vector<int> enc_perm_space(int base) {
  std::vector<int> c(64, -1);
  for (int h = 0; h < 2; ++h) {
    for (int ff = 0; ff < 5; ++ff)
      for (int j = 0; j < 6; ++j) c[h * 32 + 6 * ff + j] = base + 3 + 6 * (5 * h + ff) + j;
    if (h == 0) { c[30] = base + 0; c[31] = base + 1; } else { c[62] = base + 2; }
  }
  return c;
}
std::vector<std::vector<int>> enc_perm_motion() {
  std::vector<std::vector<int>> out(2, std::vector<int>(64, -1));
  for (int h = 0; h < 2; ++h)
    for (int ff = 0; ff < 5; ++ff)
      for (int j = 0; j < 8; ++j) out[h][8 * ff + j] = 4 + 8 * (5 * h + ff) + j;
  for (int d = 0; d < 4; ++d) out[0][40 + d] = d;
  return out;
}

template <int NET>
int pack_stream(TcNet& net, const std::vector<LayerSpec>& layers, const std::vector<float>& aux) {
  std::vector<uint8_t> stream;
  for (int l = 0; l < (int)layers.size(); ++l) {
    const LayerSpec& L = layers[l];
    const size_t stage = (size_t)L.N * 64;
    for (int c = 0; c < (int)L.chunks.size(); ++c) {
      const std::vector<int>& ch = L.chunks[WSched<NET>::chunk_at(l, c)];
      for (int sub = 0; sub < 2; ++sub) {
        std::vector<uint8_t> hi(stage, 0), lo(stage, 0);
        for (int n = 0; n < L.N; ++n)
          for (int c = 0; c < 32; ++c) {
            const int k = ch[sub * 32 + c];
            if (k < 0) continue;
            const float w = L.W[(size_t)n * L.K_total + k];
            const __half h = __float2half_rn(w);
            const __half l = __float2half_rn(w - __half2float(h));
            const uint32_t off = sw64_offset(n, c);
            memcpy(hi.data() + off, &h, 2);
            memcpy(lo.data() + off, &l, 2);
          }
        stream.insert(stream.end(), hi.begin(), hi.end());
        stream.insert(stream.end(), lo.begin(), lo.end());
      }
    }
  }
  if (stream.size() != stream_bytes_per_tile<NET>()) return STNERF_EINVAL;
  tc_free(net);
  net.blob_bytes = stream.size();
  STNERF_CUDA(cudaMalloc(&net.blob, stream.size()));
  STNERF_CUDA(cudaMemcpy(net.blob, stream.data(), stream.size(), cudaMemcpyHostToDevice));
  STNERF_CUDA(cudaMalloc((void**)&net.aux, aux.size() * sizeof(float)));
  STNERF_CUDA(cudaMemcpy(net.aux, aux.data(), aux.size() * sizeof(float), cudaMemcpyHostToDevice));
  return STNERF_OK;
}

}  // namespace

void tc_free(TcNet& net) {
  if (net.blob) cudaFree(net.blob);
  if (net.aux) cudaFree(net.aux);
  if (net.w_tail) cudaFree(net.w_tail);
  net.blob = nullptr; net.aux = nullptr; net.w_tail = nullptr; net.blob_bytes = 0;
}

size_t tc_stream_bytes(bool is_space) { return is_space ? stream_bytes_per_tile<NET_SPACE>() : stream_bytes_per_tile<NET_MOTION>(); }
size_t tc_aux_floats() { return AUX_FLOATS; }
size_t tc_tail_floats(bool is_space) { return is_space ? 48 * 128 : 0; }

int tc_export(const TcNet& net, bool is_space, uint8_t* stream_host, float* aux_host, float* tail_host) {
  if (!net.blob || !net.aux || net.blob_bytes != tc_stream_bytes(is_space) || (is_space && !net.w_tail)) return STNERF_ENOWEIGHTS;
  STNERF_CUDA(cudaMemcpy(stream_host, net.blob, net.blob_bytes, cudaMemcpyDeviceToHost));
  STNERF_CUDA(cudaMemcpy(aux_host, net.aux, AUX_FLOATS * sizeof(float), cudaMemcpyDeviceToHost));
  if (is_space) STNERF_CUDA(cudaMemcpy(tail_host, net.w_tail, tc_tail_floats(true) * sizeof(float), cudaMemcpyDeviceToHost));
  return STNERF_OK;
}

int tc_import(TcNet& net, bool is_space, int use_time, const uint8_t* stream_host, const float* aux_host, const float* tail_host) {
  tc_free(net);
  net.blob_bytes = tc_stream_bytes(is_space);
  net.use_time = use_time;
  STNERF_CUDA(cudaMalloc(&net.blob, net.blob_bytes));
  STNERF_CUDA(cudaMemcpy(net.blob, stream_host, net.blob_bytes, cudaMemcpyHostToDevice));
  STNERF_CUDA(cudaMalloc((void**)&net.aux, AUX_FLOATS * sizeof(float)));
  STNERF_CUDA(cudaMemcpy(net.aux, aux_host, AUX_FLOATS * sizeof(float), cudaMemcpyHostToDevice));
  if (is_space) {
    STNERF_CUDA(cudaMalloc((void**)&net.w_tail, tc_tail_floats(true) * sizeof(float)));
    STNERF_CUDA(cudaMemcpy(net.w_tail, tail_host, tc_tail_floats(true) * sizeof(float), cudaMemcpyHostToDevice));
  }
  return STNERF_OK;
}

int tc_pack_spacenet(TcNet& net, const float* p, bool use_time) {
  const int krgb = HID + PE_DIR + (use_time ? PE_TIME : 0);
  std::vector<float> aux(AUX_FLOATS, 0.f);
  std::vector<LayerSpec> layers;
  const int Ks[7] = {PE_POS, HID, HID, HID, HID + PE_POS, HID, HID};
  for (int i = 0; i < 7; ++i) {
    LayerSpec L;
    L.W = p; L.N = HID; L.K_total = Ks[i];
    if (i != 0) for (int k = 0; k < HID; k += 64) L.chunks.push_back(iota_chunk(k, HID));
    if (i == 0 || i == 4) L.chunks.push_back(enc_perm_space(i == 0 ? 0 : HID));   // layer 4: cat[x, PE(pos)] (spacenet.py:137)
    layers.push_back(L);
    p += (size_t)HID * Ks[i];
    memcpy(aux.data() + AUX_BIAS + i * 256, p, HID * sizeof(float));
    p += HID;
  }
  memcpy(aux.data() + AUX_WSIG, p, HID * sizeof(float)); p += HID;
  aux[AUX_BSIG] = *p++;
  LayerSpec L;                                                      // rgb_net.1: only the x part goes through the GEMM
  L.W = p; L.N = HEAD; L.K_total = krgb;
  for (int k = 0; k < HID; k += 64) L.chunks.push_back(iota_chunk(k, HID));
  layers.push_back(L);
  // dir/time tail of rgb_net.1, transposed [48][128] fp32, for head_bias_kernel
  std::vector<float> tail(48 * 128, 0.f);
  for (int n = 0; n < HEAD; ++n)
    for (int k = 0; k < krgb - HID; ++k) tail[(size_t)k * 128 + n] = p[(size_t)n * krgb + HID + k];
  p += (size_t)HEAD * krgb;
  memcpy(aux.data() + AUX_BIAS + 7 * 256, p, HEAD * sizeof(float)); p += HEAD;
  memcpy(aux.data() + AUX_WOUT, p, 3 * HEAD * sizeof(float)); p += 3 * HEAD;
  memcpy(aux.data() + AUX_BOUT, p, 3 * sizeof(float));
  net.use_time = use_time ? 1 : 0;
  const int rc = pack_stream<NET_SPACE>(net, layers, aux);
  if (rc) return rc;
  STNERF_CUDA(cudaMalloc((void**)&net.w_tail, tail.size() * sizeof(float)));
  STNERF_CUDA(cudaMemcpy(net.w_tail, tail.data(), tail.size() * sizeof(float), cudaMemcpyHostToDevice));
  return STNERF_OK;
}

int tc_pack_motionnet(TcNet& net, const float* p) {
  std::vector<float> aux(AUX_FLOATS, 0.f);
  std::vector<LayerSpec> layers;
  for (int i = 0; i < 5; ++i) {
    LayerSpec L;
    const int K = i == 0 ? PE_MOTION : HEAD;
    L.W = p; L.N = HEAD; L.K_total = K;
    if (i == 0) L.chunks = enc_perm_motion();                       // PE(84) in two 64-wide chunks (zero padded)
    else for (int k = 0; k < HEAD; k += 64) L.chunks.push_back(iota_chunk(k, HEAD));
    layers.push_back(L);
    p += (size_t)HEAD * K;
    memcpy(aux.data() + AUX_BIAS + i * 256, p, HEAD * sizeof(float));
    p += HEAD;
  }
  memcpy(aux.data() + AUX_WOUT, p, 3 * HEAD * sizeof(float)); p += 3 * HEAD;
  memcpy(aux.data() + AUX_BOUT, p, 3 * sizeof(float));
  return pack_stream<NET_MOTION>(net, layers, aux);
}


// D = A * B^T for random A (128x64, rounded to fp16), B (256x64) through the tensor-core path; max |D - reference|.
// reps > 1 (accumulation probe): all-positive operands, the product accumulated `reps` times into the same register accumulator
// (4*reps MMAs of K=16); reports the max and the MEAN SIGNED relative error against the fp64 sum -- a negative mean that grows
// with reps is the signature of round-toward-zero accumulation inside the tensor core.
int tc_selftest_accum(int reps, float* max_err_host, float* mean_signed_rel_host) {
  if (reps < 1) return STNERF_EINVAL;
  std::vector<float> Af(128 * 64), Bf(256 * 64);
  uint32_t s = 12345u;
  const bool probe = reps > 1;
  auto rnd = [&s, probe]() { s = s * 1664525u + 1013904223u; const float v = ((s >> 8) & 0xFFFF) / 65536.0f; return probe ? 0.5f + 0.5f * v : v - 0.5f; };
  for (auto& v : Af) v = __half2float(__float2half_rn(rnd()));
  for (auto& v : Bf) v = __half2float(__float2half_rn(rnd()));
  std::vector<uint8_t> stages(2 * STAGE_BYTES, 0);
  for (int sub = 0; sub < 2; ++sub)
    for (int n = 0; n < 256; ++n)
      for (int c = 0; c < 32; ++c) {
        const __half h = __float2half_rn(Bf[n * 64 + sub * 32 + c]);
        memcpy(stages.data() + sub * STAGE_BYTES + sw64_offset(n, c), &h, 2);
      }
  float *dA = nullptr, *dD = nullptr; uint8_t* dB = nullptr;
  STNERF_CUDA(cudaMalloc((void**)&dA, Af.size() * 4));
  STNERF_CUDA(cudaMalloc((void**)&dB, stages.size()));
  STNERF_CUDA(cudaMalloc((void**)&dD, 128 * 256 * 4));
  STNERF_CUDA(cudaMemcpy(dA, Af.data(), Af.size() * 4, cudaMemcpyHostToDevice));
  STNERF_CUDA(cudaMemcpy(dB, stages.data(), stages.size(), cudaMemcpyHostToDevice));
  const int smem = ABLOCK + 2 * STAGE_BYTES + 64;
  STNERF_CUDA(cudaFuncSetAttribute(wgmma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  wgmma_selftest_kernel<<<1, 256, smem>>>(dA, dB, dD, reps);
  STNERF_LAUNCH_CHECK();
  STNERF_CUDA(cudaDeviceSynchronize());
  std::vector<float> D(128 * 256);
  STNERF_CUDA(cudaMemcpy(D.data(), dD, D.size() * 4, cudaMemcpyDeviceToHost));
  cudaFree(dA); cudaFree(dB); cudaFree(dD);
  float worst = 0.f;
  double signed_rel = 0.0;
  for (int m = 0; m < 128; ++m)
    for (int n = 0; n < 256; ++n) {
      double ref = 0;
      for (int k = 0; k < 64; ++k) ref += (double)Af[m * 64 + k] * Bf[n * 64 + k];
      ref *= reps;
      worst = fmaxf(worst, fabsf((float)(ref - (double)D[m * 256 + n])));
      if (ref != 0.0) signed_rel += ((double)D[m * 256 + n] - ref) / fabs(ref);
    }
  *max_err_host = worst;
  if (mean_signed_rel_host) *mean_signed_rel_host = (float)(signed_rel / (128.0 * 256.0));
  return STNERF_OK;
}
int tc_selftest(float* max_err_host) { return tc_selftest_accum(1, max_err_host, nullptr); }

template <int NET, bool LOFIRST>
static int launch_tc_variant(const TcParams& P, int num_sms, cudaStream_t st) {
  // per-device attribute, set on every launch (one process may drive several devices; cost: microseconds)
  using S = Sched<NET>;
  auto kern = mlp_tc_kernel<NET, LOFIRST>;
  STNERF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::smem_total));
  kern<<<num_sms, NTHREADS, S::smem_total, st>>>(P);
  STNERF_LAUNCH_CHECK();
  return STNERF_OK;
}

template <int NET>
static int launch_tc(const TcParams& P, int num_sms, cudaStream_t st) {
  return P.lo_first ? launch_tc_variant<NET, true>(P, num_sms, st) : launch_tc_variant<NET, false>(P, num_sms, st);
}

bool tc_can_fuse_coarse(int n1, int n2) { return n1 == 64 && n2 >= 1 && n2 <= 256; }

int tc_launch_spacenet(const PointSrc& src, const TcNet& net, int precision, float* cbuf, float* raw,
                       float* rgb_out, float* sigma_out, int num_sms, cudaStream_t st, const FuseCoarse* fuse, bool fine_pass) {
  if (!net.blob || !net.w_tail) return STNERF_ENOWEIGHTS;
  if (!cbuf) return STNERF_EINVAL;
  // per-slot bias of rgb_net.1 (dir/time part), then the fused MLP
  PointSrc hs = src;
  if (src.mode == SRC_EXPLICIT) hs.count = nullptr;
  const long long slots_hint = src.count ? src.n_slots_cap : src.n_slots;
  long long blocks = (slots_hint + HB_SLOTS - 1) / HB_SLOTS;
  if (blocks < 1) blocks = 1;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  head_bias_kernel<<<(int)blocks, 128, 0, st>>>(hs, net.w_tail, net.aux + AUX_BIAS + 7 * 256, net.use_time, cbuf);
  STNERF_LAUNCH_CHECK();
  TcParams P;
  memset(&P, 0, sizeof(P));
  P.src = src; P.wstream = (const uint8_t*)net.blob; P.aux = net.aux; P.cbuf = cbuf;
  P.exact = precision == STNERF_PREC_TC_3XF16 || precision == STNERF_PREC_TC_MIXED || precision == STNERF_PREC_TC_3XF16_CF;
  P.single_last = precision == STNERF_PREC_TC_MIXED;
  P.raw = raw; P.rgb_out = rgb_out; P.sigma_out = sigma_out; P.lerp_force = 0;
  // exact_cf adds the corrections first where the sample placement and the positions depend on the result: the coarse pass and
  // the MotionNets (and the unit entry points).  The fine SpaceNet pass keeps the interleaved order, which streams every stage once.
  P.lo_first = precision == STNERF_PREC_TC_3XF16_CF && !fine_pass;
  if (fuse && fuse->on) {
    if (src.mode == SRC_EXPLICIT || src.S != 64 || !tc_can_fuse_coarse(fuse->n1, fuse->n2) || !fuse->t_fine) return STNERF_EINVAL;
    P.fuse = *fuse;
  }
  return launch_tc<NET_SPACE>(P, num_sms, st);
}

int tc_launch_motionnet(const PointSrc& src, const TcNet& net, int precision, const int* lerp_flag_dev,
                        int lerp_force, float* xyz_out, float* flow_out, int num_sms, cudaStream_t st) {
  if (!net.blob) return STNERF_ENOWEIGHTS;
  TcParams P;
  memset(&P, 0, sizeof(P));
  P.src = src; P.wstream = (const uint8_t*)net.blob; P.aux = net.aux;
  P.exact = precision == STNERF_PREC_TC_3XF16 || precision == STNERF_PREC_TC_MIXED || precision == STNERF_PREC_TC_3XF16_CF;      // the flow feeds positions: always split
  P.xyz_out = xyz_out; P.flow_out = flow_out; P.lerp_flag = lerp_flag_dev; P.lerp_force = lerp_force;
  P.lo_first = precision == STNERF_PREC_TC_3XF16_CF;
  return launch_tc<NET_MOTION>(P, num_sms, st);
}

}  // namespace stnerf
