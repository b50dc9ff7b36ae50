// Shared declarations of libstnerf_b200 (device structs, error plumbing, Philox).
#pragma once
#include <atomic>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/stnerf.h"

namespace stnerf {

// ---------------------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------------------
extern thread_local char g_cuda_err[512];
extern std::atomic<unsigned long long> g_launches;    // kernels launched by this library (contexts may live on several host threads)

#define STNERF_CUDA(expr)                                                                        \
  do {                                                                                           \
    cudaError_t e_ = (expr);                                                                     \
    if (e_ != cudaSuccess) {                                                                     \
      snprintf(stnerf::g_cuda_err, sizeof(stnerf::g_cuda_err), "%s:%d %s -> %s", __FILE__, __LINE__, #expr, \
               cudaGetErrorString(e_));                                                          \
      return STNERF_ECUDA;                                                                       \
    }                                                                                            \
  } while (0)

#define STNERF_LAUNCH_CHECK()                                                                    \
  do {                                                                                           \
    ++stnerf::g_launches;                                                                        \
    STNERF_CUDA(cudaGetLastError());                                                             \
  } while (0)

// ---------------------------------------------------------------------------------------------------------
// network dimensions (SURVEY App. B)
// ---------------------------------------------------------------------------------------------------------
constexpr int PE_POS = 63;      // 3 + 3*2*10   utils/dimension_kernel.py, modeling/spacenet.py:20
constexpr int PE_DIR = 27;      // 3 + 3*2*4
constexpr int PE_TIME = 21;     // 1 + 2*10
constexpr int PE_MOTION = 84;   // 4 + 4*2*10   modeling/motion_net.py:14
constexpr int HID = 256;        // SpaceNet backbone
constexpr int HEAD = 128;       // SpaceNet rgb head / MotionNet width
constexpr int SPACENET_FLOATS_NOTIME = 464260;
constexpr int SPACENET_FLOATS_TIME = 466948;
constexpr int MOTIONNET_FLOATS = 77315;

// fp32 weights of one SpaceNet, repacked K-major-transposed ([k][n], n contiguous) for the SIMT kernels.
struct SpaceNetW {
  const float* w[7];     // stage1.{0,2,4,6} (K=63,256,256,256), stage2.{0,2,4} (K=319,256,256), each [K][256]
  const float* b[7];     // [256]
  const float* w_sigma;  // [256]
  float b_sigma;
  const float* w_rgbh;   // [256+27(+21)][128]
  const float* b_rgbh;   // [128]
  const float* w_rgbo;   // [3][128] (row-major as in the checkpoint)
  float b_rgbo[3];
  int use_time;
};

struct MotionNetW {
  const float* w[5];     // [84][128], 4 x [128][128]
  const float* b[5];
  const float* w_out;    // [3][128]
  float b_out[3];
};

// Where a tile of points comes from.
enum { SRC_EXPLICIT = 0, SRC_MARCH = 1, SRC_XYZ = 2, SRC_XYZ_MAP = 3 };
struct PointSrc {
  int mode;
  // SRC_EXPLICIT: per-point arrays (unit entry points)
  const float* pos;          // (P,3)  | SRC_XYZ: compact (slot*S+k, 3) deformed positions
  const float* dirs;         // (P,3)
  const float* times;        // (P) or null
  int pos_stride, time_stride;   // SRC_EXPLICIT element strides (3 / 1 unless the inputs are interleaved)
  // SRC_MARCH / SRC_XYZ: points = (slot, k), ray = hit ? hit[slot] : slot
  const float* rays;         // (n, ray_stride): o, d, frame ids
  int ray_stride;
  // SRC_XYZ_MAP (fine pass with flow reuse): position k of a slot's S depths came from coarse sample m = src_map[ray*S + k] < n_first
  // (deformed position pos[(slot*n_first + m)*3]) or from new depth m - n_first (pos2[(slot*(S - n_first) + m - n_first)*3])
  const uint8_t* src_map;
  const float* pos2;
  int n_first;
  const int* hit;            // slot -> ray, or null (identity: background)
  const int* count;          // device-side number of slots, or null
  long long n_slots;         // slots when count == null; P for SRC_EXPLICIT (with S == 1)
  long long n_slots_cap;     // upper bound on *count (grid sizing of per-slot helper kernels)
  const float* t;            // (rays, S) depths of this layer
  int S;
  int layer;                 // frame id column = 6 + layer
  // inverse edit on marched points (layered_rfrender.py:293-303 / :467-475)
  int shift_on, scale_on;
  float shift[3], scale, pivot[3];
};

// The inverse edit of one layer and pass on a point (layered_rfrender.py:293-303 / :467-475), every op rounded on its own.
// E is PointSrc or FieldEdit: any struct with the flat fields shift_on, scale_on, shift[3], scale, pivot[3].
template <class E>
__device__ __forceinline__ void inverse_edit(const E& e, float v[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (e.shift_on) v[a] = __fsub_rn(v[a], e.shift[a]);                                        // :298 / :471
    if (e.scale_on) v[a] = __fadd_rn(__fdiv_rn(__fsub_rn(v[a], e.pivot[a]), e.scale), e.pivot[a]);   // :303 / :475
  }
}

// A marched sample p = t*d + o with separately rounded product and sum (layers/RaySamplePoint.py:103,
// layered_rfrender.py:465), then the inverse edit of the pass.  rp = the ray (o at 0..2), d = its direction.  Shared by both
// networks' SRC_MARCH fetch and the training point assembly, so all of them round alike.
__device__ __forceinline__ void march_point(const PointSrc& s, const float* rp, float tt, float dx, float dy, float dz,
                                            float v[3]) {
  v[0] = __fadd_rn(__fmul_rn(tt, dx), rp[0]);
  v[1] = __fadd_rn(__fmul_rn(tt, dy), rp[1]);
  v[2] = __fadd_rn(__fmul_rn(tt, dz), rp[2]);
  inverse_edit(s, v);
}

__device__ __forceinline__ long long src_num_points(const PointSrc& s) {
  long long slots = s.count ? (long long)(*s.count) : s.n_slots;
  return slots * (long long)s.S;
}

// The rotation edit of one layer (stnerf_set_rotation): Rt = R^T row-major, about centre c.  A rotated layer's ray is
// o' = c + R^T (o - c), d' = R^T d, each product and sum rounded on its own in this order (include/stnerf.h), so a host
// restatement in fp32 gives the same bits.  The same map takes a world point of the field (extract.cu) back into the layer.
struct RayRot {
  float Rt[9], c[3];
};
__device__ __forceinline__ void rotate_back_point(const RayRot& r, const float p[3], float out[3]) {
  const float q0 = __fsub_rn(p[0], r.c[0]), q1 = __fsub_rn(p[1], r.c[1]), q2 = __fsub_rn(p[2], r.c[2]);
#pragma unroll
  for (int a = 0; a < 3; ++a)
    out[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r.Rt[3 * a], q0), __fmul_rn(r.Rt[3 * a + 1], q1)), __fmul_rn(r.Rt[3 * a + 2], q2)),
                       r.c[a]);
}
__device__ __forceinline__ void rotate_back_dir(const RayRot& r, const float d[3], float out[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a)
    out[a] = __fadd_rn(__fadd_rn(__fmul_rn(r.Rt[3 * a], d[0]), __fmul_rn(r.Rt[3 * a + 1], d[1])), __fmul_rn(r.Rt[3 * a + 2], d[2]));
}

// The rays each layer samples along: p[i] = the caller's rays, or layer i's rotated copy (same stride, same frame ids).
struct LayerRays {
  const float* p[STNERF_MAX_LAYERS];
};

// Maps a ray's index within a call to the id that keys the Philox stream (identity by default).  A caller that renders
// an image in row-interleaved shards sets (base, width, row_stride) so every pixel draws the same uniforms as in an
// unsharded render:  id = base + (j / width) * row_stride + (j % width).
struct RayIdMap {
  long long base, row_stride;
  int width;
  __host__ __device__ unsigned long long operator()(long long j) const {
    return width > 0 ? (unsigned long long)(base + (j / width) * row_stride + (j % width)) : (unsigned long long)(base + j);
  }
};

// Scene constants as the kernels see them.
struct DevScene {
  float bmin[STNERF_MAX_LAYERS][3];
  float bmax[STNERF_MAX_LAYERS][3];
  int shown[STNERF_MAX_LAYERS];
  float near_plane, alpha2, thr_layer, thr_bkgd, boarder;
  int apply_thr;
  int n_layers;
  int fid_shared;            // all layers read frame-id column 6 (7-column rays)
};

// The scene constants of the density masks of a pass (pass_sigma).
struct PassMask {
  float near_plane, alpha2, thr_layer, thr_bkgd;
  int apply_thr;
};
__host__ __device__ inline PassMask pass_mask(const DevScene& s) { return {s.near_plane, s.alpha2, s.thr_layer, s.thr_bkgd, s.apply_thr}; }

// The density of sample (t, sg) of `layer` after the masks of its pass (layered_rfrender.py:414-422 coarse, :538-547 /
// :564-576 fine), as the compositing reads it.  factor: 0 (masked), alpha2 (layer 2, fine pass) or 1 -- torch's gradient of
// `density[mask] = 0` and of `density *= alpha`, which the training scatter records.  A kept density keeps its bits: it is
// not multiplied by 1 (a product may change a NaN's payload).
__device__ __forceinline__ float pass_sigma(const PassMask& m, int layer, bool fine, float t, float sg, float& factor) {
  float v = sg;
  bool kept = true;
  if (!fine) {
    if (layer > 0) {
      if (t < 0.0f) { v = 0.0f; kept = false; }                                       // :414
      if (m.apply_thr && v < m.thr_layer) { v = 0.0f; kept = false; }                 // :416-418
    } else if (t < m.near_plane) {
      v = 0.0f; kept = false;                                                         // :422
    }
  } else if (layer == 0) {
    if (m.apply_thr && v < m.thr_bkgd) { v = 0.0f; kept = false; }                    // :538-547
  } else {
    if (m.apply_thr && v < m.thr_layer) { v = 0.0f; kept = false; }                   // :564-566
    if (layer == 2) v = v * m.alpha2;                                                 // :575-576
  }
  factor = !kept ? 0.0f : (fine && layer == 2) ? m.alpha2 : 1.0f;
  return v;
}

// ---------------------------------------------------------------------------------------------------------
// Philox4x32-10 (production RNG when no uniforms are injected; statistically equivalent to torch.rand,
// not bit-equal -- parity runs inject uniforms).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
// uniform in [0,1) with 24 random bits, like torch.rand for float32
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t stream, uint64_t ray, uint32_t idx) {
  uint4 c = make_uint4((uint32_t)ray, (uint32_t)(ray >> 32), idx >> 2, stream);
  uint4 r = philox4x32_10(c, make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  uint32_t v = (idx & 3) == 0 ? r.x : (idx & 3) == 1 ? r.y : (idx & 3) == 2 ? r.z : r.w;
  return u01(v);
}

// ---------------------------------------------------------------------------------------------------------
// kernel launchers implemented in the .cu files (all enqueue on `st`, return STNERF_* codes)
// ---------------------------------------------------------------------------------------------------------
// geometry.cu
int launch_raygen(const float* Kinv, const float* T, int H, int W, int row0, int row_step, int n_rows,
                  const float* fids, int n_fids, float* rays, int ray_stride, cudaStream_t st);
int launch_sample(const float* rays, long long n, int ray_stride, const DevScene& scene, int n_layers, int n1,
                  const float* jitter, long long jitter_layer_stride, uint64_t seed, long long ray_base, RayIdMap idmap,
                  float* t_coarse, long long t_layer_stride, uint8_t* mask, long long mask_layer_stride,
                  int* hit, long long hit_layer_stride, int* counts, int* lerp_flags, cudaStream_t st,
                  const float* box_table = nullptr, int n_frames = 0, const LayerRays* layer_rays = nullptr);
// out (n, ray_stride) = rays with columns 0..5 replaced by the rotated (o', d'); the frame-id columns copied
int launch_rotate_rays(const float* rays, long long n, int ray_stride, const RayRot& r, float* out, cudaStream_t st);
int launch_intersect_sample(const float* rays, long long n, int ray_stride, const float* bmin, const float* bmax,
                            int is_bkgd, int n1, const float* jitter, float* t, float* xyz, uint8_t* mask,
                            float* tfar_tnear, cudaStream_t st);
int launch_posenc(const float* x, long long P, int dim, int n_freq, float* out, cudaStream_t st);

// composite.cu
struct CompositeArgs {
  const float* t;          // [layer][ray][S]
  long long t_layer_stride;
  const float* raw;        // [layer][ray][S][4]  (rgb raw, sigma raw)
  long long raw_layer_stride;
  const uint8_t* mask;     // [layer][ray] hit masks (chunk-local)
  long long mask_layer_stride;
  const float* u;          // [layer][ray][n2] injected uniforms or null
  long long u_layer_stride;
  float* t_fine;           // out (coarse pass with n2 > 0): [layer][ray][n1+n2]
  long long tf_layer_stride;
  float* z_new;            // out, optional: [layer][ray][n2] the new depths, ascending (flow reuse, see resample.cuh)
  long long zn_layer_stride;
  uint8_t* src_map;        // out, optional: [layer][ray][n1+n2] origin of every fine depth
  long long sm_layer_stride;
  float* out;              // images of this pass: [img][5*n_total], or null (coarse pass: resampling only, no images)
  unsigned skip_layers;    // bit i: layer i's own image + resampling were produced elsewhere (fused SpaceNet kernel): gather only
  int pixel_layout;        // 0: plane = rgb (N,3) | depth (N) | acc (N);  1: plane = (N,5) pixel-interleaved
  long long n_total;       // rays in the whole call (plane geometry)
  long long ray_base;      // first ray of this chunk within the call
  long long n;             // rays in this chunk
  int S, n2, fine;
  uint64_t seed;
  RayIdMap idmap;
};
// `force_generic`: run a coarse pass on the shared-memory path whatever its sample counts (stnerf_composite_pass: the register
// path and the generic path are two implementations of one function).  The generic path writes no z_new / src_map.
int launch_composite_pass(const CompositeArgs& a, const DevScene& scene, int n_layers, cudaStream_t st, bool force_generic = false);
// the sample counts whose coarse pass composites and resamples in registers (and can write z_new / src_map)
bool composite_pass_in_registers(int S, int n2, int fine);
int launch_composite_simple(const float* t, const float* rgb, const float* sigma, long long n, int S, float boarder,
                            float* color, float* depth, float* acc, float* w, cudaStream_t st);
int launch_composite_backward(const float* t, const float* rgb, const float* sigma, long long n, int S, float boarder,
                              const float* d_color, const float* d_depth, const float* d_acc, const float* d_w, float* d_rgb,
                              float* d_sigma, cudaStream_t st);
int launch_sample_pdf(const float* t, const float* w, const float* u, long long n, int n1, int n2, float* z,
                      float* t_fine, cudaStream_t st);

// mlp_simt.cu
int launch_spacenet_simt(const PointSrc& src, const SpaceNetW& w, float* raw, long long raw_slot_stride,
                         float* rgb_out, float* sigma_out, int num_sms, cudaStream_t st);
int launch_motionnet_simt(const PointSrc& src, const MotionNetW& w, const int* lerp_flag_dev, int lerp_force,
                          float* xyz_out, float* flow_out, int num_sms, cudaStream_t st);
size_t simt_smem_bytes();

// mlp_train.cu (kind 0 = SpaceNet, 1 = MotionNet; W / dW = stnerf_load_* blobs), with mlp_train_tc.cu
size_t train_saved_floats(int kind, int use_time);
size_t train_scratch_bytes(int kind, int use_time, long long P);
// prec: STNERF_TRAIN_FP32 or STNERF_TRAIN_TC_3XTF32 (validated by the caller)
int launch_spacenet_train_forward(const float* W, int use_time, const float* pos, const float* dirs, const float* times,
                                  long long P, float* rgb, float* sigma, float* saved, cudaStream_t st, int prec);
int launch_spacenet_backward(const float* W, int use_time, long long P, const float* saved, const float* d_rgb,
                             const float* d_sigma, float* dW, float* d_pos, void* scratch, cudaStream_t st, int prec);
int launch_motionnet_train_forward(const float* W, const float* xyzt, long long P, const int* lerp_flag, int lerp_force,
                                   float* flow, float* saved, cudaStream_t st, int prec);
int launch_motionnet_backward(const float* W, long long P, const float* saved, const float* d_flow, float* dW, void* scratch,
                              cudaStream_t st, int prec);

// train_march.cu (the per-sample work of a training step around the networks)
size_t train_hits_scratch_ints(long long n, int n_layers);
// totals_frac: [STNERF_MAX_LAYERS] hit counts then [STNERF_MAX_LAYERS] "any fractional frame id" flags (performer layers)
int launch_train_hits(const uint8_t* mask, long long n, int n_layers, const float* rays, int ray_stride, int fid_shared, int* hit,
                      int* scratch, int* totals_frac, cudaStream_t st);
int launch_train_points(const PointSrc& s, long long P, float* pos, float* dirs, float* times, float* xyzt, cudaStream_t st);
int launch_train_scatter(const DevScene& sc, int layer, int fine, const float* t, long long n, int S, const int* hit, long long P,
                         const float* rgb_c, const float* sigma_c, float* rgb, float* sigma, float* factor, cudaStream_t st);
int launch_train_gather(int S, const int* hit, long long P, const float* factor, const float* d_rgb, const float* d_sigma,
                        float* d_rgb_c, float* d_sigma_c, cudaStream_t st);
int launch_train_uniforms(long long n, int n2, int n_layers, uint64_t seed, RayIdMap idmap, float* u, cudaStream_t st);

// extract.cu (a layer's field at one frame; marching cubes)
struct FieldGrid {           // point (i,j,k) = origin + (i,j,k)*step, one product and one sum per axis
  float origin[3], step[3];
  int dims[3];
};
struct FieldEdit {           // the inverse edit of one layer and pass (inverse_edit), rotation first
  int shift_on, scale_on, rot_on;
  float shift[3], scale, pivot[3];
  RayRot rot;
};
// n points p0 .. p0+n-1 of `xyz` (P,3), or of the grid when xyz == null, edited -> xyzt (n,4) = (x, y, z, frame).
// With e.rot_on and dirs != null, also rdirs (n,3) = R^T dirs[p0 ..].
int launch_field_points(const float* xyz, const FieldGrid& g, long long p0, long long n, const FieldEdit& e, float frame,
                        float* xyzt, const float* dirs, float* rdirs, cudaStream_t st);

}  // namespace stnerf
