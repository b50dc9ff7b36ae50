// Warpgroup-MMA (sm_90a wgmma) evaluation of SpaceNet / MotionNet: precision modes TC_3XF16, TC_3XF16_CF, TC_MIXED and TC_F16.
#pragma once
#include "common.cuh"

namespace stnerf {

// Coarse-pass fusion (SURVEY 8a a10-a12 behind a8): with n1 = 64 a 128-point tile of the SpaceNet kernel is exactly two rays of
// one layer, so the kernel's two compositing warps composite the tile's (rgb, sigma) rows straight from shared memory
// (layers/render_layer.py:8-58), draw the n2 fine depths (utils/sample_pdf.py:18-63) and write sort(cat(t, z))
// (modeling/layered_rfrender.py:459-463) -- the coarse rgb / sigma never leave the SM, and the work hides under the next
// tile's MMAs.  Arithmetic: resample.cuh, shared with the stand-alone compositing kernel.
struct FuseCoarse {
  int on;                      // 0: the kernel only evaluates the network
  int n1, n2, layer;
  const float* u;              // injected uniforms of this layer, [ray][n2], or null -> Philox(seed, 64 + layer, ray id, j)
  uint64_t seed;
  RayIdMap idmap;
  long long ray_base;          // first ray of the chunk within the call (Philox key, image row)
  float* t_fine;               // out: this layer's [ray][n1 + n2] sorted depths
  float* z_new;                // out, optional (with src_map): this layer's [ray][n2] new depths, ascending
  uint8_t* src_map;            // out, optional: this layer's [ray][n1 + n2] origin of every fine depth (resample.cuh)
  float* img;                  // out: this layer's coarse image (one pixel per hit ray), or null
  long long n_total;           // rays of the whole call (plane geometry of img)
  int pixels;                  // img layout: 0 planes, 1 pixel-interleaved
  PassMask mask;               // density masks of the coarse pass (pass_sigma)
  float boarder;
};

// Weights of one network packed for the tensor-core kernels (see mlp_tc.cu for the layout).
struct TcNet {
  void* blob = nullptr;        // device: fp16 hi/lo weight blocks in the 128B-swizzled K-major SMEM image
  size_t blob_bytes = 0;
  float* aux = nullptr;        // device: fp32 biases / head weights
  float* w_tail = nullptr;     // device: SpaceNet rgb_net.1 columns 256.. transposed [48][128] fp32 (head_bias_kernel)
  int use_time = 0;
};

int tc_pack_spacenet(TcNet& net, const float* blob_host, bool use_time);
int tc_pack_motionnet(TcNet& net, const float* blob_host);
void tc_free(TcNet& net);
// Packed-weight cache: sizes of one network's device images, read-back and restore (no re-packing).
size_t tc_stream_bytes(bool is_space);
size_t tc_aux_floats();
size_t tc_tail_floats(bool is_space);
int tc_export(const TcNet& net, bool is_space, uint8_t* stream_host, float* aux_host, float* tail_host);
int tc_import(TcNet& net, bool is_space, int use_time, const uint8_t* stream_host, const float* aux_host, const float* tail_host);
int tc_selftest(float* max_err_host);   // one 128x256x64 warpgroup-MMA product vs a host reference
int tc_selftest_accum(int reps, float* max_err_host, float* mean_signed_rel_host);   // accumulation probe (see mlp_tc.cu)
// fine_pass: the SpaceNet evaluation of a render's fine pass, which keeps the interleaved product order in TC_3XF16_CF
int tc_launch_spacenet(const PointSrc& src, const TcNet& net, int precision, float* cbuf, float* raw, float* rgb_out,
                       float* sigma_out, int num_sms, cudaStream_t st, const FuseCoarse* fuse = nullptr, bool fine_pass = false);
bool tc_can_fuse_coarse(int n1, int n2);     // sample counts the fused compositing warps are instantiated for
int tc_launch_motionnet(const PointSrc& src, const TcNet& net, int precision, const int* lerp_flag_dev, int lerp_force,
                        float* xyz_out, float* flow_out, int num_sms, cudaStream_t st);

}  // namespace stnerf
