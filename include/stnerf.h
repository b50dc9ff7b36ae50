/*
 * stnerf.h -- C ABI of libstnerf_b200.so: the st-nerf layered ray-march hot path on H100 (sm_90a).
 *
 * The reference (DarlingHang/st-nerf) has no FFI seam: its boundary is the Python call surface
 *   modeling/layered_rfrender.py:141   LayeredRFRender.forward(rays, labels, bboxes, only_coarse, ...)
 *   utils/batchify_rays.py:51          layered_batchify_ray(model, rays, ...)
 *   engine/render.py:30                render(model, K, T, img_size, ...)
 * The Python facade in st-nerf_b200/{modeling,utils,layers,engine} keeps that surface and marshals it
 * onto the entry points below through ctypes (see INTEGRATION.md).  Each entry point cites the reference
 * code it replaces.  Paths are relative to the reference root.
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless the name ends in _host;
 *   - all functions return 0 on success or a negative STNERF_E* code; nothing throws; no hidden
 *     synchronisation: work is enqueued on `stream` (a cudaStream_t passed as void*);
 *   - the context owns its weights and a workspace; the workspace is (re)allocated only when a call
 *     asks for more rays-per-chunk / samples than any previous call (stnerf_reserve does it up front);
 *   - there is no CPU fallback: without a CUDA device every call returns STNERF_ENODEVICE.
 */
#ifndef STNERF_H_
#define STNERF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STNERF_MAX_LAYERS 8      /* l = 1 background + up to 7 performers (BASELINE config #5 uses 7) */
#define STNERF_MAX_N1 128        /* coarse samples per ray per layer                                  */
#define STNERF_MAX_S 512         /* n1 + n2                                                           */

enum {
  STNERF_OK = 0,
  STNERF_EINVAL = -1,      /* bad argument (the reference prints + exit(-1), layered_rfrender.py:162) */
  STNERF_ENODEVICE = -2,   /* no CUDA device / wrong architecture                                    */
  STNERF_ECUDA = -3,       /* a CUDA runtime call failed; stnerf_last_cuda_error() has the text      */
  STNERF_ENOWEIGHTS = -4,  /* a network needed by the call was never loaded                          */
  STNERF_ENOMEM = -5
};

/* Arithmetic mode of the two MLPs (modeling/spacenet.py:101-160, modeling/motion_net.py:34-71). */
enum {
  STNERF_PREC_FP32_SIMT = 0,   /* fp32 FFMA on CUDA cores: the bit-closest mode, validation baseline      */
  STNERF_PREC_TC_3XF16 = 1,    /* wgmma fp16 3-term split (hi*hi + lo*hi + hi*lo), fp32 accumulate:       */
                               /* ~fp32 products, meets the 1e-3 RGB gate (SURVEY App. C.3)               */
  STNERF_PREC_TC_F16 = 2,      /* wgmma single fp16 pass: fastest, does NOT meet the 1e-3 gate            */
  STNERF_PREC_TC_MIXED = 3,    /* TC_3XF16 for everything the density depends on (SpaceNet trunk + sigma head, MotionNet); */
                               /* single fp16 pass for the colour-only layer rgb_net.1 (spacenet.py:81-86): ~5 % fewer     */
                               /* MMAs; sigma and flow bit-identical to TC_3XF16, so resampling is untouched; the colour    */
                               /* sigmoid(rgb) of a sample is within ~3e-3 of TC_3XF16's on the shipped checkpoints        */
                               /* (per point, measured on one H100: tests/test_gpu_networks_f64.py; renders: DESIGN 4)     */
  STNERF_PREC_TC_3XF16_CF = 4  /* TC_3XF16 with the two correction products of every layer issued FIRST (over the whole K  */
                               /* range, then hi*hi) in the coarse pass and the MotionNets -- what the sample placement    */
                               /* depends on.  The correction terms are added while the accumulator is still small, so     */
                               /* the tensor core's rounding of its fp32 accumulation acts on them less; the hi weight     */
                               /* stages stream twice (see DESIGN 3.1)                                                     */
};

typedef struct stnerf_ctx* stnerf_handle;

typedef struct {
  int32_t n_layers;                              /* l = L+1, layer 0 = background (layered_rfrender.py:56,209) */
  int32_t space_time[STNERF_MAX_LAYERS];         /* net of layer i consumes PE(time) in its rgb head           */
                                                 /* (cfg.MODEL.USE_SPACE_TIME, layered_rfrender.py:62-67)       */
  int32_t precision;                             /* STNERF_PREC_*                                               */
  int32_t chunk_rays;                            /* rays per internal chunk; 0 = default (65536); at most 2^22-1  */
} stnerf_model_desc;

/* Per-call scene constants: what LayeredRFRender.forward derives in its prologue
 * (layered_rfrender.py:190-242) plus the attributes the renderer mutates between frames
 * (render/layered_neural_renderer.py:435-440).  All host memory. */
typedef struct {
  float bmin[STNERF_MAX_LAYERS][3];              /* box corner 0 after scale/shift edits (:230-242)             */
  float bmax[STNERF_MAX_LAYERS][3];              /* box corner 6 after edits                                    */
  int32_t shown[STNERF_MAX_LAYERS];              /* display_layers (:104-112); entry 0 is ignored like the ref. */
  /* inverse edit applied to sample points before the nets: p -= shift; p = (p - pivot)/scale + pivot           */
  int32_t shift_on[STNERF_MAX_LAYERS];           /* (:293-298) == (:467-471)                                    */
  float shift[STNERF_MAX_LAYERS][3];
  int32_t scale_coarse_on[STNERF_MAX_LAYERS];    /* (:300-303)                                                  */
  int32_t scale_fine_on[STNERF_MAX_LAYERS];      /* (:473-475), skipped when that layer's shift entry is None   */
  float scale[STNERF_MAX_LAYERS];
  float pivot[3];                                /* (centre_layer2 + centre_layer1)/2 (:221-232)                */
  float near_plane;                              /* model.near (:143,422,605)                                   */
  float alpha_layer2;                            /* model.alpha, fine pass, layer 2 only (:575-576)             */
  float density_threshold;                       /* (:416-418, 564-566)                                         */
  float bkgd_density_threshold;                  /* (:538-547)                                                  */
  float boarder_weight;                          /* cfg.MODEL.BOARDER_WEIGHT, last delta (render_layer.py:38)   */
  int32_t apply_thresholds;                      /* 1 in the retiming branch (:416,538,564), else 0             */
  int32_t shared_frame_id;                       /* 1: 7-column rays [o,d,frame_id] of the evaluator (:157-158,171):   */
                                                 /* every layer reads column 6; 0: one column per layer (retiming)      */
} stnerf_scene;

/* ---- lifetime ------------------------------------------------------------------------------------------ */
int stnerf_create(stnerf_handle* out, const stnerf_model_desc* desc_host);   /* modeling/__init__.py:5-7 build_layered_model */
void stnerf_destroy(stnerf_handle h);
int stnerf_reserve(stnerf_handle h, int n1, int n2);                         /* size the workspace up front                  */
size_t stnerf_workspace_bytes(stnerf_handle h);
const char* stnerf_strerror(int code);
const char* stnerf_last_cuda_error(void);
int stnerf_set_precision(stnerf_handle h, int precision);

/* ---- weights: load_state_dict (render/layered_neural_renderer.py:110-117) ------------------------------ */
/* blob = the net's tensors concatenated in state_dict order, fp32, nn.Linear (out,in) row-major:
 *   SpaceNet : stage1.{0,2,4,6}.{weight,bias}, stage2.{0,2,4}.{weight,bias}, density_net.0.{weight,bias},
 *              rgb_net.1.{weight,bias}, rgb_net.3.{weight,bias}      (464260 or 466948 floats, SURVEY App. B)
 *   MotionNet: motion_net.{0,2,4,6,8,10}.{weight,bias}               (77315 floats)
 * layer 0 = background; fine = 0 coarse net / 1 fine net.  MotionNets are shared by both passes.        */
int stnerf_load_spacenet(stnerf_handle h, int layer, int fine, const float* blob_host, size_t n_floats);
int stnerf_load_motionnet(stnerf_handle h, int layer, const float* blob_host, size_t n_floats);

int stnerf_set_scene(stnerf_handle h, const stnerf_scene* scene_host);
/* Per-frame boxes for rays that carry their OWN frame id: the 7-column rays of a mixed-frame batch (training / evaluation),
 * `bboxes = self.bboxes.index_select(0, rays_frame_id - 1)` (modeling/layered_rfrender.py:193).  table_host:
 * [n_frames][l][2][3] = (min, max) corner of every layer's box at every frame AFTER the scale / shift edits (:230-242), entry
 * [f][0] = the background box.  With a table set and scene.shared_frame_id = 1, ray r is clipped against row
 * (int)rays[r][6] - 1 (ids outside [1, n_frames] are clamped; the reference raises).  n_frames = 0 removes the table.      */
int stnerf_set_box_table(stnerf_handle h, const float* table_host, int n_frames);

/* Per-layer rotation edit.  The reference's LayeredNeuralRenderer takes a `rotation` argument and stores it without using it
 * (render/layered_neural_renderer.py:19,24); this is the edit it names.  Layer i (0 = background, indexed like shift / scale)
 * may carry a rotation R_i (fp32 3x3, row-major) about a centre c_i, applied on top of the scale / shift edit:
 *     world = c + R (edited(p) - c),
 * so a marched point is first rotated back, p <- c + R^T (p - c), and then goes through the unchanged inverse shift / scale.
 * The clipping region is the edited box rotated (an oriented box) and the SpaceNet sees the view direction R^T d.
 * Mechanism: the inverse edit is affine, so a rotated layer samples, marches and looks along its own copy of the rays,
 *     o' = c + R^T (o - c),   d' = R^T d,   frame-id columns unchanged,
 * with the op order  q = o - c;  o'_a = ((Rt[a][0] q0 + Rt[a][1] q1) + Rt[a][2] q2) + c_a;  d'_a = (Rt[a][0] d0 + Rt[a][1] d1)
 * + Rt[a][2] d2  (Rt = R^T, every product and sum rounded on its own).  Depths t stay world depths, so the masks, the
 * depth-merged composite, the near plane and the Philox keys are unchanged.  A hidden performer is sampled unrotated: hiding a
 * layer renders the same whether or not it is rotated.
 * on_host[l]: STNERF_ROT_OFF, STNERF_ROT_CENTRE (rotate about centre_host[i]) or STNERF_ROT_BOX (rotate about the centre of
 * layer i's box in the scene of each call, (bmin + bmax) * 0.5 in fp32: per view for stnerf_render_views).  R_host [l][9],
 * centre_host [l][3] (read for STNERF_ROT_CENTRE entries only; may be NULL when there are none).  on_host = NULL clears every
 * rotation.  Non-finite input or an unknown mode returns STNERF_EINVAL and leaves the rotation as it was.  Host-side only: the
 * rotation applies to stnerf_render*, stnerf_train_sample / stnerf_train_points and stnerf_layer_field / stnerf_layer_grid.  */
#define STNERF_ROT_OFF 0
#define STNERF_ROT_CENTRE 1
#define STNERF_ROT_BOX 2
int stnerf_set_rotation(stnerf_handle h, const int32_t* on_host, const float* R_host, const float* centre_host);
/* The rotated rays of one layer (the kernel every rotated path uses): out (n, ray_stride) = rays with columns 0..5 replaced by
 * (o', d') as above, for R_host (9, row-major) about centre_host (3).  out must not overlap rays.  Enqueue only.              */
int stnerf_rotate_rays(const float* rays, int64_t n, int ray_stride, const float* R_host, const float* centre_host, float* out,
                       void* stream);

/* ---- the hot path: LayeredRFRender.forward (layered_rfrender.py:141-734), BBOX sampling ---------------- */
/* rays: (n_rays, ray_stride) fp32, columns [o(3), d(3), frame_id_layer0 .. frame_id_layer(l-1)]
 *       (data/datasets/ray_dataset.py:276-281); ray_stride >= 6 + l  (>= 7 with scene.shared_frame_id).
 * jitter: (l, n_rays, n1) uniforms for layers/RaySamplePoint.py:98, or NULL -> in-kernel Philox(seed).
 * u:      (l, n_rays, n2) uniforms for utils/sample_pdf.py:31, or NULL -> Philox(seed).
 * out:    [2 passes: 0 coarse, 1 fine][l+1 images: 0 mixed, 1+i layer i] planes of 5*n_rays floats each,
 *         a plane = rgb (n_rays,3) | depth (n_rays) | acc (n_rays)   (the tuples of :725-734).
 *         With only_coarse the fine planes are left untouched (the facade aliases them, :721-722).
 *         The caller's current device must be the one the context was created on (else STNERF_EINVAL).
 * ray_mask: (l, n_rays) uint8, |bin_width| > 1e-5 (layers/RaySamplePoint.py:105).
 * MotionNet's lerp (modeling/motion_net.py:53) is decided once per call: any hit ray of layer i with a fractional frame id,
 * in any chunk, lerps layer i's time encoding for every ray of the call.                                 */
int stnerf_render(stnerf_handle h, const float* rays, int64_t n_rays, int ray_stride, int n1, int n2,
                  int only_coarse, const float* jitter, const float* u, uint64_t seed,
                  float* out, uint8_t* ray_mask, void* stream);

/* Keys of the in-kernel Philox stream: ray j of the following stnerf_render calls draws the uniforms of ray id
 *   base + (j / width) * row_stride + (j % width)      (width = 0: id = base + j, the default).
 * A caller that renders row-interleaved shards of an image (one process per GPU) sets base = first_row * W, width = W,
 * row_stride = n_ranks * W so that every pixel gets the same draws as in an unsharded render of the same seed.         */
int stnerf_set_ray_ids(stnerf_handle h, int64_t base, int32_t width, int64_t row_stride);

/* Same call with HOST buffers (pinned for overlap; pageable works, serialised by the driver): the rays go up chunk by chunk
 * on a copy stream while earlier chunks render, every finished chunk's slices of out / ray_mask come down on a second copy
 * stream while later chunks render; returns after everything has drained.  Replaces the `.cuda()` ... `.cpu()` bracket of
 * render_pose (render/layered_neural_renderer.py:372-392, 451-454).  This is the e2e path bench.py times.
 * Device staging is sized by stnerf_reserve_host; a call larger than anything reserved (re)allocates it first.            */
int stnerf_render_host(stnerf_handle h, const float* rays_host, int64_t n_rays, int ray_stride, int n1, int n2,
                       int only_coarse, uint64_t seed, float* out_host, uint8_t* ray_mask_host, void* stream);
/* Pre-size the device staging of the host-buffer entry points (rays, image planes, masks, per-view image buffers, copy
 * streams and events) for calls of up to `max_rays` rays, so that those calls allocate nothing.                            */
int stnerf_reserve_host(stnerf_handle h, int64_t max_rays, int ray_stride);

/* ---- the renderer-facing fast path: LayeredNeuralRenderer.render_pose / render_path ------------------------------------ */
/* (render/layered_neural_renderer.py:364-392, 401-488; data/datasets/ray_dataset.py:260-283 for the rays of a pose.)
 * One entry of a batch of poses: camera, the per-layer frame ids of the pose (`layer_frame_pair`, ray_dataset.py:276-279),
 * the scene constants of THIS frame (boxes lerped to these frame ids, per-frame shift/scale/alpha edits
 * render/layered_neural_renderer.py:435-440, thresholds) and the seed of its Philox stream.  All host memory.           */
typedef struct {
  float Kinv[9];                                 /* inverse intrinsics, row-major                                              */
  float T[16];                                   /* camera-to-world, row-major                                                  */
  float frame_ids[STNERF_MAX_LAYERS];            /* column 6+i of every ray of this view                                        */
  stnerf_scene scene;
  uint64_t seed;
} stnerf_view;
/* Renders rows row0, row0+row_step, ... (n_rows of them) of an HxW image for each of n_views poses in ONE call: rays are
 * generated on the device (never cross PCIe), and only what render_pose returns is produced -- the FINE images, mixed + one per
 * layer, pixel-interleaved: images[v*view_stride + (img*n_rows*W + pixel)*5 + {0,1,2: rgb, 3: depth, 4: acc}].  With
 * coarse_images == NULL the coarse pass only resamples (no coarse images, no merged coarse composite); with a buffer of the same
 * shape it also produces the coarse images, i.e. everything LayeredRFRender.forward returns (modeling/layered_rfrender.py:725-734).  The last requested row may lie one row_step past H-1 (equal
 * shard sizes when H is not a multiple of row_step): it is rendered as an extrapolated pixel row the caller discards.  Enqueue only; `images` is a DEVICE buffer -- e.g. one
 * rank's slice of an all-gather buffer when the rows of a view are interleaved over GPUs (row0 = rank, row_step = ranks).    */
int stnerf_render_views(stnerf_handle h, const stnerf_view* views_host, int n_views, int H, int W, int row0, int row_step,
                        int n_rows, int n1, int n2, float* images, float* coarse_images, int64_t view_stride, void* stream);
/* Full HxW frames to a HOST buffer ([n_views][l+1][H*W][5], pinned for overlap): the device->host copy of view v runs on a
 * copy stream while view v+1 renders (two device image buffers); returns after the last copy has landed.                   */
int stnerf_render_views_host(stnerf_handle h, const stnerf_view* views_host, int n_views, int H, int W, int n1, int n2,
                             float* images_host, void* stream);

/* ---- ray generation: utils/render_helpers.py:96-123 == utils/ray_sampling.py:22-72 --------------------- */
/* Kinv_host = inverse(K) (3x3 row-major), T_host = camera-to-world (4x4 row-major).  Writes rows
 * row0, row0+row_step, ... (n_rows of them) of an HxW image: rays[(k*W + j)*ray_stride + 0..5] = o,d and
 * columns 6..6+n_frame_ids-1 = frame_ids_host (data/datasets/ray_dataset.py:276-281).                     */
int stnerf_raygen(const float* Kinv_host, const float* T_host, int H, int W, int row0, int row_step, int n_rows,
                  const float* frame_ids_host, int n_frame_ids, float* rays, int ray_stride, void* stream);

/* ---- per-stage entry points (unit parity against the reference function named) ------------------------ */
/* layers/RaySamplePoint.py:8-62 + :85-105 for one box.  t (n,n1), xyz (n,n1,3) or NULL, mask (n) uint8,
 * tfar_tnear (n,2) or NULL = intersection()'s return.                                                     */
int stnerf_intersect_sample(const float* rays, int64_t n, int ray_stride, const float* bmin_host,
                            const float* bmax_host, int is_bkgd, int n1, const float* jitter,
                            float* t, float* xyz, uint8_t* mask, float* tfar_tnear, void* stream);
/* layers/render_layer.py:25-58.  t (n,S), rgb (n,S,3), sigma (n,S) -> color (n,3), depth (n), acc (n), w (n,S)|NULL */
int stnerf_composite(const float* t, const float* rgb, const float* sigma, int64_t n, int S, float boarder,
                     float* color, float* depth, float* acc, float* w, void* stream);
/* utils/sample_pdf.py:18-63 (+ the sort of layered_rfrender.py:462 when t_fine != NULL).
 * t (n,n1), w (n,n1) full weights (the [1:-1] slice is taken inside), u (n,n2) -> z (n,n2)|NULL, t_fine (n,n1+n2)|NULL */
int stnerf_sample_pdf(const float* t, const float* w, const float* u, int64_t n, int n1, int n2,
                      float* z, float* t_fine, void* stream);
/* One compositing pass of stnerf_render on explicit network outputs: the density masks of modeling/layered_rfrender.py:412-422
 * (coarse) / :538-547, 564-576 (fine), every hit layer's own VolumeRenderer.forward, the depth-ordered merge of :425-448 /
 * :587-606 and, in a coarse pass with n2 > 0, sample_pdf + the sort of :459-463 -- the kernel the render path launches, with
 * no context.  Uses near_plane, the thresholds, alpha_layer2, boarder_weight and shown[] of `scene_host`.
 * t (l,n,S), raw (l,n,S,4) = rgb logits + raw sigma, mask (l,n) uint8 (row 0 is ignored: the background is always hit; may be
 * NULL when l = 1), u (l,n,n2) or NULL = Philox stream 64+layer of `seed`, keyed by the ray index.
 * fine = 0: 3 <= S <= STNERF_MAX_N1, n2 >= 0, S + n2 <= STNERF_MAX_S;  fine = 1: 1 <= S <= STNERF_MAX_S, n2 = 0.
 * images (l+1, 5n): image 0 merged, 1+i layer i; pixel_layout 0 = rgb (n,3) | depth (n) | acc (n), 1 = (n,5) interleaved.
 *   NULL with n2 > 0: the pass only resamples.  A layer the ray misses gets a zero pixel.
 * t_fine (l,n,S+n2): sort(cat(t, z)) of every HIT (ray, layer); rows of missed layers are not written.  Required iff n2 > 0.
 * z_new (l,n,n2) ascending new depths and src_map (l,n,S+n2) the origin of every fine depth (k < S: coarse sample k, S + e:
 *   new depth e): both or neither, and only where the register-resident resampling runs and an origin fits a byte
 *   (S + n2 <= 256, n2 <= 256); STNERF_EINVAL elsewhere.  With STNERF_PASS_GENERIC=1 in the environment a coarse pass takes the
 *   shared-memory path whatever its sample counts (the path of n2 > 256), which writes t_fine only.                       */
int stnerf_composite_pass(const stnerf_scene* scene_host, int n_layers, int fine, const float* t, const float* raw,
                          const uint8_t* mask, const float* u, uint64_t seed, int64_t n, int S, int n2, int pixel_layout,
                          float* images, float* t_fine, float* z_new, uint8_t* src_map, void* stream);
/* utils/dimension_kernel.py:24-33.  x (P,dim) -> out (P, dim*(1+2*n_freq)) */
int stnerf_positional_encoding(const float* x, int64_t P, int dim, int n_freq, float* out, void* stream);
/* modeling/spacenet.py:101-160.  pos (P,3), dirs (P,3), times (P)|NULL -> rgb (P,3) raw, sigma (P) raw.
 * In STNERF_PREC_TC_3XF16_CF both passes' weights run with the correction products first.
 * Here and in stnerf_motionnet, P = 0 succeeds without reading or writing anything (the pointers may be NULL). */
int stnerf_spacenet(stnerf_handle h, int layer, int fine, const float* pos, const float* dirs, const float* times,
                    int64_t P, float* rgb, float* sigma, void* stream);
/* stnerf_spacenet in the weight-stage schedule stnerf_render uses for pass `fine`: the same call except in
 * STNERF_PREC_TC_3XF16_CF, whose fine pass keeps the interleaved order (corrections first in the coarse pass only).  A render's
 * SpaceNet outputs are this call's on the same points, bit for bit, in every precision.                                  */
int stnerf_spacenet_pass(stnerf_handle h, int layer, int fine, const float* pos, const float* dirs, const float* times,
                         int64_t P, float* rgb, float* sigma, void* stream);
/* modeling/motion_net.py:34-71.  xyzt (P,4) -> flow (P,3).  lerp_mode: -1 = decide like the reference
 * (any non-integer t in the batch, :53), 0/1 = force.                                                      */
int stnerf_motionnet(stnerf_handle h, int layer, const float* xyzt, int64_t P, int lerp_mode, float* flow,
                     void* stream);

/* ---- geometry: a layer's density field at one frame, and marching cubes ------------------------------------------------------
 * The field of layer `layer` in pass `fine` (0 coarse nets, 1 fine nets) at frame `frame_id` is what stnerf_render's network for
 * that layer and pass gives at a world point, in the context's precision and with its scene (stnerf_set_scene):
 *   1. the pass' inverse edit, rounded as the render rounds it: p -= shift (modeling/layered_rfrender.py:293-298 / :467-471),
 *      then p = (p - pivot)/scale + pivot with scale_coarse_on (fine = 0, :300-303) or scale_fine_on (fine = 1, :473-475);
 *   2. a performer (layer >= 1): flow = MotionNet(p, frame_id) and p += flow, one round-to-nearest fp32 add (:340-356 /
 *      :495-510); the time encoding is lerped exactly when frame_id is fractional (modeling/motion_net.py:53 for one frame);
 *   3. SpaceNet(p, dir, frame_id) (:397-409 / :552-563): the time input is frame_id when the net consumes time.
 * The networks run as stnerf_motionnet / stnerf_spacenet run them: in STNERF_PREC_TC_3XF16_CF the fine SpaceNet, too, adds
 * its correction products first, where the render's fine pass interleaves them (stnerf_spacenet_pass).
 * Layer and weight errors return STNERF_EINVAL / STNERF_ENOWEIGHTS; a call before stnerf_set_scene returns STNERF_EINVAL.   */
typedef struct {
  float origin[3];                               /* point (i,j,k) = origin + (i,j,k)*step: one fp32 product and one fp32 sum  */
  float step[3];                                 /* per axis, each rounded on its own                                        */
  int32_t dims[3];                               /* values are [dims0][dims1][dims2], C order, x slowest                      */
} stnerf_grid;
/* xyz (P,3) world points, dirs (P,3) view directions -> rgb (P,3) raw logits, sigma (P) raw.  rgb = NULL: sigma only, and dirs
 * may then be NULL too.  P = 0 succeeds without touching a pointer.  Enqueue only.                                             */
int stnerf_layer_field(stnerf_handle h, int layer, int fine, float frame_id, const float* xyz, const float* dirs, int64_t P,
                       float* rgb, float* sigma, void* stream);
/* The field's sigma on a grid (dims >= 2 per axis, finite origin and steps, else STNERF_EINVAL) -> sigma [dims0][dims1][dims2].
 * Equal, bit for bit, to stnerf_layer_field on the grid's points.  The grid is evaluated in chunks of 2^20 points in
 * stream-ordered device scratch of a size that does not depend on dims; enqueue only (no host synchronisation).               */
int stnerf_layer_grid(stnerf_handle h, int layer, int fine, float frame_id, const stnerf_grid* grid_host, float* sigma,
                      void* stream);
/* Marching cubes of a sigma grid (no context; the grid as above, with steps > 0).  A corner is inside when v > level; NaN is
 * outside.  A vertex lies on every grid edge whose endpoints differ in that test, at p0 + (level - v0)/(v1 - v0)*(p1 - p0) in
 * fp32 (at the outside endpoint when v0 or v1 is not finite).  Grid point (i,j,k) owns the vertices of its +x, +y, +z edges,
 * in that order, and vertices are numbered grid-point-major, so neighbouring cells share them: the mesh is indexed.  Triangles
 * come cell-major from a 256-case table that cuts every ambiguous face the same way from both of its cells (the inside corners
 * are kept apart), so a surface that stays off the grid border is closed; they are wound so that their normals point from
 * inside to outside (toward lower values).  Identical calls give identical bits.
 * Use: scratch of stnerf_mc_scratch_bytes bytes (0 = invalid grid); stnerf_mc_count fills it and returns the vertex and face
 * counts (one device->host copy: the only host synchronisation; STNERF_EINVAL when the vertex count does not fit int32);
 * stnerf_mc_fill, with the same sigma, grid, level and scratch, writes verts (V,3) fp32 and faces (F,3) int32.             */
size_t stnerf_mc_scratch_bytes(const stnerf_grid* grid_host);
int stnerf_mc_count(const float* sigma, const stnerf_grid* grid_host, float level, void* scratch, size_t scratch_bytes,
                    int64_t* n_verts_host, int64_t* n_faces_host, void* stream);
int stnerf_mc_fill(const float* sigma, const stnerf_grid* grid_host, float level, void* scratch, size_t scratch_bytes,
                   float* verts, int32_t* faces, void* stream);

/* ---- training: differentiable SpaceNet / MotionNet (no context) ------------------------------------------------------------
 * Training precision of the _prec entry points below; the entry points without _prec are STNERF_TRAIN_FP32.               */
enum {
  STNERF_TRAIN_FP32 = 0,       /* fp32 FFMA on CUDA cores; the forward is bit-identical to STNERF_PREC_FP32_SIMT            */
  STNERF_TRAIN_TC_3XTF32 = 1   /* every GEMM of a layer with 128 or more outputs (SpaceNet trunk + rgb_net.1, MotionNet
                                  motion_net.0-.8: forward, input deltas, weight gradients) on wgmma with 3xTF32 products
                                  (Alo*Bhi + Ahi*Blo + Ahi*Bhi, tf32 hi/lo split, fp32 accumulate, promoted into an fp32 total
                                  every 32 k): ~22 significant bits per product with fp32's exponent range.  The 1- and 3-wide
                                  heads stay fp32.  Its forward is NOT bit-identical to any STNERF_PREC_* render mode.       */
};
/* ---- fp32 on CUDA cores unless a _prec entry point is given STNERF_TRAIN_TC_3XTF32 ---------------------------------------
 * `weights` is a DEVICE blob in the stnerf_load_* order above (state_dict order, nn.Linear (out,in) row-major), read in place;
 * `d_weights` receives the gradient of every tensor in the same order and size (464260 / 466948 / 77315 floats).
 * A training forward fills `saved` (stnerf_train_saved_floats floats) with what the backward of the same points needs: the
 * encodings and the post-ReLU activations, feature-major.  `scratch` is stnerf_train_scratch_bytes bytes of device memory the
 * call may overwrite.  Products and sums are fp32; the forward's outputs are bit-identical to STNERF_PREC_FP32_SIMT.  Weight
 * and bias gradients are sums over the points in an order fixed by P alone (no atomics): identical calls, identical bits.
 * P = 0 succeeds (a backward then zeroes d_weights); P < 0 and missing required pointers return STNERF_EINVAL.
 * kind: 0 = SpaceNet, 1 = MotionNet; use_time: the SpaceNet's rgb head consumes PE(time) (rgb_net.1 width 304).          */
size_t stnerf_train_saved_floats(int kind, int use_time, int64_t P);
size_t stnerf_train_scratch_bytes(int kind, int use_time, int64_t P);
/* modeling/spacenet.py:101-160 (bins mode and maxs/mins are the caller's).  pos, dirs (P,3), times (P) | NULL -> rgb (P,3),
 * sigma (P) raw. */
int stnerf_spacenet_train_forward(const float* weights, int use_time, const float* pos, const float* dirs, const float* times,
                                  int64_t P, float* rgb, float* sigma, float* saved, void* stream);
/* Gradient of spacenet.py:101-160 for d_rgb (P,3), d_sigma (P): d_weights, and d_pos (P,3) through the encoding of
 * utils/dimension_kernel.py:24-33 and both of its uses (:135, the skip concatenation :137), or d_pos = NULL for none.
 * Directions and times get no gradient (modeling/layered_rfrender.py:272,314-315 detach them). */
int stnerf_spacenet_backward(const float* weights, int use_time, int64_t P, const float* saved, const float* d_rgb,
                             const float* d_sigma, float* d_weights, float* d_pos, void* scratch, size_t scratch_bytes,
                             void* stream);
/* modeling/motion_net.py:34-71.  xyzt (P,4) -> flow (P,3); lerp_mode as in stnerf_motionnet. */
int stnerf_motionnet_train_forward(const float* weights, const float* xyzt, int64_t P, int lerp_mode, float* flow, float* saved,
                                   void* scratch, size_t scratch_bytes, void* stream);
/* Gradient of motion_net.py:34-71 for d_flow (P,3): d_weights only (xyzt is detached, layered_rfrender.py:314-315). */
int stnerf_motionnet_backward(const float* weights, int64_t P, const float* saved, const float* d_flow, float* d_weights,
                              void* scratch, size_t scratch_bytes, void* stream);
/* The same four calls in a training precision (STNERF_TRAIN_*; the `saved` layout is the same for both).  A backward must
 * run in the precision of the forward that filled `saved`.  An unknown precision, or a scratch buffer smaller than
 * stnerf_train_scratch_bytes_prec reports, returns STNERF_EINVAL (stnerf_train_scratch_bytes_prec then returns 0). */
size_t stnerf_train_scratch_bytes_prec(int kind, int use_time, int64_t P, int precision);
int stnerf_spacenet_train_forward_prec(const float* weights, int use_time, const float* pos, const float* dirs, const float* times,
                                       int64_t P, float* rgb, float* sigma, float* saved, int precision, void* stream);
int stnerf_spacenet_backward_prec(const float* weights, int use_time, int64_t P, const float* saved, const float* d_rgb,
                                  const float* d_sigma, float* d_weights, float* d_pos, void* scratch, size_t scratch_bytes,
                                  int precision, void* stream);
int stnerf_motionnet_train_forward_prec(const float* weights, const float* xyzt, int64_t P, int lerp_mode, float* flow,
                                        float* saved, void* scratch, size_t scratch_bytes, int precision, void* stream);
int stnerf_motionnet_backward_prec(const float* weights, int64_t P, const float* saved, const float* d_flow, float* d_weights,
                                   void* scratch, size_t scratch_bytes, int precision, void* stream);
/* Gradient of layers/render_layer.py:8-58 (gen_weight + VolumeRenderer.forward) for stnerf_composite's outputs.
 * d_color (n,3), d_depth (n), d_acc (n), d_w (n,S): any may be NULL (zero).  -> d_rgb (n,S,3), d_sigma (n,S).
 * t gets no gradient (the reference detaches every depth it composites, layered_rfrender.py:314,461).
 * Recomputes the forward from (t, rgb, sigma); deterministic (no atomics).  n = 0 touches no pointer.            */
int stnerf_composite_backward(const float* t, const float* rgb, const float* sigma, int64_t n, int S, float boarder,
                              const float* d_color, const float* d_depth, const float* d_acc, const float* d_w,
                              float* d_rgb, float* d_sigma, void* stream);

/* ---- training: the per-sample work of a differentiable LayeredRFRender.forward around the networks ------------------------
 * (modeling/layered_rfrender.py:141-734 as stnerf_render computes it; the networks are the stnerf_*_train_* calls above and the
 * compositing is stnerf_composite / stnerf_composite_backward / stnerf_sample_pdf.)  Every call uses the context's scene
 * (stnerf_set_scene) and box table; n = 0 succeeds; bad arguments return STNERF_EINVAL.                                      */
/* layers/RaySamplePoint.py:8-107 for every layer (the sampling of stnerf_render, jitter (l,n,n1) or NULL = Philox stream i
 * with `seed`) -> t (l,n,n1), mask (l,n) uint8, and, per performer layer i >= 1, hit[i*n + j] = the j-th ray whose box was hit
 * in ASCENDING ray order (the boolean index `[ray_mask[i]]` of :343-356 / :400-413; block counts, an exclusive scan, then the
 * writes -- deterministic, unlike the render's block-claimed lists).  hit_counts_host[i] = the number of hit rays (n for
 * layer 0), any_frac_host[i] = 1 iff a hit ray's frame id of layer i is fractional (modeling/motion_net.py:53).  HOST
 * arrays of l ints: the call copies them back and synchronizes `stream` once -- they size the saved activations.          */
int stnerf_train_sample(stnerf_handle h, const float* rays, int64_t n, int ray_stride, int n1, const float* jitter, uint64_t seed,
                        float* t, uint8_t* mask, int32_t* hit, int32_t* hit_counts_host, int32_t* any_frac_host, void* stream);
/* The network inputs of one layer and pass in hit order (layered_rfrender.py:293-303 + :340-356 + :397-413 coarse,
 * :465-475 + :495-510 + :552-566 fine): m rays (hit == NULL and m = n for the background, else the hit list of the layer),
 * S depths each in t (n,S).  Point j*S+k: pos = t*d + o with the pass' inverse edit, rounded as stnerf_render rounds it
 * (bit-identical); dirs = d; times = frame-id column 6+layer (6 for 7-column rays); xyzt = (pos, time), MotionNet's input.
 * Any output may be NULL.                                                                                                    */
int stnerf_train_points(stnerf_handle h, int layer, int fine, const float* rays, int64_t n, int ray_stride, const float* t, int S,
                        const int32_t* hit, int64_t m, float* pos, float* dirs, float* times, float* xyzt, void* stream);
/* `rgbs[i][idx] = ...; density[i][idx] = ...` with the pass' density masks (layered_rfrender.py:412-422 coarse: t < 0 for a
 * performer, t < near for the background, the thresholds when the scene applies them; :538-547 / :564-576 fine: thresholds,
 * alpha on layer 2).  Compact rgb_c (m*S,3), sigma_c (m*S) in hit order -> dense rgb (n,S,3), sigma (n,S), zeros for rays
 * not in the list, and factor (m*S): 0 where masked, the alpha factor, or 1 -- what stnerf_train_gather multiplies by.    */
int stnerf_train_scatter(stnerf_handle h, int layer, int fine, const float* t, int64_t n, int S, const int32_t* hit, int64_t m,
                         const float* rgb_c, const float* sigma_c, float* rgb, float* sigma, float* factor, void* stream);
/* Backward of stnerf_train_scatter: d_rgb (n,S,3), d_sigma (n,S) (either may be NULL = zero) -> d_rgb_c (m*S,3),
 * d_sigma_c (m*S) = d_sigma * factor, in hit order.  A masked sample gets a zero gradient, as torch gives `density[mask] = 0`. */
int stnerf_train_gather(stnerf_handle h, int S, const int32_t* hit, int64_t m, const float* factor, const float* d_rgb,
                        const float* d_sigma, float* d_rgb_c, float* d_sigma_c, void* stream);
/* utils/sample_pdf.py:31 without injected uniforms: u (l,n,n2) = the Philox draws stnerf_render makes for the fine resampling
 * with this seed (stream 64+layer, keyed by the ray id), so a training forward places the render's fine samples.             */
int stnerf_train_uniforms(stnerf_handle h, int64_t n, int n2, uint64_t seed, float* u, void* stream);

/* Packed-weight image (cache next to the checkpoint; replaces re-running the state_dict -> MMA-layout packing that follows
 * render/layered_neural_renderer.py:109-117 `torch.load` + `load_state_dict`).  `export` writes every loaded network's
 * device images (fp32 SIMT layout, fp16 hi/lo tensor-core stream, fp32 bias/head block) into a HOST buffer; with
 * `host_buf == NULL` it only reports the size.  `import` validates the image against the context (layer count, per-layer
 * time inputs, sizes) before touching any network and restores the weights without re-packing.  Byte-for-byte the same
 * device state as `stnerf_load_*` on the original tensors, so renders are bit-identical.                                   */
int stnerf_weights_export(stnerf_handle h, void* host_buf, size_t capacity, size_t* bytes_needed);
int stnerf_weights_import(stnerf_handle h, const void* host_buf, size_t bytes);

/* ---- training ray pool: data/datasets/ray_dataset.py:339-460 + utils/ray_sampling.py:75-240 ---------------------------
 * A pool entry is 16 bytes (uint32 x4): pixel (row * W + col) | camera + frame slot << 16 | r, g, b, label bytes | layer.
 *
 * Selection of one (image, layer), replacing the per-camera ray_sampling_label_label (ray_sampling.py:194-240: keep
 * label == layer) and ray_sampling_label_bbox (:75-175: keep the rows [r0,r1) x cols [c0,c1) of the box's projected
 * rectangle).  `label` is a DEVICE map of H*W uint8 (label_is_float = 0) or fp32 (1) values, or NULL for the constant map
 * `const_label` (frame_dataset.py:278-284).  Kept pixels are compacted in row-major order; no atomic decides the order.
 * stnerf_td_select_count enqueues the per-tile counts and their scan into `scratch` (stnerf_td_select_scratch_ints(H, W)
 * ints); scratch[scratch_ints - 1] is then the number of kept pixels.  stnerf_td_select_write (same arguments, same
 * scratch, after the count) writes pool entries (rgb = DEVICE H*W*3 uint8, uint8 labels only) and/or the pixel indices.
 * rect_host = {r0, r1, c0, c1} for STNERF_TD_BY_RECT.  Bad arguments return STNERF_EINVAL.                                */
#define STNERF_TD_BY_LABEL 0
#define STNERF_TD_BY_RECT 1
int64_t stnerf_td_select_scratch_ints(int H, int W);
int stnerf_td_select_count(const void* label, int label_is_float, int const_label, int H, int W, int mode, int layer,
                           const int* rect_host, int* scratch, void* stream);
int stnerf_td_select_write(const void* label, int label_is_float, int const_label, const uint8_t* rgb, int H, int W,
                           int mode, int layer, const int* rect_host, int camera, int frame_slot, const int* scratch,
                           void* pool, int* pixels, void* stream);
/* One training batch from B pool indices (int32 or int64 `idx`, DEVICE), replacing Ray_Frame_Layer_Dataset.__getitem__
 * (ray_dataset.py:459-460) + default collate: rays (B, 6 + time_col) by the same arithmetic as stnerf_raygen, with frame id
 * frame_base + frame slot in column 6 when time_col = 1 (:416-418); rgbs (B,3) = byte / 255; labels, bbox_labels (B,1);
 * bboxes (B,8,3); near_far (B,2).  Tables (DEVICE fp32): cams [n_geom][n_cams][24] = K^-1 (9) | R (9) | origin (3) | W | 2
 * unused; boxes [n_layers][n_frames][24]; near_far [n_layers][n_frames][n_cams][2].  geom_of_layer_host[l] picks layer
 * l's camera table.  Enqueues one kernel; no host sync, no allocation.                                                    */
int stnerf_td_batch(const void* pool, const void* idx, int idx_is_64, int64_t B, const float* cams,
                    const int* geom_of_layer_host, int n_layers, int n_cams, const float* boxes, const float* near_far,
                    int n_frames, float frame_base, int time_col, float* rays, float* rgbs, float* labels,
                    float* bbox_labels, float* bboxes, float* near_far_out, void* stream);

/* Tensor-core plumbing self-test: one 128x256x64 fp16 product through the library's warpgroup-MMA descriptors, swizzled
 * layouts, bulk copy and accumulator fragment; writes max |D - host reference| (expected < 1e-3).                           */
int stnerf_selftest_umma(float* max_err_host);
/* Accumulation probe: the same 128x256x64 product of all-POSITIVE fp16 operands accumulated `reps` times into one register
 * accumulator (4*reps MMAs of K=16).  Reports max |D - fp64 sum| and the mean SIGNED relative error: how the tensor core
 * rounds when it adds into an fp32 accumulator (a negative mean growing with reps = round-toward-zero accumulation), which
 * bounds how close the fp16x3 split can get to the reference's fp32 GEMMs (DESIGN.md 4).                          */
int stnerf_selftest_umma_accum(int reps, float* max_err_host, float* mean_signed_rel_err_host);

/* Diagnostic read-back of the sample depths of the LAST chunk rendered by stnerf_render (parity tooling: which depths did
 * utils/sample_pdf.py:18-63 + the sort of modeling/layered_rfrender.py:462 produce for these rays?).
 * what = 0: coarse depths of `layer`, (n_rays, n1) floats;  what = 1: fine depths, (n_rays, n1+n2) floats;  what = 2: the new
 * depths in ascending order, (n_rays, n2) floats;  what = 3: the origin of every fine depth, (n_rays, n1+n2) BYTES (k < n1:
 * coarse sample k, n1 + e: new depth e) -- 2 and 3 exist only when that render reused the coarse pass' flow in the fine pass
 * (a tensor-core mode, n1 + n2 <= 256), STNERF_EINVAL otherwise.  dst is a DEVICE buffer of n_rays*S elements; n_rays must not
 * exceed the rays of that chunk and S must be the row length named above.  Rows of rays that miss `layer` are stale.      */
int stnerf_debug_read_depths(stnerf_handle h, int what, int layer, void* dst, int64_t n_rays, int S, void* stream);

/* Number of kernels this library has launched since load (bench.py's gpu_launches claim). */
uint64_t stnerf_launch_count(void);

/* ---- measurement: per-kernel-class device times taken with CUDA events on the launching stream ----------- */
/* classes: 0 SpaceNet MLP, 1 MotionNet MLP, 2 sampling, 3 compositing/resampling.  `points` = network
 * evaluations (classes 0,1) or rays (2) / ray-passes (3) processed, so callers can turn ms into FLOP/s or B/s. */
typedef struct {
  double ms[4];
  double points[4];
  uint64_t launches[4];
} stnerf_profile;
int stnerf_profile_begin(stnerf_handle h);                       /* start recording (adds two events per launch)   */
int stnerf_profile_end(stnerf_handle h, stnerf_profile* out_host); /* drain the device, stop recording, return totals */

#ifdef __cplusplus
}
#endif
#endif /* STNERF_H_ */
