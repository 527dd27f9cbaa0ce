/*
 * mvpraymarch_b200 -- C-ABI of the H100 (sm_90a) MVP raymarcher.
 *
 * This is the drop-in boundary for ava-256's hot path: every entry point below replaces one function of
 * the reference's pybind11 module `mvpraymarchlib` (reference paths relative to /root/reference):
 *
 *   mvp_raymarch_forward   <- raymarch_forward   extensions/mvpraymarch/mvpraymarch.cpp:180-280
 *                             (+ compute_aabb    extensions/mvpraymarch/mvpraymarch.cpp:146-178, which the
 *                              reference's Python calls right before it, mvpraymarch.py:81-82: building the
 *                              acceleration structure is part of the forward call here)
 *   mvp_raymarch_backward  <- raymarch_backward  extensions/mvpraymarch/mvpraymarch.cpp:282-396
 *   mvp_build_accel        <- compute_aabb       extensions/mvpraymarch/mvpraymarch.cpp:146-178
 *                             (stand-alone form, for callers that want to build once and march many times)
 *   mvp_workspace_bytes    <- the tensors build_accel allocates, extensions/mvpraymarch/mvpraymarch.py:21-84
 *   mvp_compute_raydirs    <- compute_raydirs_forward  extensions/utils/utils.cpp:46-82 (pybind module `utilslib`;
 *                             the step right before the raymarcher, SURVEY.md section 8f row 1)
 *   mvp_camera (struct)    <- the same call fused away: given the camera parameters compute_raydirs takes
 *                             (models/autoencoder.py:240), the render kernels generate each tile's rays in their prologue
 *                             (extensions/utils/utils_kernel.cu:32-46) and raypos / raydir / tminmax never exist in HBM
 *
 * and two entry points that replace eager PyTorch chains of the callers either side of the path (no native reference
 * counterpart; SURVEY.md section 8f rows 2 and 4):
 *
 *   mvp_composite_*        <- models/raymarchers/mvpraymarcher.py:50-51 (NHWC -> NCHW rgb / alpha split),
 *                             models/colorcals/colorcal.py:26-29 (w * rgb + b), models/autoencoder.py:262-270 (matting)
 *   mvp_assemble_payload_* <- models/decoders/rgb.py:128-143, models/decoders/geometry.py:180-185 (image -> slab
 *                             re-layout), models/decoders/assembler.py:261 (relu(rgb * 25 + 100), relu(alpha), cat)
 *
 * Conventions (same ownership model as the reference: the caller owns every buffer, outputs are written in
 * place; unlike the reference nothing is allocated inside and everything runs on the caller's stream):
 *   - all pointers are DEVICE pointers to contiguous fp32 (or int32) arrays, except the template and its gradient, which may be
 *     bfloat16 (MVP_FLAG_TPLATE_BF16, and the bf16 forms mvp_assemble_payload_*_bf16 / mvp_sum_views_bf16); no torch types;
 *   - `stream` is a cudaStream_t passed as void*;
 *   - return value: 0 = ok, < 0 = invalid argument (MVP_ERR_*), > 0 = a cudaError_t from the launch;
 *   - thread-safe and re-entrant: no global state.
 *
 * Tensor layouts (SURVEY.md terminology table):
 *   raypos, raydir [N,H,W,3]   tminmax [N,H,W,2]
 *   primpos [N,K,3]  primrot [N,K,3,3] (row-major)  primscale [N,K,3] (inverse half-extents)
 *   tplate  [N,K,TD,TH,TW,4] channels-last RGBA      warp [N,K,WD,WH,WW,3] channels-last (algo 1)
 *   rayrgba [N,H,W,4]  raysat [N,H,W,3]  rayaux [N,H,W,4] (int32, opaque; written by forward, read by backward)
 */
#ifndef MVPRAYMARCH_B200_H_
#define MVPRAYMARCH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVP_ABI_VERSION 8

#define MVP_OK 0
#define MVP_ERR_NULL (-1)      /* a required pointer is NULL */
#define MVP_ERR_SHAPE (-2)     /* non-positive or unsupported dimension (H, W < 32768; K >= 1) */
#define MVP_ERR_STEPSIZE (-3)  /* stepsize must be finite and > 0 */
#define MVP_ERR_WORKSPACE (-4) /* workspace too small or misaligned (256 B) */
#define MVP_ERR_ALGO (-5)      /* algo must be 0 (no warp field) or 1 (warp field, primsampler.h:53-58) */
#define MVP_ERR_ALIGN (-6)     /* a vector-accessed buffer is misaligned: tplate, rayrgba, grad_rayrgba, grad_tplate, rayaux,
                                * clear_grad_* need 16 bytes (tplate, grad_tplate 8 with MVP_FLAG_TPLATE_BF16; grad_tplate 16
                                * again with MVP_FLAG_GRAD_TPLATE_F32), tminmax 8,
                                * everything else 4 */
#define MVP_ERR_STRUCT (-7)    /* args->struct_size != sizeof(the struct this library was built with) */
#define MVP_ERR_CAMERA (-8)    /* camera.volradius must be finite and > 0 */

typedef struct mvp_shape {
    int32_t N, H, W, K, TD, TH, TW;
} mvp_shape;

/* flags */
#define MVP_FLAG_ACCEL_VALID 1u /* workspace already holds the accel structure of these primitives+rays */
#define MVP_FLAG_ZERO_GRADS 2u  /* backward only: the library zero-fills the gradient buffers on `stream` before it
                                 * accumulates into them (replaces the caller's zeros_like of mvpraymarch.py:240-246) */
#define MVP_FLAG_SHARED_PRIMS 4u /* primpos/primrot/primscale/tplate/warp (and their gradients) have a batch dimension of
                                 * ONE that all N views share: [1,K,...] instead of [N,K,...] (SURVEY.md section 8e
                                 * "optional fast path"); gradients of all views accumulate into the one set.  Must be the
                                 * same in mvp_build_accel / forward / backward calls that share a workspace. */
#define MVP_FLAG_TPLATE_BF16 8u  /* forward and backward: tplate, grad_tplate and clear_grad_tplate point to bfloat16, not fp32
                                 * (same [N,K,TD,TH,TW,4] channels-last layout, 8 bytes per voxel; tplate and grad_tplate 8-byte
                                 * aligned, clear_grad_tplate 16).  The output is exactly that of the fp32 kernels on the widened
                                 * template; grad_tplate is accumulated in bf16 (round to nearest even per reduction).  Everything
                                 * else stays fp32.  Must be the same in a forward and the backward that follows it.  The library
                                 * supports it iff mvp_build_config() lists TPLATE_BF16=1 (an older one ignores the bit). */
#define MVP_FLAG_GRAD_TPLATE_F32 16u /* forward and backward, with MVP_FLAG_TPLATE_BF16: the template is still read as bfloat16, but
                                 * grad_tplate and clear_grad_tplate point to FP32 buffers [N,K,TD,TH,TW,4] (16 bytes per voxel,
                                 * 16-byte aligned) and the backward accumulates into them with fp32 reductions, like the fp32
                                 * kernels: every gradient, the template's included, is that of the fp32 kernels on the widened
                                 * template up to the order of the fp32 atomics, and images, raysat and rayaux are those of the bf16
                                 * path.  Without MVP_FLAG_TPLATE_BF16 it changes nothing (an fp32 template's gradient is fp32).
                                 * Like MVP_FLAG_TPLATE_BF16 it must be the same in a forward and the backward that follows it: the
                                 * forward sizes its clear of clear_grad_tplate by it.  The library supports it iff
                                 * mvp_build_config() lists GRAD_TPLATE_F32=1 (an older one ignores the bit). */
#define MVP_FLAG_NO_TPLATE_GRAD 32u /* forward and backward: no gradient of the template or the warp field is wanted.  grad_tplate,
                                 * grad_warp, clear_grad_tplate and clear_grad_warp may then be NULL, and are neither read nor
                                 * written if they are not.  The backward computes the transform gradients (and with
                                 * mvp_raymarch_backward_rays the ray gradients) without the payload-gradient scatter, its most
                                 * expensive part; they equal those of the full backward up to the order of the fp32 atomics.
                                 * MVP_FLAG_GRAD_TPLATE_F32 has no effect with it.  Without this flag or the next one a NULL gradient
                                 * pointer is MVP_ERR_NULL.  The library supports it iff mvp_build_config() lists GRAD_SELECT=1. */
#define MVP_FLAG_RAY_GRADS_ONLY 64u /* forward and mvp_raymarch_backward_rays: only the ray gradients are wanted.  The rule above
                                 * extends to every primitive gradient (grad_primpos / primrot / primscale / tplate / warp and every
                                 * clear_grad_*): they may be NULL and are ignored.  The backward skips the payload scatter and the
                                 * transform-gradient sums.  mvp_raymarch_backward with this flag returns MVP_ERR_NULL: it would have
                                 * no output.  MVP_FLAG_ZERO_GRADS zero-fills only the buffers a call's flags request. */
#define MVP_FLAG_DETERMINISTIC 128u /* forward: the clear_grad_primpos / primrot / primscale / tplate buffers are the int64 sums of the
                                 * mvp_raymarch_backward_deterministic call that follows (8 bytes per entry, four entries per voxel
                                 * whatever the template's type) and are cleared as such.  The backward ignores the bit: the entry
                                 * point chooses the mode.  The library supports it iff mvp_build_config() lists DETERMINISTIC=1. */
#define MVP_FLAG_TEST_TINY_LISTS 0x100u /* test hook: forward keeps at most 16 saved tile-list entries per view, so almost
                                 * every tile takes the backward's rebuild path */

/* The pinhole cameras of the N views, exactly the arguments of the reference's compute_raydirs (extensions/utils/utils.py:21-51,
 * kernel utils_kernel.cu:12-52) on the integer pixel grid (its `pixelcoords` = (W, H) tuple form): ray (n, h, w) starts at
 * viewpos[n] / volradius and points along normalize(viewrot[n]^T ((w - princpt.x) / focal.x, (h - princpt.y) / focal.y, 1)).
 * A call that gets a camera (viewpos != NULL) generates the rays inside the kernels -- bit-identical to what
 * mvp_compute_raydirs writes -- and ignores raypos / raydir / tminmax, which may then be NULL: 32 bytes per ray that are neither
 * written by a ray-generation pass nor read by forward and backward, and no camera fit over the ray field in the accel build.
 * All four pointers or none; volradius finite and > 0.  Must be the same in every call that shares a workspace. */
typedef struct mvp_camera {
    const float *viewpos;    /* [N,3]   camera centres (same unit as volradius) */
    const float *viewrot;    /* [N,3,3] row-major; rows = camera x, y, z axes in world coordinates */
    const float *focal;      /* [N,2]   focal lengths in pixels (x, y) */
    const float *princpt;    /* [N,2]   principal point in pixels (x, y) */
    float volradius;         /* world units of the unit cube's half edge (models/autoencoder.py: self.volradius) */
    uint32_t reserved;       /* 0 */
} mvp_camera;

typedef struct mvp_forward_args {
    uint32_t struct_size;    /* = sizeof(mvp_forward_args); a truncated or stale caller-side struct is rejected */
    mvp_shape shape;
    float stepsize, fadescale, fadeexp;
    uint32_t flags;
    const float *raypos, *raydir, *tminmax;   /* may be NULL when `camera` is given */
    const float *primpos, *primrot, *primscale;
    const float *tplate;
    float *rayrgba;          /* out; may be NULL when rayrgb_nchw / rayalpha_nchw are given */
    float *raysat;           /* out, NULL when no gradient will be taken (mvpraymarch.py:147-152) */
    int32_t *rayaux;         /* out, NULL iff raysat is NULL */
    void *workspace;         /* >= mvp_workspace_bytes(shape), 256-byte aligned */
    size_t workspace_bytes;
    /* algo 1 only (reference: PrimSamplerTW<true>): warp field [N,K,WD,WH,WW,3] channels-last, sampled at the slab
     * coordinate; the payload is then sampled at the warped position (zero outside the slab).  algo 0 ignores these. */
    const float *warp;
    int32_t WD, WH, WW;
    int32_t algo;            /* 0 or 1 (mvpraymarch.py:303) */
    /* Optional image-plane outputs, written by the render kernel's epilogue (both or neither): rayrgb [N,3,H,W] and
     * rayalpha [N,1,H,W] -- what models/raymarchers/mvpraymarcher.py:50-51 makes of rayrgba with a permute and two
     * .contiguous() copies (SURVEY.md section 8f row 2). */
    float *rayrgb_nchw;
    float *rayalpha_nchw;
    /* Optional marching order [N,K] int32 ([1,K] with MVP_FLAG_SHARED_PRIMS): order[n][j] = index of the slab marched j-th.
     * NULL = the reference's fixed order (utils.h:740-742).  This is the `sortedobjid` of the reference's usebvh=True branch
     * (mvpraymarch.py:46-55; codes from mvp_compute_morton) applied as an indirection instead of a gather of the primitive
     * tensors.  Must be a permutation of 0..K-1 and the same in every call that shares the workspace. */
    const int32_t *order;
    /* Optional (each may be NULL): the gradient buffers of the mvp_raymarch_backward call that will follow, shapes as in
     * mvp_backward_args.  A gradient-mode forward (raysat != NULL) zero-fills them from inside its render kernel -- every warp
     * clears one slice with streaming stores before it renders its tile; the kernel is issue bound and the DRAM write path idle,
     * so the 134 MB per view cost nothing measurable, where a memset pass (MVP_FLAG_ZERO_GRADS in the backward, or the caller's
     * zeros_like of mvpraymarch.py:265-268) costs 1.4 ms per 80 views.  16-byte aligned; ignored when raysat is NULL;
     * clear_grad_warp is used for algo 1 only. */
    float *clear_grad_primpos, *clear_grad_primrot, *clear_grad_primscale, *clear_grad_tplate, *clear_grad_warp;
    mvp_camera camera;       /* optional (camera.viewpos != NULL): rays generated in the kernels, see mvp_camera */
} mvp_forward_args;

typedef struct mvp_backward_args {
    uint32_t struct_size;    /* = sizeof(mvp_backward_args) */
    mvp_shape shape;
    float stepsize, fadescale, fadeexp;
    uint32_t flags;          /* MVP_FLAG_ACCEL_VALID if `workspace` is the one the forward call filled: besides the accel
                              * structure it then holds each tile's slab list and each ray's first step as the forward (called
                              * with raysat != NULL) saved them, and the backward loads them instead of rebuilding; without the
                              * flag, or for tiles that did not fit, everything is rebuilt from the inputs */
    const float *raypos, *raydir, *tminmax;
    const float *primpos, *primrot, *primscale;
    const float *tplate;
    const float *grad_rayrgba; /* [N,H,W,4]; NULL when the gradient comes as image planes (grad_rayrgb_nchw / grad_rayalpha_nchw) */
    const float *raysat;       /* from forward */
    const int32_t *rayaux;     /* from forward */
    float *grad_primpos, *grad_primrot, *grad_primscale; /* out, accumulated into: caller zero-fills (or MVP_FLAG_ZERO_GRADS) */
    float *grad_tplate;        /* out, accumulated into: caller zero-fills (or MVP_FLAG_ZERO_GRADS) */
    void *workspace;
    size_t workspace_bytes;
    const float *warp;         /* algo 1 only */
    float *grad_warp;          /* algo 1 only; out, accumulated into: caller zero-fills */
    int32_t WD, WH, WW;
    int32_t algo;
    /* The incoming gradient as image planes [N,3,H,W] + [N,1,H,W] (both, with grad_rayrgba == NULL), read by the kernel's
     * prologue: the adjoint of the fused epilogue above; replaces the contiguous() copy of mvpraymarch.py:264. */
    const float *grad_rayrgb_nchw;
    const float *grad_rayalpha_nchw;
    const int32_t *order;      /* as in the forward call */
    mvp_camera camera;         /* as in the forward call */
} mvp_backward_args;

int mvp_abi_version(void);
/* Build-time knobs of the kernels in this library, e.g. "FWD_OPAQUE=2 LIST_REUSE=1 ..." (for bench / bug reports). */
const char *mvp_build_config(void);
const char *mvp_error_string(int code);

/* Bytes of scratch the accel structure + per-call state need for this shape (0 for an invalid shape). */
size_t mvp_workspace_bytes(const mvp_shape *shape);

/* Build the acceleration structure (camera fit, primitive records, screen rectangles, tile-row lists). */
int mvp_build_accel(const mvp_shape *shape, uint32_t flags, const int32_t *order, const float *raypos, const float *raydir,
                    const float *primpos, const float *primrot, const float *primscale,
                    void *workspace, size_t workspace_bytes, void *stream);
/* The same from the camera parameters instead of the ray field (see mvp_camera): no pass over the rays at all. */
int mvp_build_accel_camera(const mvp_shape *shape, uint32_t flags, const int32_t *order, const mvp_camera *camera,
                           const float *primpos, const float *primrot, const float *primscale,
                           void *workspace, size_t workspace_bytes, void *stream);

/* 30-bit Morton codes of slab centres that the caller has normalised to the unit cube (mvpraymarch.py:46-50):
 * compute_morton of the reference (extensions/mvpraymarch/mvpraymarch.cpp:106-121, bvh.cu:20-57).
 * centre [N,K,3] -> code [N,K] int32.  Sorting a view's codes gives the `order` the raymarch calls take. */
int mvp_compute_morton(int32_t N, int32_t K, const float *centre, int32_t *code, void *stream);

int mvp_raymarch_forward(const mvp_forward_args *args, void *stream);
int mvp_raymarch_backward(const mvp_backward_args *args, void *stream);
/* mvp_raymarch_backward plus the gradients of the rays, in the ray-tensor and in the camera form (args->camera): everything
 * mvp_raymarch_backward does, and grad_raypos, grad_raydir [N,H,W,3] and grad_tminmax [N,H,W,2] are WRITTEN (not accumulated),
 * one value per ray, rays that take no sample included.  The gradient is that of the image with every discrete decision of the
 * march held fixed (candidate lists, first lattice step, the strict validity test, the saturating sample, the 512-entry cap):
 * with the ray's samples x_j = raypos + raydir (tmin + j stepsize) up to and including the saturating one,
 *   grad_raypos = sum_j dL/dx_j,   grad_raydir = sum_j (tmin + j stepsize) dL/dx_j,   grad_tminmax = (<raydir, grad_raypos>, 0),
 * which is what autograd gives for the reference's PyTorch loop (extensions/mvpraymarch/mvpraymarch.py:567-633) with its sample
 * positions left attached.  grad_raypos / grad_raydir 4-byte aligned, grad_tminmax 8;
 * argument errors are returned before any device work.  The library supports it iff mvp_build_config() lists RAY_GRADS=1. */
int mvp_raymarch_backward_rays(const mvp_backward_args *args, float *grad_raypos, float *grad_raydir, float *grad_tminmax,
                               void *stream);

/* Several subjects' (or frames') views in one launch.  view_set: device int32 [N]; view n renders primitive set view_set[n] of
 * nsets, 1 <= nsets <= N.  primpos / primrot / primscale / tplate / warp, `order` and every gradient and clear_grad_* buffer then
 * have a leading dimension of nsets instead of N ([nsets,K,...]); the gradients of all views of a set accumulate into that set, and
 * a set that no view references gets zero gradients.  Every flag composes as in mvp_raymarch_forward / mvp_raymarch_backward(_rays),
 * except MVP_FLAG_SHARED_PRIMS (the one-set form is nsets = 1 with an all-zero map): with it the call returns MVP_ERR_SHAPE.
 * The map is input from outside the program and is not range-checked on the host: a view whose entry is outside [0, nsets) renders
 * empty (zero colour and alpha, raysat unset), contributes no gradient and gets zero ray gradients; nothing is read or written out
 * of bounds, and the other views are unaffected.  A workspace filled by a sets forward is valid (MVP_FLAG_ACCEL_VALID) only for a
 * sets backward with the same map.  Argument errors are returned before any device work: view_set NULL is MVP_ERR_NULL, nsets
 * outside [1, N] MVP_ERR_SHAPE, a view_set that is not 4-byte aligned MVP_ERR_ALIGN.
 * The backward computes the ray gradients of mvp_raymarch_backward_rays when all three ray pointers are non-NULL and none when all
 * three are NULL; any other combination is MVP_ERR_NULL.  mvp_workspace_bytes is unchanged (its per-slab records are sized N * K).
 * mvp_build_accel / mvp_build_accel_camera have no sets form: a sets call builds its acceleration structure itself.
 * The library supports these iff mvp_build_config() lists VIEW_SETS=1. */
int mvp_raymarch_forward_sets(const mvp_forward_args *args, const int32_t *view_set, int32_t nsets, void *stream);
int mvp_raymarch_backward_sets(const mvp_backward_args *args, const int32_t *view_set, int32_t nsets,
                               float *grad_raypos, float *grad_raydir, float *grad_tminmax, void *stream);

/* The camera form (args->camera, required: MVP_ERR_NULL without it) at arbitrary sample positions: ray (n, h, w) is the camera's ray
 * through pixelcoords[n,h,w] (device fp32 [N,H,W,2], 8-byte aligned), the ray mvp_compute_raydirs makes from the same pixelcoords,
 * bit for bit; no ray tensor is read or written.  The acceleration structure takes a per-view axis-aligned affine map
 * px = ox + sx w, py = oy + sy h from three corners of the view's coordinates and verifies every coordinate against it (to 0.05 of
 * a grid step): the integer grid, crops, strides and pixel-centre offsets keep their slab rectangles; a view that fails the check
 * renders the same image with every slab a candidate for every tile (slower, like a ray field whose camera fit fails).
 * view_set NULL: per-view or shared primitives as in mvp_raymarch_forward / mvp_raymarch_backward(_rays) (nsets ignored); non-NULL:
 * the sets form, with the rules and argument errors of mvp_raymarch_forward_sets.  The backward computes the ray gradients of
 * mvp_raymarch_backward_rays when all three ray pointers are non-NULL and none when all three are NULL (any other combination is
 * MVP_ERR_NULL); pixelcoords gets no gradient (the camera's, via mvp_compute_raydirs_backward with the same pixelcoords).  A
 * workspace filled by a pixels forward is valid (MVP_FLAG_ACCEL_VALID) for a pixels backward with the same pixelcoords, and for a
 * ray-tensor backward of the rays mvp_compute_raydirs makes from them (the same rays, bit for bit).
 * Argument errors are returned before any device work.  mvp_build_accel_camera has no pixels form.  The library supports these iff
 * mvp_build_config() lists CAMERA_PIXELS=1. */
int mvp_raymarch_forward_pixels(const mvp_forward_args *args, const float *pixelcoords, const int32_t *view_set, int32_t nsets,
                                void *stream);
int mvp_raymarch_backward_pixels(const mvp_backward_args *args, const float *pixelcoords, const int32_t *view_set, int32_t nsets,
                                 float *grad_raypos, float *grad_raydir, float *grad_tminmax, void *stream);

/* Reproducible primitive gradients: mvp_raymarch_backward with grad_primpos / primrot / primscale / tplate summed in 64-bit two's-
 * complement fixed point, so that they depend only on the inputs -- not on the order in which warps are scheduled, on which tiles
 * the 512-entry kernels take, or on the order of the views.  The images of the forward are unchanged.
 *   - The backward runs twice.  The measure pass finds, per gradient tensor, the largest |value| M that goes into one reduction (a
 *     merged voxel group's payload sum, or a warp's transform sum over one slab visit); the tensor's quantum is q = 2^(e - 38) with
 *     2^e the smallest power of two >= M (q >= 2^-126).  The accumulate pass adds llrint(value / q) to the int64 sums with integer
 *     reductions, and a conversion writes (float)sum * q into the gradient buffers, which are WRITTEN, not accumulated into (a bf16
 *     template gradient rounded once more, to nearest even).
 *   - Limits: an entry must take fewer than 2^24 reductions (every term is at most 2^38 in magnitude); the result keeps 38 bits
 *     below the tensor's largest reduction, so an entry far smaller than that loses relative precision.
 *   - An entry that received a non-finite value comes out NaN, and no other entry does.
 *   - acc_primpos [nsets,K,3], acc_primrot [nsets,K,9], acc_primscale [nsets,K,3], acc_tplate [nsets,K,TD,TH,TW,4] (NULL with
 *     MVP_FLAG_NO_TPLATE_GRAD): caller-owned int64 scratch, 8-byte aligned, zero on entry -- cleared by the gradient-mode forward
 *     called with MVP_FLAG_DETERMINISTIC and these buffers as clear_grad_*, or by MVP_FLAG_ZERO_GRADS here.  nsets is N per view,
 *     1 with MVP_FLAG_SHARED_PRIMS, or the sets call's nsets.  det_max: caller-owned uint32 [4] (4-byte aligned), written.
 *   - pixelcoords: NULL, or the pixels form of mvp_raymarch_backward_pixels; view_set: NULL, or the sets form with the rules and
 *     argument errors of mvp_raymarch_backward_sets.  Per-view, shared and set primitives, Morton `order`, camera rays, image
 *     planes, fp32 and bf16 templates (MVP_FLAG_GRAD_TPLATE_F32 included) and MVP_FLAG_NO_TPLATE_GRAD are supported.
 *   - algo 1 is MVP_ERR_ALGO; MVP_FLAG_RAY_GRADS_ONLY is MVP_ERR_NULL (this entry point computes no ray gradients).
 * It launches the render kernels twice and one conversion kernel per gradient tensor.  Argument errors are returned before any
 * device work.  The library supports it iff mvp_build_config() lists DETERMINISTIC=1. */
int mvp_raymarch_backward_deterministic(const mvp_backward_args *args, int64_t *acc_primpos, int64_t *acc_primrot, int64_t *acc_primscale,
                                        int64_t *acc_tplate, uint32_t *det_max, const float *pixelcoords, const int32_t *view_set,
                                        int32_t nsets, void *stream);

/* Pinhole ray generation + unit-cube clip (reference: extensions/utils/utils_kernel.cu:12-52).
 * viewpos [N,3], viewrot [N,3,3], focal [N,2], princpt [N,2], pixelcoords [N,H,W,2] or NULL (integer grid);
 * outputs raypos, raydir [N,H,W,3], tminmax [N,H,W,2]. */
int mvp_compute_raydirs(int32_t N, int32_t H, int32_t W, const float *viewpos, const float *viewrot, const float *focal,
                        const float *princpt, const float *pixelcoords, float volradius, float *raypos, float *raydir,
                        float *tminmax, void *stream);
/* Adjoint of mvp_compute_raydirs (and of the rays an mvp_camera call generates): the per-ray gradients grad_raypos, grad_raydir
 * [N,H,W,3] and grad_tminmax [N,H,W,2] (8-byte aligned, like pixelcoords) are chained through o = viewpos / volradius, the
 * unit-cube clip of tmin (the face the forward's min/max chain selects; zero where tmin is clamped to 0; tmax has no gradient),
 * d = e / |e|, e = viewrot^T (u, v, 1) and u = (px - princpt.x) / focal.x, v = (py - princpt.y) / focal.y into grad_viewpos [N,3],
 * grad_viewrot [N,3,3], grad_focal [N,2] and grad_princpt [N,2], which are ACCUMULATED into: the caller zero-fills them.  Nothing
 * goes to pixelcoords or volradius.  One thread per ray; the 16 per-view sums are reduced per block and added with one atomic per
 * block and value, so the result is deterministic up to the order of those atomics. */
int mvp_compute_raydirs_backward(int32_t N, int32_t H, int32_t W, const float *viewpos, const float *viewrot, const float *focal,
                                 const float *princpt, const float *pixelcoords, float volradius, const float *grad_raypos,
                                 const float *grad_raydir, const float *grad_tminmax, float *grad_viewpos, float *grad_viewrot,
                                 float *grad_focal, float *grad_princpt, void *stream);

/* Image epilogue (SURVEY.md section 8f row 2).  rayrgba [N,H,W,4] (16-byte aligned) ->
 *   irgbrec  [N,3,H,W] = (ccw[n,c] * rgb + ccb[n,c]) + (1 - alpha) * bg[n,c,h,w]      (each op rounded once, like eager torch)
 *   rayalpha [N,1,H,W] = alpha                                                        (optional)
 * ccw, ccb [N,3]: per-view colour calibration, both NULL for none; bg [N,3,H,W] or NULL for a black background. */
int mvp_composite_forward(int32_t N, int32_t H, int32_t W, const float *rayrgba, const float *ccw, const float *ccb,
                          const float *bg, float *irgbrec, float *rayalpha, void *stream);
/* Adjoint of the above.  grad_rayrgba [N,H,W,4] is written (not accumulated) contiguous channels-last, which is what
 * mvp_raymarch_backward takes.  grad_ccw / grad_ccb [N,3] (both or neither) are ACCUMULATED into: caller zero-fills;
 * grad_bg [N,3,H,W] is written.  rayrgba is needed only when grad_ccw or grad_bg is requested. */
int mvp_composite_backward(int32_t N, int32_t H, int32_t W, const float *rayrgba, const float *ccw, const float *bg,
                           const float *grad_irgbrec, const float *grad_rayalpha, float *grad_rayrgba, float *grad_ccw,
                           float *grad_ccb, float *grad_bg, void *stream);

/* Payload hand-off (SURVEY.md section 8f row 4).  tex [N, B*3, hb*B, wb*B] (channel d*3+c), opacity [N, B, hb*B, wb*B]
 * (channel d) -> tplate [N, hb*wb, B, B, B, 4] with
 *   tplate[n, i*wb+j, d, y, x, c<3] = relu(tex[n, d*3+c, i*B+y, j*B+x] * rgb_scale + rgb_bias),
 *   tplate[n, i*wb+j, d, y, x, 3]   = relu(opacity[n, d, i*B+y, j*B+x]).
 * The reference hard-codes rgb_scale = 25, rgb_bias = 100 (assembler.py:261).  1 <= B <= 64. */
int mvp_assemble_payload_forward(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tex, const float *opacity,
                                 float rgb_scale, float rgb_bias, float *tplate, void *stream);
/* Adjoint: grad_tex / grad_opacity (same shapes as tex / opacity) are written; `tplate` is the forward output (relu mask). */
int mvp_assemble_payload_backward(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tplate, const float *grad_tplate,
                                  float rgb_scale, float *grad_tex, float *grad_opacity, void *stream);
/* The same with a bfloat16 template (the layout MVP_FLAG_TPLATE_BF16 reads: 8 bytes per texel).  Forward: the fp32 values above,
 * each rounded once to bf16 (nearest even; NaN stays NaN).  Backward: grad_tplate is bf16, widened exactly, masked where the bf16
 * tplate is > 0 and multiplied by rgb_scale in fp32; grad_tex / grad_opacity stay fp32.  A relu output in (0, 2^-134] rounds to
 * bf16 zero, so its gradient is masked, where the fp32 chain would pass it.  tplate and grad_tplate need 8-byte alignment (the
 * 16-byte vector variant is taken when they, tex / opacity or grad_tex / grad_opacity are 16-byte aligned and B % 4 == 0).
 * The library supports these iff mvp_build_config() lists EPILOGUE_BF16=1. */
int mvp_assemble_payload_forward_bf16(int32_t N, int32_t hb, int32_t wb, int32_t B, const float *tex, const float *opacity,
                                      float rgb_scale, float rgb_bias, void *tplate, void *stream);
int mvp_assemble_payload_backward_bf16(int32_t N, int32_t hb, int32_t wb, int32_t B, const void *tplate, const void *grad_tplate,
                                       float rgb_scale, float *grad_tex, float *grad_opacity, void *stream);

/* One subject's primitives materialised per view (what the decoders' batch dimension is in models/autoencoder.py:214-233
 * when all items of a batch show the same subject): dst[v, i] = src[i] for v < n_views, i < count floats.  One pass of
 * streaming 16-byte stores (scalar when count % 4 != 0 or a pointer is not 16-byte aligned); `expand().contiguous()` does the
 * same at a quarter of the rate.  count < 2^32 * 1024. */
int mvp_expand_views(const float *src, float *dst, size_t count, int32_t n_views, void *stream);
/* Its adjoint, and the local step of the per-subject gradient reduction (SURVEY.md section 8e: the views of a step share one
 * subject's primitives, their gradients are summed before the one all-reduce): dst[i] = sum over v < n_views of src[v, i], added
 * in view order (deterministic), one pass over the per-view gradients.  Same alignment rule as mvp_expand_views; n_views >= 1. */
int mvp_sum_views(const float *src, float *dst, size_t count, int32_t n_views, void *stream);
/* The same over bfloat16 views: src [n_views, count] bf16, each value widened exactly and added in fp32 in view order, so an fp32
 * dst (dst_bf16 = 0) equals mvp_sum_views of the widened source bit for bit; a bf16 dst (dst_bf16 != 0) gets that sum rounded
 * once (nearest even).  src 2-byte aligned, dst 4 (fp32) or 2 (bf16); 16-byte accesses when count % 8 == 0 and both pointers
 * are 16-byte aligned.  A bf16 tensor is expanded with mvp_expand_views as 4-byte words (count / 2, even counts). */
int mvp_sum_views_bf16(const void *src, void *dst, size_t count, int32_t n_views, int32_t dst_bf16, void *stream);

/* Test / diagnostics helper (host only, no device work): given a HOST copy of a workspace that a gradient-mode forward
 * has filled, counts the tiles whose slab list the forward saved for the backward (`saved`, lists with >= 1 entry) and the
 * tiles it had to mark not-saved because the list storage was full (`not_saved`; the backward rebuilds those). */
int mvp_debug_saved_tiles(const mvp_shape *shape, const void *host_workspace_copy, int *saved, int *not_saved);
/* Diagnostics builds only (-DMVP_TILE_CLOCKS=1, scripts/tile_clocks.py): byte offset of the per-tile clock records in the workspace. */
size_t mvp_debug_tileclk_offset(const mvp_shape *shape);
/* Test / diagnostics helper (host only, no device work): byte offset in the workspace of the int32 count of "heavy" tiles, the
 * tiles whose slab list did not fit the fast render kernel's list and that the 512-entry kernel rendered.  Every forward and
 * backward call resets it first, so the 4 bytes read after a call are that call's count; 0 for an invalid shape. */
size_t mvp_debug_heavy_offset(const mvp_shape *shape);
/* Test / diagnostics helper (host only, no device work): byte offset in the workspace of the int32 [N] per-view flags of the last
 * acceleration build: non-zero where the view's camera could not be used to cull slabs (a failed camera fit, a degenerate camera,
 * pixelcoords off an axis-aligned map), so that every slab was a candidate on it; 0 for an invalid shape. */
size_t mvp_debug_view_fallback_offset(const mvp_shape *shape);

/* Number of kernels the last forward / backward call of this shape launches (for bench.py's gpu_launches).  A pixels call
 * (mvp_raymarch_forward_pixels / mvp_raymarch_backward_pixels) without MVP_FLAG_ACCEL_VALID launches one more: the check of its
 * coordinates against an affine map. */
int mvp_forward_launch_count(uint32_t flags);
int mvp_backward_launch_count(uint32_t flags);

#ifdef __cplusplus
}
#endif
#endif /* MVPRAYMARCH_B200_H_ */
