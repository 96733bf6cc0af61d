/*
 * sparf_b200 -- C ABI of the SPARF ray-marching hot path on the H100 (sm_90a).
 *
 * The reference (google-research/sparf) has NO FFI: its boundary for this path is the Python class
 * contract `Graph` / `NeRF` (source/models/renderer.py:28, source/models/frequency_nerf.py:72).  This
 * header is the C ABI we put UNDER that contract; each entry point names the reference code it
 * replaces.  Host-side mirror: sparf_b200/{renderer,frequency_nerf,camera}.py (ctypes, see
 * INTEGRATION.md for the binding a reference maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to fp32 (or int64 where stated) unless marked "host";
 *   - tensors are dense row-major; "R" = rays in the batch (B images x n rays flattened), "S" =
 *     samples per ray; per-sample tensors are [R,S] / [R,S,3];
 *   - all work is enqueued on `stream` (a cudaStream_t); nothing synchronises the device;
 *   - the caller owns every buffer incl. the workspace (sparf_workspace_bytes); no hidden allocation;
 *   - return value 0 = success, otherwise a SPARF_ERR_* code; sparf_last_error() gives the text
 *     (thread-local).  No exceptions cross the ABI.
 *   - gradient outputs of *_backward are ACCUMULATED (+=) into the given buffers so that several
 *     render passes of one step can share one flat gradient buffer (the caller zeroes it once).
 *
 * Process-level state (all of it): the thread-local error string; a launch counter (sparf_launch_count); per device,
 * lazily: the SM count.  Every call enqueues on `stream` only, so a call sequence is capturable into a CUDA graph.
 * A workspace must not be shared by calls running concurrently on different streams.
 */
#ifndef SPARF_B200_H_
#define SPARF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPARF_B200_VERSION 100 /* 0.1.0 */
#define SPARF_MAX_TRUNK 12
#define SPARF_MAX_L 16

enum {
  SPARF_OK = 0,
  SPARF_ERR_INVALID = 1,     /* bad argument / unsupported configuration */
  SPARF_ERR_CUDA = 2,        /* a CUDA runtime call or kernel launch failed */
  SPARF_ERR_WORKSPACE = 3,   /* workspace too small */
  SPARF_ERR_UNSUPPORTED = 4  /* valid request that this build/engine cannot serve */
};

/* Which arithmetic evaluates the MLP GEMMs. */
enum {
  SPARF_ENGINE_AUTO = 0,
  SPARF_ENGINE_SIMT_FP32 = 1, /* CUDA-core FFMA, fp32 throughout (bit-level twin of the reference) */
  SPARF_ENGINE_TC_3X = 2, /* Hopper wgmma: x*W = x_lo*W_hi + x_hi*W_lo + x_hi*W_hi on 16-bit halves (fp16 in the
                             forward, bf16 for gradients), fp32 accumulation: the parity engine */
  SPARF_ENGINE_TC_1X = 3, /* wgmma, single 16-bit pass ("fast", NOT within the 1e-4 parity bound) */
  SPARF_ENGINE_TC_3X_W1 = 4 /* TC_3X forward and input / pose gradients (parity), but the weight gradients dW = G^T X in
                               ONE bf16 pass over the hi halves.  Non-default, reduced precision (8-bit factors; the
                               rounding errors average over the batch) */
};

typedef void* sparf_stream_t; /* cudaStream_t */

/*
 * View of one reference `NeRF` module (frequency_nerf.py:87-134): trunk `mlp_feat.{i}` and colour
 * head `mlp_rgb.{0,1}`; weights are the nn.Linear tensors themselves, [out,in] row-major fp32.
 *   trunk layer i: in = (i==0 ? E3 : width) + (i==skip_layer ? E3 : 0), out = width (+1 on the last:
 *                  row 0 = raw density, rows 1.. = features), E3 = 3 + 6*L_xyz
 *   head 0: in = width + Ev, out = head_width, Ev = 3 + 6*L_view;  head 1: in = head_width, out = 3
 * BARF coarse-to-fine (frequency_nerf.py:244-257): if use_c2f, the kernel reads the device scalar
 * `progress` (NeRF.progress) and applies w_j = (1-cos(pi*clamp((p-c2f_start)/c2f_range*L - j,0,1)))/2.
 */
typedef struct SparfMLP {
  int32_t n_trunk;    /* 8 */
  int32_t width;      /* 256 */
  int32_t head_width; /* 128 */
  int32_t skip_layer; /* 4; -1 = none */
  int32_t L_xyz;      /* 10 */
  int32_t L_view;     /* 4 */
  int32_t use_c2f;    /* opt.barf_c2f is not None */
  float c2f_start;    /* float(start) */
  float c2f_range;    /* float(end - start), the subtraction done in double like the reference's python floats */
  const float* progress; /* device scalar, may be NULL iff !use_c2f */
  const float* trunk_w[SPARF_MAX_TRUNK];
  const float* trunk_b[SPARF_MAX_TRUNK];
  const float* head_w[2];
  const float* head_b[2];
} SparfMLP;

/* Gradient destinations, same shapes as SparfMLP's tensors (param.grad storage). Accumulated. */
typedef struct SparfMLPGrad {
  float* trunk_w[SPARF_MAX_TRUNK];
  float* trunk_b[SPARF_MAX_TRUNK];
  float* head_w[2];
  float* head_b[2];
} SparfMLPGrad;

/* ---------------------------------------------------------------- misc */
int sparf_version(void);
const char* sparf_last_error(void);
/* number of CUDA kernels this library has launched so far in this process (bench.py: gpu_launches) */
uint64_t sparf_launch_count(void);
/* 1 if `engine` can run on the current device (the tensor-core engines need an sm_90 device) */
int sparf_engine_available(int engine);

/* ---------------------------------------------------------------- rays
 * camera.get_center_and_ray / get_center_and_ray_at_pixels (source/utils/camera.py:347-416), computed
 * only for the requested pixels (the reference builds the whole H*W grid and indexes it,
 * renderer.py:273-291).  pose_w2c [B,3,4], intr_inv [B,3,3] = K^-1 (host code inverts K).
 *   ray_idx: int64 [n] (shared, idx_per_image=0) or [B,n] (idx_per_image=1), pixel = (x+0.5,y+0.5),
 *            idx = y*W+x;   or pixels: fp32 [n,2] / [B,n,2] used as given (no +0.5).
 * Exactly one of ray_idx / pixels is non-NULL.  Outputs origins, dirs: [B*n,3].
 */
int sparf_raygen_forward(int32_t B, int32_t n, int32_t W, const float* pose_w2c, const float* intr_inv,
                         const int64_t* ray_idx, const float* pixels, int32_t per_image,
                         float* origins, float* dirs, sparf_stream_t stream);
/* d(origins), d(dirs) [B*n,3] -> d(pose_w2c) [B,3,4], accumulated (+=).  d_pixels (optional, float-pixel path only):
 * gradient w.r.t. the pixel locations, same shape as `pixels` -- written for per-image pixels [B,n,2], accumulated (+=,
 * caller zeroes) for a shared [n,2] list.  The reference's get_center_and_ray_at_pixels is differentiable in the pixels
 * and the depth-consistency loss relies on it (depth_cons_loss.py:247-283). */
int sparf_raygen_backward(int32_t B, int32_t n, int32_t W, const float* pose_w2c, const float* intr_inv,
                          const int64_t* ray_idx, const float* pixels, int32_t per_image,
                          const float* d_origins, const float* d_dirs, float* d_pose_w2c, float* d_pixels,
                          sparf_stream_t stream);

/* ---------------------------------------------------------------- depth samples
 * Graph.sample_depth (renderer.py:383-419) and sample_depth_diff_max_range_per_ray (:595-624).
 *   t[r,k] = ((u + k)/S) * range + near,  u = rand[r,k] (rand != NULL) or 0.5, or 1.0 when far_per_ray
 *   is given (then range = far_per_ray[r] - near);  inverse != 0 -> t = 1/(t + 1e-8).
 */
int sparf_sample_depth(int32_t R, int32_t S, float near, float range, int32_t inverse, const float* rand,
                       const float* far_per_ray, float* t, sparf_stream_t stream);

/* Graph.sample_depth_from_pdf + cat + sort (renderer.py:421-456, :334-336).
 *   weights [R,S], t_coarse [R,S], u [S_fine] = mid-points of the shared grid, bins = linspace(near,far,S+1)
 *   outputs t_fine [R,S_fine] (may be NULL) and t_all [R,S+S_fine] ascending.
 *   Limit: S + S_fine <= 4096 (one block per ray sorts S+S_fine values in shared memory); larger -> SPARF_ERR_INVALID. */
int sparf_sample_pdf_merge(int32_t R, int32_t S, int32_t S_fine, float near, float far, const float* weights,
                           const float* t_coarse, const float* u, float* t_fine, float* t_all,
                           sparf_stream_t stream);

/* ---------------------------------------------------------------- MLP
 * NeRF.forward_samples (frequency_nerf.py:260-281): x = o + t*d, positional encoding, trunk, softplus
 * density (+ noise[R,S] on the raw value when non-NULL), colour head, sigmoid.
 * Outputs sigma [R,S], rgb [R,S,3].
 * sparf_mlp_workspace_bytes: `backward` = 0 forward call (sparf_mlp_forward or sparf_mlp_forward_tape), 1
 * sparf_mlp_backward (recompute), 2 sparf_mlp_backward_tape.
 */
size_t sparf_mlp_workspace_bytes(const SparfMLP* mlp, int32_t R, int32_t S, int32_t backward, int32_t engine);
int sparf_mlp_forward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                      const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                      void* workspace, size_t workspace_bytes, sparf_stream_t stream);
/* Backward of the above (activations are recomputed, nothing is kept from the forward call).
 * d_sigma [R,S], d_rgb [R,S,3] -> parameter grads (+=) and, when non-NULL, d_origins/d_dirs [R,3] (+=). */
int sparf_mlp_backward(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                       const float* dirs, const float* t, const float* noise, const float* d_sigma,
                       const float* d_rgb, const SparfMLPGrad* grad, float* d_origins, float* d_dirs,
                       void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* Tape variants: the TRAINING forward additionally keeps, in a caller-held `tape`, what the backward needs (encodings,
 * trunk and colour-head activations, the softplus argument), so that sparf_mlp_backward_tape skips the recompute.  The
 * tape must stay untouched between the two calls, and both take the same `engine`; sparf_mlp_backward_tape reads the
 * forward's `rgb` output.  sparf_mlp_tape_bytes returns 0 when no tape is offered (a tape above 16 GB): use the
 * recompute pair then.  Outputs and numerics are identical to sparf_mlp_forward / sparf_mlp_backward. */
size_t sparf_mlp_tape_bytes(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S);
int sparf_mlp_forward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                           const float* dirs, const float* t, const float* noise, float* sigma, float* rgb,
                           void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                           sparf_stream_t stream);
int sparf_mlp_backward_tape(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const float* origins,
                            const float* dirs, const float* t, const float* sigma, const float* rgb,
                            const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad, float* d_origins,
                            float* d_dirs, void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                            sparf_stream_t stream);
/* The taped pair with a row count read on the device, for passes over the samples an occupancy grid keeps, whose count
 * the host never reads (sparf_occupancy_count writes it to device memory), so that a training step stays one CUDA graph.
 * The arguments are those of the taped pair, with R = C a capacity that sizes the tape (sparf_mlp_tape_bytes(C, 1)),
 * the workspace (sparf_mlp_workspace_bytes(C, 1, 0 or 2)) and the chunk loop, and rows (device int64) = K, the rows
 * processed; K > C counts as C, K < 0 as 0.  S must be 1 (one-sample rays, the compaction's layout) and the engine
 * TC_3X, TC_1X or TC_3X_W1 (AUTO resolving to one of them); otherwise SPARF_ERR_UNSUPPORTED or SPARF_ERR_INVALID.
 *   - sigma, rgb, d_origins and d_dirs have the bits of the taped pair called with R = K on rows [0, K); the parameter
 *     gradients agree up to the order of their float atomics (each GEMM unit's partial sums are the same);
 *   - rows [K, C) of the inputs (origins, dirs, t, noise, sigma, rgb, d_sigma, d_rgb) are never read, and the same rows
 *     of the outputs (sigma, rgb, d_origins, d_dirs) never written;
 *   - every kernel processes min(chunk rows, K - chunk start) rows; a chunk wholly past K costs one launch per kernel
 *     that returns at once.  The weight-gradient GEMMs split their k-ranges in the kernel from K, as the host splits
 *     them from R in the taped pair.
 * The tape is left for sparf_mlp_backward_tape_rows with the same rows, which must hold the same K. */
int sparf_mlp_forward_tape_rows(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const int64_t* rows,
                                const float* origins, const float* dirs, const float* t, const float* noise, float* sigma,
                                float* rgb, void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                                sparf_stream_t stream);
int sparf_mlp_backward_tape_rows(const SparfMLP* mlp, int32_t engine, int32_t R, int32_t S, const int64_t* rows,
                                 const float* origins, const float* dirs, const float* t, const float* sigma,
                                 const float* rgb, const float* d_sigma, const float* d_rgb, const SparfMLPGrad* grad,
                                 float* d_origins, float* d_dirs, void* tape, size_t tape_bytes, void* workspace,
                                 size_t workspace_bytes, sparf_stream_t stream);
/* Moving rows between a dense [.., width] layout and the compacted one of a grid pass (kept sample k < K is dense row
 * sample_idx[k], increasing, as sparf_occupancy_emit / sparf_contracted_emit write it), reading K (device int64) on the
 * device; C is the capacity of the compacted buffers, width in [1, 4].  No atomics, no synchronisation.
 *   scatter: dst[sample_idx[k]] = src[k] (the caller zeroes the skipped rows of dst);
 *   gather:  dst[k] = src[sample_idx[k]] (rows [K, C) of dst are not written);
 *   ray_sum: dst[r] (written, r < R) = the sum over the kept rows k of ray r (sample_idx[k] / S == r) of src[k], added
 *            in increasing k from 0: the per-ray gradients of origins and dirs from the per-sample ones. */
int sparf_compact_scatter(int64_t C, const int64_t* K, const int64_t* sample_idx, int32_t width, const float* src,
                          float* dst, sparf_stream_t stream);
int sparf_compact_gather(int64_t C, const int64_t* K, const int64_t* sample_idx, int32_t width, const float* src,
                         float* dst, sparf_stream_t stream);
int sparf_compact_ray_sum(int64_t R, int32_t S, int64_t C, const int64_t* K, const int64_t* sample_idx, int32_t width,
                          const float* src, float* dst, sparf_stream_t stream);

/* ---------------------------------------------------------------- early ray termination in training
 * A training pass (train / test-optim, with or without gradients; sparf_b200/termination.py train_forward_samples) over
 * the windows of the inference termination below, without a host round trip, with one tape and one backward per pass.
 *   kept set:  exactly the inference rule (same windows [k0, min(k0 + window, S)), the same tau update, op order and
 *              tau_max = fp32(-ln eps), a NaN tau stays alive, the box or contracted grid lookup when a grid is given),
 *              except that sigma is the training pass's own output: with density noise (drawn dense by the caller, as
 *              on the grid path) sigma = softplus(raw + noise).
 *   layout:    ends [W + 1] (device int64, W = ceil(S / window), ends[0] = 0 set by the caller).  Window w compacts its
 *              kept samples, in increasing r*S + k, to rows [ends[w], ends[w + 1]) of capacity-R*S buffers (sample_idx,
 *              origins_k, dirs_k, t_k): sparf_termination_append (box grid, or bits = NULL: none) and
 *              sparf_contracted_append take the arguments of the count / emit pair plus (ends, w), run count, scan and
 *              emit on one workspace (sparf_termination_workspace_bytes(R, k1 - k0)) and write ends[w + 1] = ends[w] + K_w.
 *              64-bit offsets, no atomics; rows outside [ends[w], ends[w + 1]) are not written.
 *   outputs:   sigma and rgb equal the dense training pass's with sigma = rgb = 0 at the skipped samples, bit for bit:
 *              every kept sample is evaluated as a one-sample ray by sparf_mlp_forward_tape_span.  Gradients are those of
 *              that masked pass; skipped samples get none.  One sparf_mlp_backward_tape_rows with rows = &ends[W] over
 *              capacity C = R*S runs the pass's backward.  d_origins / d_dirs (sparf_compact_ray_sum_segments) have the
 *              bits of sparf_compact_ray_sum over the same kept set; parameter gradients agree up to float atomic order.
 *   bounds:    against the non-terminated pass with the same t and noise, those of the inference termination below.
 *   host:      only W is known on the host; no count is read back, so a step that uses it can be one CUDA graph.
 * Tensor-core engines only (TC_3X, TC_1X, TC_3X_W1).
 *
 * sparf_mlp_forward_tape_span: sparf_mlp_forward_tape_rows over the device-side row span [*begin, min(*end, *begin +
 * cap)) of capacity-C buffers: it reads origins, dirs, t, noise and writes sigma, rgb and the tape's rows (the tape of C
 * rows, sparf_mlp_tape_bytes(C, 1)) at those global rows; cap sizes the chunk loop and the workspace
 * (sparf_mlp_workspace_bytes(cap, 1, 0)), whose images stay call-local.  The caller keeps *end <= C.  Rows outside the
 * span are neither read nor written.  sigma, rgb and the tape rows have the bits sparf_mlp_forward_tape_rows gives on
 * the same rows moved to row 0, so a tape written by several spans is read by one sparf_mlp_backward_tape_rows with
 * R = C and rows = the last span's end.
 * sparf_compact_scatter_span / _gather_span: sparf_compact_scatter / _gather over rows [ends[w], ends[w + 1]) only, at
 * most C (the window's capacity, R * window) of them.
 * sparf_compact_ray_sum_segments: sparf_compact_ray_sum over the W segments [ends[w], ends[w + 1]): per ray, the rows of
 * each segment in window order, each in increasing k, from 0. */
int sparf_mlp_forward_tape_span(const SparfMLP* mlp, int32_t engine, int32_t C, int32_t cap, const int64_t* begin,
                                const int64_t* end, const float* origins, const float* dirs, const float* t,
                                const float* noise, float* sigma, float* rgb, void* tape, size_t tape_bytes,
                                void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_compact_scatter_span(int64_t C, const int64_t* ends, int32_t w, const int64_t* sample_idx, int32_t width,
                               const float* src, float* dst, sparf_stream_t stream);
int sparf_compact_gather_span(int64_t C, const int64_t* ends, int32_t w, const int64_t* sample_idx, int32_t width,
                              const float* src, float* dst, sparf_stream_t stream);
int sparf_compact_ray_sum_segments(int64_t R, int32_t S, int32_t W, const int64_t* ends, const int64_t* sample_idx,
                                   int32_t width, const float* src, float* dst, sparf_stream_t stream);

/* ---------------------------------------------------------------- density queries
 * NeRF.compute_raw_density (frequency_nerf.py:149-170): the trunk alone at M arbitrary points [M,3] (x = p; no view
 * direction, no colour head).  Outputs raw [M], the density row before the softplus, without noise, and, when feat is
 * not NULL, feat [M,width] = relu of the last trunk layer's feature rows.  The BARF mask applies as in the MLP entry
 * points.  These calls read no head tensor: SparfMLP.head_* and SparfMLPGrad.head_* may be NULL.  M may exceed 2^31;
 * M = 0 is a no-op.  Engines as for the MLP (AUTO: TC_3X on sm_90, else SIMT_FP32).
 * sparf_density_workspace_bytes: `backward` = 0 sparf_density_forward, 1 sparf_density_backward, 2
 * sparf_density_gradient (never more than 1).  A forward without feat skips the last layer's feature GEMM (the density
 * row reads the layer below). */
size_t sparf_density_workspace_bytes(const SparfMLP* mlp, int64_t M, int32_t backward, int32_t engine);
int sparf_density_forward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, float* raw, float* feat,
                          void* workspace, size_t workspace_bytes, sparf_stream_t stream);
/* Backward of the above (recomputes the forward).  d_raw [M] and d_feat [M,width] may each be NULL (a zero gradient).
 * Trunk parameter gradients (+=) into grad's trunk fields and, when non-NULL, d_points [M,3] (+=). */
int sparf_density_backward(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, const float* d_raw,
                           const float* d_feat, const SparfMLPGrad* grad, float* d_points, void* workspace,
                           size_t workspace_bytes, sparf_stream_t stream);
/* The point gradient of the density: grad_points [M,3] (written, not added) = d raw / d x at each point, raw as
 * sparf_density_forward computes it (no noise, the BARF mask at progress); normals are -grad_points / |grad_points|.
 * It equals, bit for bit, the d_points sparf_density_backward adds to zeros for d_raw = 1 and d_feat = NULL, on every
 * engine: the same input-gradient kernels on the same operand images, each ReLU mask H > 0 read from the recomputed fp32
 * activations instead of the bits the weight-gradient GEMMs write.  It computes no weight or bias gradient (no
 * SparfMLPGrad) and reads no head tensor.  M = 0 is a no-op; M may exceed 2^31.  Workspace:
 * sparf_density_workspace_bytes(mlp, M, 2, engine). */
int sparf_density_gradient(const SparfMLP* mlp, int32_t engine, int64_t M, const float* points, float* grad_points,
                           void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- marching cubes
 * A triangle mesh of the iso-surface of a dense fp32 volume vol [nx][ny][nz] (row-major, k fastest), in index space,
 * vertex-deduplicated: what mcubes.marching_cubes(volume, iso) returns, computed on the device.  Mesh extraction from a
 * density grid (BARF's extract_mesh over opt.trimesh; sparf_b200/mesh.py).
 *   inside:    vol >= iso (NaN is outside).  Cell (i,j,k), i < nx-1, j < ny-1, k < nz-1, has case index
 *              sum over corners c of inside(corner c) << c, corner c at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1).
 *   vertices:  one per crossing lattice edge (one end inside, one outside), owned by its lower end p and its axis a, at
 *              p + s e_a with s = (iso - vol[p]) / (vol[p + e_a] - vol[p]) in fp32; the coordinate along a is
 *              float(p_a) + s, the others are exact.  Ordered by (linear index of p, a).
 *   triangles: cells in linear order, each cell's triangles in table order; int64 vertex ids.  (v1 - v0) x (v2 - v0)
 *              points from the inside toward the outside.  Where no lattice point on the volume's border is inside, the
 *              mesh is closed and consistently oriented: every undirected edge lies in exactly two triangles, once in
 *              each direction.
 * Deterministic (identical bytes on every run).  Non-finite values cause no out-of-bounds access; only the mesh near
 * them is unspecified.  Every extent must be >= 2 (SPARF_ERR_INVALID otherwise).
 * Two calls on one stream with one workspace: sparf_mcubes_count writes totals [2] = {V, F} (device int64) and leaves
 * per-point offsets in the workspace; sparf_mcubes_emit, enqueued after it on the same stream with the same volume, iso
 * and workspace, reads them and writes verts [V,3] fp32 and faces [F,3] int64.  The caller reads the totals to size
 * the outputs.  Neither call synchronises; both are capturable.  Workspace: 8 B per lattice point + 16 B per 2048
 * points (0 for an invalid extent). */
#define SPARF_MCUBES_MAX_TRIS 5
size_t sparf_mcubes_workspace_bytes(int64_t nx, int64_t ny, int64_t nz);
int sparf_mcubes_count(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, int64_t* totals, void* workspace,
                       size_t workspace_bytes, sparf_stream_t stream);
int sparf_mcubes_emit(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, float* verts, int64_t* faces,
                      void* workspace, size_t workspace_bytes, sparf_stream_t stream);
/* Masked marching cubes: the same two-call contract, workspace and arguments, for volumes whose unobserved points are
 * NaN (the TSDF volumes of sparf_tsdf_integrate).  A cell with a non-finite corner emits no triangle, and a vertex is
 * emitted only if an emitted triangle uses it; the remaining vertices keep the dense order (linear index of the owner
 * point p, then axis) and are renumbered 0, 1, ...; positions, triangle order and orientation are the dense ones.  So on
 * a volume without NaN or infinity the output is byte-identical to sparf_mcubes_count / _emit's, and where observed
 * inside space meets unobserved space no false surface appears. */
int sparf_mcubes_count_masked(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, int64_t* totals,
                              void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_mcubes_emit_masked(const float* vol, int64_t nx, int64_t ny, int64_t nz, float iso, float* verts,
                             int64_t* faces, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
/* Host only: the case table, table [256][3 * SPARF_MCUBES_MAX_TRIS] (host int8).  Row c lists the triangles of case c
 * as cell-edge ids, three per triangle, padded with -1.  Edge e = 4a + m runs along axis a from the corner whose
 * offsets along the two other axes b < b' are (m & 1, m >> 1); its vertex is owned by that corner.  The table is
 * generated from one rule per cube face (sparf_b200/csrc/mcubes_table.py): inside corners never connect across a face,
 * so two cells sharing a face cut it the same way. */
int sparf_mcubes_table(int8_t* table);

/* ---------------------------------------------------------------- sparse marching cubes
 * The mesh of the same lattice as above for res large enough that the dense volume does not fit, with the density
 * evaluated only in blocks near the surface (sparf_b200/mesh.py, extract_mesh_sparse).
 *   lattice:   BARF's, [res+1]^3 points over axis [res+1] (fp32, host-computed linspace(r0, r1, res+1); axis 0 = x).
 *              res is a multiple of B = SPARF_MCUBES_BLOCK = 8 in [8, 8192].  Block b = (bi, bj, bk), nb = res / 8 per
 *              axis, linear index (bi*nb + bj)*nb + bk, owns the lattice points [8b, 8b+8] on each axis ((B+1)^3 = 729,
 *              faces shared with its neighbours) and the 8^3 cells between them.
 *   coarse:    sigma [nb+1]^3 at the lattice points whose indices are all multiples of 8 (axis[::8]).
 *   active:    block b is active iff the coarse points with indices [b-1, b+2] per axis, clipped to [0, nb], contain a
 *              NaN, or both a value >= iso and a value < iso (the occupancy build's dilation-1 window, over blocks).
 *              A feature smaller than a block that no coarse point of a window sees is missed: this is the trade-off
 *              against the dense extractor.
 *   output:    the dense mesh (sparf_mcubes_count / _emit) of the full lattice without the triangles of cells in
 *              inactive blocks and without the vertices no remaining triangle uses; the remaining vertices keep their
 *              order (linear index of the owner point p, then axis) and are renumbered 0, 1, ...; positions, triangle
 *              order and orientation are the dense ones.  So when every cell with a crossing lies in an active block,
 *              the output is byte-identical to the dense one.  Deterministic; 64-bit ids.
 * Classification: sparf_mcubes_sparse_classify reads coarse and writes slots [nb^3] (int32: -1 for an inactive block,
 * else the block's rank among the active blocks in linear order) and n_active (device int64).  The caller reads
 * n_active; sparf_mcubes_sparse_blocks then writes block_ids [n_active] (int64, increasing).  Workspace:
 * sparf_mcubes_sparse_workspace_bytes(res, 0, 0).
 * Points: sparf_mcubes_sparse_points writes points [n_blocks * 729][3] for the active blocks [b0, b0 + n_blocks): per
 * block its 729 points, k fastest, point (i, j, k) = (axis[i], axis[j], axis[k]).  axis is a device copy.
 * Marching cubes: sigma_blocks [n_active][9][9][9] (fp32; the density at those points), slots and block_ids as above.
 * sparf_mcubes_sparse_count writes totals [2] = {V, F} (device int64) with a workspace of
 * sparf_mcubes_sparse_workspace_bytes(res, n_active, 0) bytes.  sparf_mcubes_sparse_emit writes verts [V][3] (fp32,
 * index space) and faces [F][3] (int64) into buffers of max_verts and max_faces rows, with a workspace of
 * sparf_mcubes_sparse_workspace_bytes(res, n_active, max_verts) bytes; it recomputes what it needs and takes nothing
 * from count but the caller's capacities, so max_verts >= V and F <= max_faces <= 2560 n_active (5 triangles per
 * cell) are required; rows past the capacities are never written.  Both are capturable and neither synchronises.
 * Workspace: the larger of 4 B per block (the classification's flags) and 8 B x (2 + 128) per active block + 44 B per
 * vertex of capacity, plus scan / sort scratch; 0 for invalid sizes (res, n_active > nb^3, 64 n_active or max_verts
 * >= 2^31) and where no CUDA device is current (the scratch is sized for the device).  Invalid arguments give
 * SPARF_ERR_INVALID.  sparf_mcubes_sparse_blocks needs no call when n_active is 0. */
#define SPARF_MCUBES_BLOCK 8
size_t sparf_mcubes_sparse_workspace_bytes(int32_t res, int64_t n_active, int64_t max_verts);
int sparf_mcubes_sparse_classify(const float* coarse, int32_t res, float iso, int32_t* slots, int64_t* n_active,
                                 void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_mcubes_sparse_blocks(const int32_t* slots, int32_t res, int64_t* block_ids, sparf_stream_t stream);
int sparf_mcubes_sparse_points(const float* axis, int32_t res, const int64_t* block_ids, int64_t b0, int64_t n_blocks,
                               float* points, sparf_stream_t stream);
int sparf_mcubes_sparse_count(const float* sigma_blocks, int32_t res, const int32_t* slots, const int64_t* block_ids,
                              int64_t n_active, float iso, int64_t* totals, void* workspace, size_t workspace_bytes,
                              sparf_stream_t stream);
int sparf_mcubes_sparse_emit(const float* sigma_blocks, int32_t res, const int32_t* slots, const int64_t* block_ids,
                             int64_t n_active, float iso, int64_t max_verts, int64_t max_faces, float* verts,
                             int64_t* faces, void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- TSDF fusion
 * Coloured meshes from rendered depth and colour maps (sparf_b200/tsdf.py): the maps of B views are integrated into a
 * truncated signed distance volume, whose zero level the masked marching cubes above extracts.
 *   volume:    BARF's lattice, n points per axis at axis [n] (fp32, device; mesh.lattice_axis(res, range), n = res + 1),
 *              point (i, j, k) = (axis[i], axis[j], axis[k]), linear index (i*n + j)*n + k (axis 0 = x, k fastest).  The
 *              caller owns the state: tsdf [n^3] (initially 1), weight [n^3] (initially 0), color [n^3][3] (initially 0).
 *   views:     pose_w2c [B,3,4] = (R | t), intr [B,3,3] = K (its last row is taken to be (0, 0, 1)), depth [B,H,W] =
 *              camera z-depth (the renderer's t: a camera-space ray has z = 1), rgb [B,H,W,3] or NULL, valid [B,H,W]
 *              (uint8, nonzero = valid) or NULL = all valid.
 *   rule:      every lattice point p takes the views b = 0 .. B-1 in order, each op rounded to nearest (no FMA):
 *                x_r = __fadd_rn(__fadd_rn(__fadd_rn(R_r0 p_x, R_r1 p_y), R_r2 p_z), t_r)   (products __fmul_rn)
 *                skip the view unless x_z > 0;
 *                u = __fdiv_rn(K_00 x_x + K_01 x_y + K_02 x_z, x_z), v = __fdiv_rn(K_10 x_x + K_11 x_y + K_12 x_z, x_z)
 *                    (the sums left to right, as x_r's); skip unless 0 <= u < W and 0 <= v < H;
 *                pixel (floor u, floor v): this inverts the ray generation above, whose pixel centres sit at +0.5, so
 *                    a point on the ray of pixel (i, j) lands in pixel (i, j);
 *                skip if valid is 0 there, or unless d = depth[b, floor v, floor u] is finite and > 0;
 *                s = __fsub_rn(d, x_z); skip if s < -trunc (the point is occluded);
 *                f = min(1, __fdiv_rn(s, trunc)); W' = W + 1; tsdf += (f - tsdf) / W'; color += (rgb - color) / W' per
 *                    channel, only when rgb is given; W = W'.
 *              The updates equal (W tsdf + f) / (W + 1) and (W color + rgb) / (W + 1); written as increments they leave
 *              a value that every view observes alike exactly unchanged.  Observation weight 1.
 *   writes:    each point's state once, after all views: no atomics, deterministic, no synchronisation, capturable.
 *              color is neither read nor written when rgb is NULL (it may then be NULL).
 * SPARF_ERR_INVALID for n < 2 or n^3 > 2^38, trunc not finite or <= 0, B, H or W < 1, H or W > 2^24, B*H*W > 2^60, and
 * NULL for a required pointer. */
int sparf_tsdf_integrate(const float* axis, int32_t n, float trunc, int32_t B, int32_t H, int32_t W,
                         const float* pose_w2c, const float* intr, const float* depth, const float* rgb,
                         const uint8_t* valid, float* tsdf, float* weight, float* color, sparf_stream_t stream);

/* ---------------------------------------------------------------- mesh components
 * Floater removal for the meshes above (sparf_b200/mesh.py, keep_components): the connected components of a triangle
 * mesh, and the mesh of a chosen subset of them.  The extractors' meshes are vertex-welded (one vertex per crossing
 * lattice edge), so connectivity is read from the face ids alone.
 *   input:       faces [F][3] (int64) over V vertices, every id in [0, V); 0 <= V, F <= INT32_MAX, F = 0 when V = 0.
 *                Ids outside [0, V) cause no out-of-bounds access; the results are then unspecified.
 *   connected:   two vertices are connected when some face holds both; the components are the connected classes of
 *                vertices, so two triangles that share one vertex are in one component.  A vertex that no face uses is
 *                a component of its own (with 0 faces); degenerate faces (repeated ids) are allowed.
 *   labels:      labels [V] (int32): a component's label is the rank of its smallest vertex id among all components'
 *                smallest vertex ids, so labels run 0 .. C-1 in order of first vertex.  The definition depends neither
 *                on the schedule nor on the order of the faces: identical bytes on every run.
 *   face counts: face_counts [C] (int64): the faces of each component, counted by the label of each face's first
 *                vertex (integer atomics: deterministic).
 *   selection:   keep [C] (uint8, nonzero = kept).  The kept vertices (those of kept components) in their original
 *                order are renumbered 0 .. V'-1, vert_ids [V'] (int64, increasing) gets each one's old id, and the kept
 *                faces (those whose first vertex is kept) are written in their original order with renumbered ids,
 *                faces_out [F'][3] (int64).  labels must be sparf_mesh_components' labels of the same faces.
 * sparf_mesh_components writes labels and n_components (device int64, C); the caller reads C to size face_counts and
 * keep.  sparf_mesh_component_faces zeroes and fills face_counts.  sparf_mesh_select_count writes totals [2] = {V', F'}
 * (device int64) and leaves the output offsets in the workspace; sparf_mesh_select_emit, enqueued after it on the same
 * stream with the same arguments and workspace, writes vert_ids and faces_out.  Workspace (shared by all calls):
 * sparf_mesh_components_workspace_bytes(V, F), 4 B per vertex + 4 B per face + scan scratch; 0 for invalid sizes and
 * where no CUDA device is current (the scratch is sized for the device).  No call synchronises; all are capturable.  No
 * kernel runs over an empty vertex or face set; the device counts are still written.  Invalid sizes (also C > V) give
 * SPARF_ERR_INVALID. */
size_t sparf_mesh_components_workspace_bytes(int64_t n_verts, int64_t n_faces);
int sparf_mesh_components(const int64_t* faces, int64_t n_faces, int64_t n_verts, int32_t* labels, int64_t* n_components,
                          void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_mesh_component_faces(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                               int64_t n_components, int64_t* face_counts, sparf_stream_t stream);
int sparf_mesh_select_count(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                            const uint8_t* keep, int64_t n_components, int64_t* totals, void* workspace,
                            size_t workspace_bytes, sparf_stream_t stream);
int sparf_mesh_select_emit(const int64_t* faces, int64_t n_faces, int64_t n_verts, const int32_t* labels,
                           const uint8_t* keep, int64_t n_components, int64_t* vert_ids, int64_t* faces_out,
                           void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- mesh simplification
 * Quadric-error edge collapses (Garland-Heckbert) down to a face budget (sparf_b200/mesh.py, simplify), in parallel
 * rounds whose every decision is a minimum or a sort: the result does not depend on the schedule.
 *   input:     vertices [V][3] (fp32), faces [F][3] (int64, ids in [0, V): the caller checks), attrs [V][A] (fp32,
 *              A >= 0, interpolated, not part of the error); V <= INT32_MAX, F <= INT32_MAX / 3.  Open, non-manifold and
 *              degenerate input is allowed.
 *   classes:   each round, over the live faces: an edge is interior in exactly 2 of them, boundary in 1, non-manifold in
 *              3 or more; a vertex is locked on a non-manifold edge or a face with repeated ids, boundary on a boundary
 *              edge.  Locked vertices never move and are never removed; boundary vertices never move.
 *   quadrics:  per face, with c = (p1 - p0) x (p2 - p0) in fp64, n = c / |c|, n4 = (n, -n.p0), w = |c| / 2:
 *              q_ij = (w n4_i) n4_j for ij = 00 01 02 03 11 12 13 22 23 33 (0 when |c| = 0).  Q[v] = the sum over v's
 *              faces in increasing face id.  Every fp64 operation is rounded on its own (no FMA contraction).
 *   edges:     indexed by rank among the unique (lo, hi) id pairs of the live faces.  (a, b), a < b, is collapsible when
 *              interior, neither end locked, not both boundary; valid when also (link condition) its faces abc and abd
 *              have c != d, a and b have no common neighbour but c and d, and not both acd and bcd are faces; and
 *              (fold check) every live face around a or b that does not hold both and has a nonzero old normal
 *              (p1 - p0) x (p2 - p0) keeps a positive dot product of its new (end replaced by v*) and old normals.
 *   v*:        (fp32) with one boundary end, that end (it survives); else the minimiser of v^T (Q[a] + Q[b]) v by
 *              Cramer's rule when |det A| > 1e-10 tr(A)^3 and |v* - mid|^2 <= |b - a|^2 (mid = (a + b) / 2); else the
 *              cheapest of a, b, fp32(mid), ties in that order.  cost = fp32(max(v*^T Q v*, 0)), key = cost bits << 32 | e.
 *   round:     k = ceil((F_live - target) / 2); the candidates are the k valid edges with the smallest keys (all valid
 *              edges when fewer).  Each candidate atomicMin's its key onto every vertex of every live face around a or
 *              b, and wins when it holds all of them.  A winner collapses into s (its boundary end, else a; r the
 *              other): pos[s] = v*, Q[s] = Q[s] + Q[r], attrs[s] = fp32(attrs[a] + t (attrs[b] - attrs[a])) with t the
 *              projection of v* on a -> b clamped to [0, 1] (0 when a = b in space); its 2 faces die, r becomes s in
 *              the others, and the live faces are compacted in their order.
 *   output:    the vertices never removed, in increasing id (vert_ids [V'] int64, V' = V - the collapses), their
 *              positions and attrs, and the live faces in input order with renumbered ids (int64).
 * sparf_mesh_simplify_init copies the input into the workspace and builds the quadrics; counts [2] (device int64) =
 * {F, 0}.  sparf_mesh_simplify_round (n_live = counts[0] as last read, k >= 1) runs one round and writes counts =
 * {F_live, winners}; the caller stops when F_live <= target or winners = 0.  sparf_mesh_simplify_emit (n_live = F_live)
 * writes the output.  With no round the output is the input, byte for byte.  Workspace (one for all three calls):
 * sparf_mesh_simplify_workspace_bytes(V, F, A) = 110 + 4A B per vertex + 145 B per face + sort / scan scratch over 3F
 * entries; 0 for invalid sizes and where no CUDA device is current.  No call synchronises; all are capturable.
 * Invalid sizes or NULL pointers give SPARF_ERR_INVALID. */
size_t sparf_mesh_simplify_workspace_bytes(int64_t n_verts, int64_t n_faces, int32_t n_attrs);
int sparf_mesh_simplify_init(const float* vertices, const int64_t* faces, const float* attrs, int64_t n_verts,
                             int64_t n_faces, int32_t n_attrs, int64_t* counts, void* workspace,
                             size_t workspace_bytes, sparf_stream_t stream);
int sparf_mesh_simplify_round(int64_t n_verts, int64_t n_faces, int32_t n_attrs, int64_t n_live, int64_t k,
                              int64_t* counts, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_mesh_simplify_emit(int64_t n_verts, int64_t n_faces, int32_t n_attrs, int64_t n_live, float* vertices,
                             float* attrs, int64_t* vert_ids, int64_t* faces, void* workspace, size_t workspace_bytes,
                             sparf_stream_t stream);

/* ---------------------------------------------------------------- mesh distance
 * Exact closest-point queries against a target surface (sparf_b200/mesh.py, compare: Chamfer distance and F-score):
 * for each query point the nearest primitive of a triangle mesh or a point cloud, found over a uniform grid.
 *   target:  vertices [V][3] (fp32, finite) and either faces [F][3] (int64; a triangle target, F >= 0) or n_faces = -1
 *            (a point target: the primitives are the vertices).  0 <= V, F <= INT32_MAX; F > 0 needs V > 0.  A face with
 *            an id outside [0, V) is never found (no out-of-bounds access).
 *   grid:    the box is the target's bounding box (over all V vertices, NaN coordinates skipped) padded on every side
 *            by max(1e-3 of its largest extent, 1e-6 of its largest |coordinate|, 1e-20), so flat targets get a
 *            volume.  Cells per axis: given (each >= 1, at most 2^24 cells), or automatic (all 0): with P primitives,
 *            about T = min(2^24, P^1.5) cubic cells of side h = cbrt(box volume / T), n_a = clamp(ceil(extent_a / h), 1,
 *            2^24), h grown by 1.25x until at most 2^24 cells.  A surface sampled by P primitives crosses about P^(2/3)
 *            ... P of such cells, so a crossed cell holds about one point or a few triangle entries.  The cell size
 *            per axis is extent_a / n_a.  A point is entered in its one cell; a triangle in every cell its bounding box
 *            overlaps (cell of x = clamp(floor((x - lo) / cell), 0, n - 1) in fp32).  CSR: cell_start [n_cells + 1]
 *            (int32) and prims [entries] (int32 primitive ids, increasing within a cell); entries <= INT32_MAX.
 *   query:   points [N][3] (fp32) -> dist [N] (fp32), index [N] (int64), closest [N][3] (fp32): the minimum over every
 *            primitive of (d, id), d = sqrt(|p - q|^2) with q the primitive's closest point to p, ties to the
 *            smallest id; a miss (no primitive with d <= max_dist) gives inf / -1 / NaN.  q of a point is the point;
 *            of a triangle abc the nearest of: the projection onto its plane when n = ab x ac != 0 and the projection
 *            lies inside (face region; preferred on ties), and the clamped projections onto ab, bc, ca (edge and vertex
 *            regions; ties in that order), so zero-area, collinear and repeated-vertex triangles are exact too.  Every
 *            fp32 operation of it is rounded on its own: d and q are one function of (p, primitive), and the result is
 *            the same bytes for every grid, including 1 x 1 x 1 (brute force).  The search visits Chebyshev shells of
 *            cells around p's clamped cell and stops once every plane bounding the visited cells lies farther from p
 *            than min(d_best, max_dist) (strictly, after shrinking the bound by 2^-18 (|p|_inf + the box's largest
 *            |coordinate|) for rounding), or the whole grid is visited.  max_dist >= 0 (+inf allowed).
 * sparf_distance_grid_count writes *grid (device) and totals [2] = {entries, n_cells} (device int64) with a workspace of
 * sparf_distance_grid_workspace_bytes(P, 0); the caller reads the totals to size cell_start and prims, and
 * sparf_distance_grid_fill, with the same target and grid and a workspace of sparf_distance_grid_workspace_bytes(P,
 * entries) (8 B per primitive + 12 B per entry + scan / sort scratch; 0 for invalid sizes and where no CUDA device is
 * current), writes them.  sparf_distance_query reads the target, grid, cell_start and prims and needs no workspace.  No
 * call synchronises; all are capturable.  An empty target (P = 0) gives an all-zero grid, totals {0, 0}, cell_start
 * [1] = {0}, and a query of all misses; N = 0 is a no-op; no kernel runs over an empty set.  Invalid sizes, max_dist < 0 or NaN, and NULL pointers
 * give SPARF_ERR_INVALID. */
typedef struct SparfDistanceGrid {
  float lo[3];       /* the padded box's low corner */
  float cell[3];     /* the cell size per axis */
  int32_t dims[3];   /* cells per axis (all 0 for an empty target) */
  int32_t reserved;
} SparfDistanceGrid;
size_t sparf_distance_grid_workspace_bytes(int64_t n_prims, int64_t n_entries);
int sparf_distance_grid_count(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                              int32_t cells_x, int32_t cells_y, int32_t cells_z, SparfDistanceGrid* grid,
                              int64_t* totals, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_distance_grid_fill(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                             const SparfDistanceGrid* grid, int64_t n_cells, int64_t n_entries, int32_t* cell_start,
                             int32_t* prims, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_distance_query(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                         const SparfDistanceGrid* grid, const int32_t* cell_start, const int32_t* prims,
                         const float* points, int64_t n_points, float max_dist, float* dist, int64_t* index,
                         float* closest, sparf_stream_t stream);

/* ---------------------------------------------------------------- mesh ray cast
 * First hits of rays on a triangle mesh (sparf_b200/mesh.py: render, visible_faces, cull) over the grid, cell_start and
 * prims of sparf_distance_grid_count / _fill for that mesh (n_faces >= 0; a point grid is refused).
 *   rays:    origins [N][3], dirs [N][3] (fp32; d need not be unit: t is in units of d, so a pixel ray of raygen with
 *            camera-space z = 1 gives t = camera z-depth) -> t [N] (fp32), face [N] (int64), bary [N][3] (fp32): the
 *            minimum over every triangle of (t, id) with t_min <= t <= t_max, ties to the smallest id, and the hit's
 *            barycentrics (U, V, W) / det of the face's vertices 0, 1, 2 (each in [0, 1], summing to 1 up to rounding).
 *            A miss gives inf / -1 / NaN; so does a ray with a non-finite component or d = 0.
 *   hit:     the watertight test of Woop, Benthin and Wald (JCGT 2013): k = the axis of the largest |d| (the first on
 *            ties), kx = k + 1, ky = k + 2 (mod 3); per vertex A = v - o, Ax = A[kx] - (d[kx] / d[k]) A[k], Ay likewise,
 *            Az = (1 / d[k]) A[k]; U = Cx By - Cy Bx, V = Ax Cy - Ay Cx, W = Bx Ay - By Ax,
 *            recomputed in fp64 from the same fp32 Ax .. Cy when any is exactly 0; a hit when U, V, W are all >= 0 or
 *            all <= 0, det = U + V + W != 0 and (b - a) x (c - a) != 0 exactly (in fp64: a zero-area triangle is never
 *            hit); t = (U Az + V Bz + W Cz) / det.  Every fp32 operation is rounded on its own (no contraction): the hit
 *            is one function of (ray, triangle), and a shared edge gives exactly opposite edge functions in its two
 *            triangles, so a ray through an edge or vertex of a closed mesh cannot pass between them.  Triangles are
 *            two-sided.  A face with an id outside [0, V) is never hit.
 *   walk:    the slabs of cells perpendicular to k in ray order, clipped to [t_min, t_max] and the grid's box; in each,
 *            the cells the ray's segment in the slab covers (padded by 2^-18 (|o|_inf + the box's largest
 *            |coordinate|)); after each slab it stops once the slab's far plane, moved back by 2^-14 of that scale, gives
 *            a t that, shrunk by 2^-20 of itself, is strictly greater than the best.  The result is the same bytes for every grid, including 1
 *            x 1 x 1 (brute force); DESIGN §3.1.15 gives the argument.
 * No workspace.  No call synchronises; it is capturable.  N = 0 is a no-op; an empty mesh (F = 0) gives all misses.
 * Invalid sizes, t_min < 0, t_max < t_min, NaN bounds and NULL pointers give SPARF_ERR_INVALID. */
int sparf_raycast(const float* vertices, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                  const SparfDistanceGrid* grid, const int32_t* cell_start, const int32_t* prims,
                  const float* origins, const float* dirs, int64_t n_rays, float t_min, float t_max, float* t,
                  int64_t* face, float* bary, sparf_stream_t stream);

/* ---------------------------------------------------------------- occupancy grid
 * Empty-space skipping for inference renders (sparf_b200/occupancy.py): a bitfield over the box [r0, r1]^3 split into
 * res^3 cells, built from the density lattice sigma [res+1]^3 of mesh.density_grid (lattice point (a,b,c) at
 * linspace(r0, r1, res+1)[a, b, c], axis 0 = x, c fastest), and a per-sample lookup that compacts the samples a render
 * must evaluate into the inputs of sparf_mlp_forward.
 *   cells:   cell (i,j,k) has linear index (i*res + j)*res + k and is bit idx & 31 of word idx >> 5 of
 *            bits [ceil(res^3 / 32)] (uint32).  Bits past res^3 in the last word are 0.
 *   build:   a cell is occupied iff a lattice point within one cell of it, indices [c-1, c+2] on each axis clipped to
 *            [0, res], has sigma >= thres or NaN: the corners of the cell and of its 26 neighbours (dilation radius 1).
 *   lookup:  sample (r,k) is at x = o[r] + t[r,k] * d[r] per axis in the fp32 op order of the MLP encoder
 *            (__fadd_rn(o, __fmul_rn(d, t))); u = __fmul_rn(__fdiv_rn(__fsub_rn(x, r0), __fsub_rn(r1, r0)), res).
 *            The sample is KEPT if any u is NaN, < 0 or >= res (outside the box: always evaluated) or if cell
 *            ((int)u_x, (int)u_y, (int)u_z) is occupied; otherwise it is skipped.
 * sparf_occupancy_build writes bits; it needs no workspace.  1 <= res <= 4096.
 * Compaction: two calls on one stream with one workspace (sparf_occupancy_workspace_bytes(R, S): 4 B per 4 samples + 8 B
 * per 2048 samples, 0 for invalid sizes).  sparf_occupancy_count reads origins, dirs [R,3], t [R,S] and the bits, and
 * writes K (device int64) = the number of kept samples, leaving tile-local offsets in the workspace.
 * sparf_occupancy_emit, enqueued after it with the same arguments and workspace, writes for the kept samples, in
 * increasing order of r*S + k: sample_idx [K] (int64, r*S + k), origins_k, dirs_k [K,3] (the ray's o and d) and t_k [K]
 * (t[r,k]): sparf_mlp_forward with R = K, S = 1 on them evaluates exactly the kept samples.  The caller reads K to size
 * the outputs.  R * S may exceed 2^31 (offsets are 64-bit); R = 0 gives K = 0.  No atomics: the output is
 * deterministic.  Neither call synchronises; both are capturable. */
int sparf_occupancy_build(const float* sigma, int32_t res, float thres, uint32_t* bits, sparf_stream_t stream);
size_t sparf_occupancy_workspace_bytes(int64_t R, int32_t S);
int sparf_occupancy_count(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t,
                          const uint32_t* bits, int32_t res, float r0, float r1, int64_t* K, void* workspace,
                          size_t workspace_bytes, sparf_stream_t stream);
int sparf_occupancy_emit(int64_t R, int32_t S, const float* origins, const float* dirs, const float* t,
                         const uint32_t* bits, int32_t res, float r0, float r1, int64_t* sample_idx, float* origins_k,
                         float* dirs_k, float* t_k, void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- early ray termination
 * Inference renders stop evaluating a ray once it is opaque (sparf_b200/termination.py).  A pass's S samples per ray
 * are split into windows [k0, min(k0 + window, S)), k0 = 0, window, 2*window, ...; every ray is alive in the first.
 * A window evaluates (the MLP) the samples of the alive rays, and with an occupancy grid only those the grid keeps;
 * every other sample counts as sigma = 0, rgb = 0.  After each window every alive ray r adds the window's optical
 * depth to its running tau[r] (fp32, 0 at the start), sequentially in k, each op rounded to nearest (no contraction):
 *   len  = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)))   (d = dirs[r])
 *   gap  = k + 1 < S ? __fsub_rn(t[r,k+1], t[r,k]) : 1e10f
 *   tau  = __fadd_rn(tau, __fmul_rn(sigma[r,k], __fmul_rn(gap, len)))
 * with sigma [R,S] the pass's output so far (0 at every skipped sample, so 0 * inf gives a NaN tau).  The ray dies
 * when tau > tau_max, where tau_max = fp32(-ln eps) is computed by the caller (eps = 0: +inf, nothing dies); a NaN
 * tau keeps the ray alive.  A dead ray's later samples are all skipped.  The composite of such a pass differs from the
 * dense one (same t) only by the mass behind a transmittance exp(-tau) < eps: |d opacity| < eps, |d rgb| < eps (2 eps
 * with an opaque background), |d depth| < eps * max t, up to the composite's own fp32 rounding.
 * Compaction of one window: sparf_termination_count / _emit, the two-call contract of sparf_occupancy_count / _emit
 * (same outputs, in increasing order of r*S + k, one workspace) over the samples k in [k0, k1) of the rays with
 * alive[r] != 0 (uint8 [R]; NULL = all alive).  bits = NULL: no grid (res, r0, r1 ignored); otherwise a sample must
 * also be KEPT by the occupancy lookup above.  Workspace: sparf_termination_workspace_bytes(R, k1 - k0) (the
 * occupancy workspace of R x (k1 - k0) samples; 0 for invalid sizes).  0 <= k0 < k1 <= S.
 * sparf_termination_update: for each ray with alive[r] != 0, adds the samples k in [k0, k1) to tau [R] (in / out) as
 * above and clears alive[r] when tau > tau_max.  Rays with alive[r] == 0 are untouched.
 * No atomics; none of the calls synchronises.  A render's loop over the windows reads K once per window on the host,
 * so that loop cannot be captured into a CUDA graph. */
size_t sparf_termination_workspace_bytes(int64_t R, int32_t window);
int sparf_termination_count(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                            const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, float r0, float r1,
                            int64_t* K, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_termination_emit(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                           const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, float r0, float r1,
                           int64_t* sample_idx, float* origins_k, float* dirs_k, float* t_k, void* workspace,
                           size_t workspace_bytes, sparf_stream_t stream);
int sparf_termination_update(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* sigma, const float* t,
                             const float* dirs, float tau_max, float* tau, uint8_t* alive, sparf_stream_t stream);
/* the appending compaction of window w for training termination (section above sparf_mlp_forward_tape_span) */
int sparf_termination_append(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                             const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, float r0, float r1,
                             int64_t* ends, int32_t w, int64_t* sample_idx, float* origins_k, float* dirs_k, float* t_k,
                             void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- contracted occupancy grid
 * An occupancy grid over all of space for inverse-depth and unbounded scenes (sparf_b200/occupancy.py with
 * contraction = (center, radius)): the world is mapped (mip-NeRF 360's contraction, in the inf-norm) into the cube
 * [-2, 2]^3, and the grid's res^3 cells split that cube.  center[3] and radius (fp32) set the map; the cells and bits
 * are laid out as the box grid's above.
 *   lookup:  sample (r,k), every op rounded to nearest (no contraction into FMAs), per axis a:
 *              x_a = __fadd_rn(o_a, __fmul_rn(d_a, t))              (the MLP encoder's x, as in the box lookup)
 *              y_a = __fdiv_rn(__fsub_rn(x_a, c_a), radius),  m = max_a |y_a|
 *              v_a = y_a if m <= 1, else __fmul_rn(__fmul_rn(y_a, q), __fsub_rn(2, q)) with q = __fdiv_rn(1, m)
 *              u_a = __fmul_rn(__fmul_rn(__fadd_rn(v_a, 2), 0.25f), (float)res)
 *            The sample is KEPT if any u_a is NaN or outside [0, res), or if cell ((int)u_x, (int)u_y, (int)u_z) is
 *            occupied; otherwise it is skipped.  Infinite or NaN coordinates give a NaN u: kept.  For m > 2^24,
 *            __fsub_rn(2, q) rounds to 2, so u can reach exactly res: kept as well.
 *   build:   the lattice axis is linspace(-2, 2, res+1) in fp32 (mesh.lattice_axis).  Lattice point v with
 *            n = ||v||_inf < 2 stands for the world point center + radius * y, y = v for n <= 1 and v / (n (2 - n))
 *            beyond (the inverse of the lookup's map); sigma there is the softplus of sparf_density_forward, as in
 *            mesh.density_grid.  Points with n = 2 lie at infinity and are not evaluated: their sigma is NaN.  The
 *            unchanged sparf_occupancy_build (dilation 1, NaN occupied) then writes the bits, so the outer two-cell
 *            shell (a cell index 0, 1, res-2 or res-1 on some axis) is always occupied: samples with
 *            ||x - center||_inf >= radius / (2 - (2 - 8 / res)) = radius * res / 8 (res >= 8) are always evaluated.
 * Compaction of one window: sparf_contracted_count / _emit, the two-call contract of sparf_termination_count / _emit
 * (same outputs in increasing order of r*S + k, same workspace, sparf_termination_workspace_bytes(R, k1 - k0);
 * 0 <= k0 < k1 <= S; alive NULL = all alive) with the contracted lookup in place of the box lookup.  With alive = NULL,
 * k0 = 0 and k1 = S it is the plain grid compaction.  bits is required (when R > 0), 1 <= res <= 4096, center is a
 * host float[3] of finite values read during the call, radius is finite and > 0.  No atomics; neither call
 * synchronises. */
int sparf_contracted_count(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                           const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, const float* center,
                           float radius, int64_t* K, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_contracted_emit(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                          const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, const float* center,
                          float radius, int64_t* sample_idx, float* origins_k, float* dirs_k, float* t_k,
                          void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_contracted_append(int64_t R, int32_t S, int32_t k0, int32_t k1, const float* origins, const float* dirs,
                            const float* t, const uint8_t* alive, const uint32_t* bits, int32_t res, const float* center,
                            float radius, int64_t* ends, int32_t w, int64_t* sample_idx, float* origins_k, float* dirs_k,
                            float* t_k, void* workspace, size_t workspace_bytes, sparf_stream_t stream);

/* ---------------------------------------------------------------- occupancy grid update
 * Keeping a box or contracted grid current inside a training step (sparf_b200/occupancy.py update_): each cell keeps a
 * decaying density, a fixed budget of random cells is re-sampled and the bits are re-thresholded (Instant-NGP's
 * update).  Its cost is set by the budget, not by res^3, and every size is fixed, so it can be captured in a CUDA graph.
 *   density: fp32 [res^3], indexed by the cell's linear index like the bits.  occupancy.build_grid(ema=True) starts it
 *            at the max over the cell's 8 corner lattice points of the build's sigma, NaN and +inf mapped to FLT_MAX;
 *            the bits it builds are the dilated ones of sparf_occupancy_build.
 *   interior: a box grid's every cell; a contracted grid's cells with every index in [2, res-3] (res >= 8).  The
 *            contracted grid's outer two-cell shell is never sampled or changed and stays occupied.
 *   sample:  N = n_uniform + n_occupied samples from u_cell [N] and u_jit [N,3] (fp32, in [0, 1)); I = the interior
 *            cell count, K = the number of occupied interior cells in the bits before the update (kept on the device).
 *            Sample i < n_uniform takes interior cell number min(floor((double)u_cell[i] * I), I-1) in increasing
 *            linear index; sample i >= n_uniform the min(floor((double)u_cell[i] * K), K-1)-th occupied interior cell
 *            in increasing linear index, or the uniform rule when K = 0.  Its cell (c_x, c_y, c_z) goes to cells[i]
 *            (int64 linear index) and its point to points[i] (fp32 [N,3]), computed in fp64 with every op rounded to
 *            nearest (no FMA) and rounded once to fp32:
 *              box:        x_a = r0 + (c_a + u_jit[i,a]) * (r1 - r0) / res
 *              contracted: v_a = -2 + (c_a + u_jit[i,a]) * 4 / res, n = ||v||_inf, x = center + radius * y with
 *                          y = v (n <= 1) or v / (n (2 - n)): the world point of occupancy.contracted_warp.
 *   ema:     with s_i = sigma[i] (NaN and +inf mapped to FLT_MAX), for every interior cell c
 *              density[c] = max(__fmul_rn(decay, density[c]), max over {i: cells[i] = c} of s_i)
 *            (cells with no sample just decay), then for every cell bits = !(density < thres), the contracted shell
 *            always set.  sigma must be >= 0 or NaN (the softplus of the density query).  max is exact and order-
 *            independent, so the result is deterministic bit for bit although duplicates combine through atomics.
 * sparf_occupancy_sample: center = NULL for a box grid over [r0, r1]^3 (finite, r1 > r0), else a host float[3] of finite
 * values read during the call (r0, r1 ignored; radius finite and > 0).  0 <= n_uniform, n_occupied <= 2^30; 1 <= res <=
 * 4096.  Samples outside [0, 1) are clamped into the rules' ranges.  sparf_occupancy_ema: contracted != 0 for a
 * contracted grid; 0 <= N <= 2^31; 0 < decay <= 1; cells outside [0, res^3) are ignored.  Both calls take one workspace
 * of sparf_occupancy_sample_workspace_bytes(res) bytes (0 for an invalid res; the ema uses 4 B per cell of it, the
 * sample about 4 B per 32 cells); the ema does not read what the sample left there.  No call synchronises; all are
 * capturable. */
size_t sparf_occupancy_sample_workspace_bytes(int32_t res);
int sparf_occupancy_sample(int32_t res, const uint32_t* bits, float r0, float r1, const float* center, float radius,
                           int64_t n_uniform, int64_t n_occupied, const float* u_cell, const float* u_jit, int64_t* cells,
                           float* points, void* workspace, size_t workspace_bytes, sparf_stream_t stream);
int sparf_occupancy_ema(int32_t res, int32_t contracted, int64_t n, const int64_t* cells, const float* sigma, float decay,
                        float thres, float* density, uint32_t* bits, void* workspace, size_t workspace_bytes,
                        sparf_stream_t stream);

/* ---------------------------------------------------------------- compositing
 * NeRF.composite (frequency_nerf.py:283-343).  Outputs: rgb_map [R,3], depth/opacity/depth_var/rgb_var
 * [R], weights [R,S], all_cumulated [R] (= T at sample S-2).  white_bg: rgb += 1 - opacity.  S >= 2, no upper limit.
 */
int sparf_composite_forward(int32_t R, int32_t S, const float* sigma, const float* rgb, const float* t,
                            const float* dirs, int32_t white_bg, float* rgb_map, float* depth,
                            float* opacity, float* depth_var, float* rgb_var, float* weights,
                            float* all_cumulated, sparf_stream_t stream);
/* Grads of (rgb_map, depth, opacity[, weights]) -> d_sigma [R,S], d_rgb [R,S,3] (written, not
 * accumulated) and d_dirs [R,3] (+=, through the ray length; may be NULL).  Any of g_rgb_map / g_depth / g_opacity /
 * g_weights may be NULL (that output has no gradient).  Limit: S <= 4096 (each ray keeps 2*S floats in shared memory;
 * above S = 1536 the kernel opts into more than 48 KB); larger -> SPARF_ERR_INVALID. */
int sparf_composite_backward(int32_t R, int32_t S, const float* sigma, const float* rgb, const float* t,
                             const float* dirs, int32_t white_bg, const float* g_rgb_map,
                             const float* g_depth, const float* g_opacity, const float* g_weights,
                             float* d_sigma, float* d_rgb, float* d_dirs, sparf_stream_t stream);

/* ---------------------------------------------------------------- losses
 * 2*mean Huber(delta=0.5) of pred-target over n elements (base_losses.py:155-156): writes the scalar
 * loss (+=, pre-scaled by `scale`) and d_pred = scale * dLoss/dpred. */
int sparf_huber2_fwd_bwd(int64_t n, const float* pred, const float* target, float scale, float* loss,
                         float* d_pred, sparf_stream_t stream);

/* mip-NeRF-360 distortion regulariser of the renderer's (t, weights) [R,S] (regularization_losses.py:20-48 as called
 * from base_losses.py:166-172; default off in the reference's configs): loss += scale * mean over rays; d_w [R,S] and,
 * if not NULL, d_t [R,S] are WRITTEN with scale * dLoss/d.  O(S) per ray (prefix sums over the monotone mid-points)
 * instead of the reference's [S-1, S-1] matrix. */
/* ---------------------------------------------------------------- stand-alone positional encoding
 * FrequencyEmbedder.__call__ + the BARF mask of NeRF.positional_encoding (frequency_nerf.py:47-69, 229-258) as a tensor
 * op: x [n, channels] -> out [n, 2 * channels * L] (per channel L sines then L cosines, f_j = 2^j pi, times the c2f
 * weight when use_c2f).  The MLP entry points fuse this; it exists so that the mirrored methods work on their own.
 * Backward: d_out -> d_x [n, channels] (written). */
int sparf_posenc_forward(int64_t n, int32_t channels, int32_t L, const float* x, int32_t use_c2f, float c2f_start,
                         float c2f_range, const float* progress, float* out, sparf_stream_t stream);
int sparf_posenc_backward(int64_t n, int32_t channels, int32_t L, const float* x, int32_t use_c2f, float c2f_start,
                          float c2f_range, const float* progress, const float* d_out, float* d_x, sparf_stream_t stream);

int sparf_distortion_fwd_bwd(int32_t R, int32_t S, const float* t, const float* w, float scale, float* loss,
                             float* d_w, float* d_t, sparf_stream_t stream);

/* ---------------------------------------------------------------- parameter update (SURVEY.md 8f.1)
 * One optimiser group over FLAT fp32 buffers of n elements: non-finite-gradient check (a bad gradient skips the
 * update), clip_grad_norm_(max_norm; <= 0: none), torch.optim.Adam (betas, eps, no weight decay / amsgrad) with
 * lr = lr0 * gamma^(k-1) [* min(1, k / warmup_steps) if warmup_steps > 0] at iteration k = step[1] + 1 and bias
 * corrections of update t = step[0] + 1; then step[1] = k and, unless skipped, step[0] = t.  Replaces iter_based_trainer.py:128-147 (after_backward), nerf_trainer.py:181-204 (Adam +
 * ExponentialLR) and joint_pose_nerf_trainer.py:513-549 (update_parameters).  `step` (two int64) and `scratch`
 * (>= 4 doubles, zero before the first call) live in device memory: no host round trip, CUDA-graph capturable. */
int sparf_adam_step(int64_t n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t* step,
                    double* scratch, double lr0, double gamma, double warmup_steps, double beta1, double beta2,
                    double eps, double max_norm, sparf_stream_t stream);

/* ---------------------------------------------------------------- diagnostics
 * The forward GEMM kernel of the tensor-core engines in one bf16 pass (operand layout, wgmma descriptors, accumulator
 * fragment mapping): D[128,128] = bf16(A[128,K]) * bf16(B[128,K])^T, K in {64,...,256}.  `packed` is unused (kept for
 * ABI stability).  Used by tests/test_tc_engine.py. */
int sparf_tc_selftest(const float* A, const float* B, int32_t K, void* packed, float* D, sparf_stream_t stream);
/* Same for the weight-gradient kernel: D[128,128] = G[rows,128]^T X[rows,128], rows in {64, 128}. */
int sparf_tc_selftest_tn(const float* G, const float* X, int32_t rows, float* D, sparf_stream_t stream);
/* The operand images a GEMM epilogue writes, chained through three 3-pass bf16 GEMMs, M in [1, 1024]:
 * D = X W1 (X [M,128], W1 [128,96]) is written only as a row image, a transposed image and db[96] = column sums of D;
 * Y[M,128] = [D | E] W2^T (E [M,40], W2 [128,136]) reads the row image as the first segment of a two-segment operand;
 * Z[96,128] = D^T X reads the transposed image.  Exact on small integers. */
int sparf_tc_selftest_images(const float* X, const float* W1, const float* E, const float* W2, int32_t M, float* Y, float* Z,
                             float* db, sparf_stream_t stream);
/* The same chain with every GEMM grid capped at max_ctas CTAs (max_ctas <= 0: one per SM, as the engines run), so each
 * CTA of the persistent GEMM kernel walks several work units and its copy ring wraps across them. */
int sparf_tc_selftest_persistent(const float* X, const float* W1, const float* E, const float* W2, int32_t M, float* Y,
                                 float* Z, float* db, int32_t max_ctas, sparf_stream_t stream);
/* The fused colour-head backward of the tensor-core engines against the kernels it replaces, on the same inputs:
 * d_rgb, rgb [M,3], d_sigma, raw [M], hid [M,HW], W9 [3,HW]; M in [1, 2^20], HW a multiple of 8 in [8, 512].  img gets,
 * each after a fill with 0xFFFF, four bf16 images (row_passes / tr_passes: 1 or 3, hi only or hi and lo): the fused
 * kernel's row image of Ghid [M,HW] (ceil(M/128) * ceil(HW/32) * 8192 elements) and its transposed image (ceil(HW/128) *
 * ceil(M/32) * 8192), then the same two packed from the fp32 Ghid of the old path.  graw [2,M]: the fused kernel's
 * density gradient, then the old path's.  Both halves must be bit-identical. */
int sparf_tc_selftest_head(const float* d_rgb, const float* rgb, const float* d_sigma, const float* raw, const float* hid,
                           const float* W9, int32_t M, int32_t HW, int32_t row_passes, int32_t tr_passes, uint16_t* img,
                           float* graw, sparf_stream_t stream);
/* The density backward's last-layer kernel of the tensor-core engines against masking in fp32, packing and summing, on
 * the same inputs: d_raw [M], d_feat, feat [M,W]; M in [1, 2^20], W a multiple of 8 in [8, 512].  img gets, each after
 * a fill with 0xFFFF, four bf16 images (row_passes / tr_passes: 1 or 3): the kernel's row image of G = (feat > 0) *
 * d_feat (ceil(M/128) * ceil(W/32) * 8192 elements) and its transposed image (ceil(W/128) * ceil(M/32) * 8192), then
 * the same two packed from the fp32 G.  sums [2, W+1] (zeroed first): the kernel's sum of d_raw and column sums of G,
 * then colsum_kernel's.  The images must be bit-identical; the sums are where the inputs sum exactly in any order. */
int sparf_tc_selftest_featgrad(const float* d_raw, const float* d_feat, const float* feat, int32_t M, int32_t W,
                               int32_t row_passes, int32_t tr_passes, uint16_t* img, float* sums, sparf_stream_t stream);
/* The weight-gradient GEMM as the engines run it, with the ReLU mask bits its operand pack writes: dW[N,K] (zeroed
 * first) gets sum_m G[m][n] X[m / div][k] for k < Kv (0 elsewhere), with G [M,N] fp32 packed as its transposed bf16 image and both
 * operands split in `passes` (1 or 3) passes; X has rows of ldx >= K floats.  bits (may be NULL) [M, ceil(K/32)] gets
 * bit k % 32 of word k / 32 of row m = (X[m / div][k] > 0).  M in [1, 2^20], N and K in [1, 512], div >= 1; max_ctas > 0
 * caps the grid (else one CTA per SM). */
int sparf_tc_selftest_wgrad(const float* G, const float* X, int32_t M, int32_t N, int32_t K, int32_t Kv, int32_t ldx,
                            int32_t div, int32_t passes, int32_t max_ctas, float* dW, uint32_t* bits, sparf_stream_t stream);
/* The same GEMM with a device row count: M is a capacity, of which the GEMM sums the rows m < *rows (device, int64). */
int sparf_tc_selftest_wgrad_rows(const float* G, const float* X, int32_t M, int32_t N, int32_t K, int32_t Kv, int32_t ldx,
                                 int32_t div, int32_t passes, int32_t max_ctas, const int64_t* rows, float* dW,
                                 uint32_t* bits, sparf_stream_t stream);
/* The input-gradient GEMM's two ReLU masks against each other, 3-pass bf16: D = (X > 0) * (G W), G [M,N], W [N,K],
 * X [M,K] fp32 row-major, written only as its row and transposed images, once with the fp32 mask X and once with the
 * bits of X > 0 that the weight-gradient GEMM G^T X writes.  img gets, after a fill with 0xFFFF, the fp32-mask run's
 * row image (ceil(M/128) * ceil(K/32) * 8192 elements) and transposed image (ceil(K/128) * ceil(M/32) * 8192), then the
 * bit-mask run's two; they must be bit-identical.  M in [1, 2^20], N in [1, 512], K even in [2, 512]; max_ctas > 0
 * caps the grids. */
int sparf_tc_selftest_mask_bits(const float* G, const float* W, const float* X, int32_t M, int32_t N, int32_t K,
                                int32_t max_ctas, uint16_t* img, sparf_stream_t stream);
/* The trunk forward of width 256 as the tensor-core engines run it, in one fused kernel that keeps a row tile's
 * activations in shared memory (chain != 0), or layer by layer through GEMMs chained by row images (chain == 0), on the
 * same inputs: enc [M, E3p] (E3p = E3 rounded up to 32 <= 64, zero padded), W = the nt layers' [256, ldw_l] weights one
 * after another (ldw_l = (l == 0 ? E3 : 256) + (l == skip ? E3 : 0)), bias [nt, 256]; passes 1 or 3, f16 != 0: fp16
 * halves, else bf16.  H [nt, M, 256]: layer l is written iff bit l of outputs (bit nt-2 is required; without bit nt-1
 * the last layer is not computed).  last (may be NULL): the last layer's row image, ceil(M/128) * 8 * 8192 elements.
 * rows (may be NULL): M is a capacity and *rows (device) the rows computed.  max_ctas > 0 caps the grids.  Both runs must
 * write the same bytes. */
int sparf_tc_selftest_chain(const float* enc, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                            const float* bias, int32_t passes, int32_t f16, int32_t max_ctas, int32_t chain,
                            uint32_t outputs, const int64_t* rows, float* H, uint16_t* last, sparf_stream_t stream);
/* The fused forward (every output) with the ReLU masks it writes for the chained backward: bits [nt-2][M][8] uint32, bit
 * n & 31 of word [l][m][n >> 5] = H[l][m][n] > 0, layers 0 ... nt-3. */
int sparf_tc_selftest_chain_bits(const float* enc, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                                 const float* bias, int32_t passes, int32_t f16, int32_t max_ctas, const int64_t* rows,
                                 float* H, uint32_t* bits, sparf_stream_t stream);
/* The trunk backward's input gradients of layers nt-2 ... 1 (width 256, bf16 halves), fused (chain != 0) or through the
 * layer-by-layer input-gradient GEMMs with bit masks (chain == 0), on the same inputs: G [M, 256] the gradient of layer
 * nt-2's output, W as sparf_tc_selftest_chain's, bits [nt-2][M][8] the masks of H[0] ... H[nt-3].  Writes tr [nt-2]
 * transposed images of G[0] ... G[nt-3] (wg_passes; 2 * ceil(M/32) * 8192 elements each), db [nt-2][256] their column
 * sums and, when row is not NULL (skip <= nt-3), row [2] the row images of G[0] and G[skip] (dg_passes; ceil(M/128) * 8 *
 * 8192 elements each).  rows and max_ctas as sparf_tc_selftest_chain's.  Both runs must write the same image bytes. */
int sparf_tc_selftest_dgrad_chain(const float* G, int32_t M, int32_t E3, int32_t nt, int32_t skip, const float* W,
                                  const uint32_t* bits, int32_t dg_passes, int32_t wg_passes, int32_t max_ctas,
                                  int32_t chain, const int64_t* rows, uint16_t* tr, uint16_t* row, float* db,
                                  sparf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SPARF_B200_H_ */
