/*
 * morefusion_b200.h -- C ABI of libmorefusion_sm90a.so
 *
 * Drop-in boundary for the volumetric-pose hot path of wkentaro/morefusion
 * (SURVEY.md section 8).  The reference has no native library: each entry point
 * below replaces one chainer.Function / Link method (cited per function, paths
 * relative to the reference checkout).  A binding only needs ctypes/cffi: plain
 * pointers, sizes and scalars -- no torch, chainer or cupy types.
 *
 * Conventions
 *   - every pointer named in/out is a DEVICE pointer unless marked "host";
 *     tensors are dense, C-contiguous, float32 / int32 as in the reference.
 *   - grids are [X,Y,Z] (z fastest), batched [B,C,X,Y,Z]; flat voxel index
 *     ix*Y*Z + iy*Z + iz (average_voxelization_3d.py:92-96).
 *   - quaternions are (w,x,y,z); transforms are row-major 4x4.
 *   - the caller owns all memory including `workspace`; kernels never allocate,
 *     never retain pointers past the call, never synchronise the host, and are
 *     safe under CUDA-graph capture.  Work is enqueued on `stream`
 *     (a cudaStream_t passed as void*).
 *   - return value: 0 = ok; <0 = invalid argument (MF_E_*); >0 = cudaError_t.
 *   - `flags` (device int32, may be NULL) receives OR-ed MF_FLAG_* bits so the
 *     host binding can raise the reference's ValueError lazily.
 */
#ifndef MOREFUSION_B200_H_
#define MOREFUSION_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MF_OK 0
#define MF_E_BADARG (-1)      /* null pointer / negative size */
#define MF_E_TOOLARGE (-2)    /* B*X*Y*Z (or P*K) does not fit in int32 keys */
#define MF_E_WORKSPACE (-3)   /* workspace smaller than *_workspace_bytes() */
#define MF_E_UNSUPPORTED (-4) /* shape outside what the kernel family covers */

#define MF_FLAG_NAN_POINTS 1      /* "points include nan" (average_voxelization_3d.py:13-14,47-48) */
#define MF_FLAG_UNSORTED_BATCH 2  /* batch_indices not non-decreasing (informational) */
#define MF_FLAG_BAD_BATCH_INDEX 4 /* batch index outside [0,B): point dropped */

int mf_abi_version(void);
/* number of SMs / device name the library sees (diagnostics for the binding) */
int mf_device_sm_count(int device);

/* ------------------------------------------------------------------------
 * a1  average_voxelization_3d
 *     replaces AverageVoxelization3D.forward_gpu / backward_gpu
 *     (morefusion/functions/geometry/average_voxelization_3d.py:43-118, :147-220)
 * values [N,C] points [N,3] batch_indices [N] -> matrix [B,C,X,Y,Z], counts [B,X,Y,Z]
 * Two launches (keys; gather + fill): every output voxel is written exactly once (no
 * memset, no atomics on HBM, nothing in `workspace` needs initialising); per-voxel sums
 * are taken in ascending point order (deterministic).
 * ------------------------------------------------------------------------ */
size_t mf_average_voxelization_3d_workspace_bytes(int64_t n_points);
/* byte offset inside `workspace` of an int32 copy of the MF_FLAG_* word of the last call (so a
 * binding needs no separate flags allocation; `flags` below may then be NULL) */
size_t mf_average_voxelization_3d_flags_offset(void);
int mf_average_voxelization_3d_fwd(
    const float* values, const float* points, const int32_t* batch_indices,
    int64_t n_points, int channels, int batch_size,
    float origin_x, float origin_y, float origin_z, float pitch,
    int X, int Y, int Z,
    float* matrix, int32_t* counts,
    void* workspace, size_t workspace_bytes, int32_t* flags, void* stream);
/* diagnostics: writes B*planes*V zero floats with one of five store patterns (see
 * csrc/voxelization.cu, scripts/fill_patterns.py) */
int mf_debug_fill_probe(float* out, int batch_size, int planes, int64_t V, int mode, void* stream);
int mf_average_voxelization_3d_bwd(
    const float* gmatrix, const int32_t* counts,
    const float* points, const int32_t* batch_indices,
    int64_t n_points, int channels, int batch_size,
    float origin_x, float origin_y, float origin_z, float pitch,
    int X, int Y, int Z,
    float* gvalues, void* stream);

/* ------------------------------------------------------------------------
 * a6  max_voxelization_3d
 *     replaces MaxVoxelization3D.forward_gpu / backward_gpu
 *     (morefusion/functions/geometry/max_voxelization_3d.py:57-143, :145-185)
 * winner per voxel = max intensity, lowest point id on exact ties.
 * ------------------------------------------------------------------------ */
size_t mf_max_voxelization_3d_workspace_bytes(int batch_size, int X, int Y, int Z);
int mf_max_voxelization_3d_fwd(
    const float* values, const float* points, const int32_t* batch_indices,
    const float* intensities,
    int64_t n_points, int channels, int batch_size,
    float origin_x, float origin_y, float origin_z, float pitch,
    int X, int Y, int Z,
    float* matrix, int32_t* indices,
    void* workspace, size_t workspace_bytes, int32_t* flags, void* stream);
int mf_max_voxelization_3d_bwd(
    const float* gmatrix, const int32_t* indices,
    int64_t n_points, int channels, int batch_size, int X, int Y, int Z,
    float* gvalues, void* stream);

/* ------------------------------------------------------------------------
 * a5  interpolate_voxel_grid
 *     replaces InterpolateVoxelGrid.forward_gpu / backward_gpu
 *     (morefusion/functions/geometry/interpolate_voxel_grid.py:159-214, :216-268)
 * voxelized [B,C,X,Y,Z], points [P,3] (voxel units), batch_indices [P] -> values [P,C]
 * `channels_last` != 0 reads/writes the grid as [B,X,Y,Z,C] (internal layout of
 * the 3D-CNN path; same arithmetic).
 * Every row of `values` is written.  A point whose batch index is outside
 * [0, batch_size) gets a row of +0.0 (the reference reads out of bounds there)
 * and adds nothing to `gvoxelized`.  Rows of the other points are bit-identical
 * on every kernel path.
 * ------------------------------------------------------------------------ */
int mf_interpolate_voxel_grid_fwd(
    const float* voxelized, const float* points, const int32_t* batch_indices,
    int64_t n_points, int batch_size, int channels, int X, int Y, int Z,
    int channels_last, float* values, void* stream);
int mf_interpolate_voxel_grid_bwd(
    const float* gvalues, const float* points, const int32_t* batch_indices,
    int64_t n_points, int batch_size, int channels, int X, int Y, int Z,
    int channels_last, float* gvoxelized /* fully written */, void* stream);
/* The kernel the two calls above launch for a shape (`backward` selects the
 * call) on a device with `n_sm` SMs, as an MF_INTERP_* id, and in *cg (host)
 * its channel group: the channels one CTA covers (1 for the one-thread-per-
 * (point, channel) kernels, 0 when nothing is launched).  Host code only: no
 * CUDA call.  Both calls dispatch through it.  Returns MF_E_BADARG for the
 * arguments they reject. */
#define MF_INTERP_NONE 0           /* forward, no points: nothing to write */
#define MF_INTERP_FWD_STREAM 1     /* persistent CTAs, double-buffered planes, cached points */
#define MF_INTERP_FWD_PLANES 2     /* CG channel planes per CTA in shared memory */
#define MF_INTERP_FWD_SIMPLE 3     /* one thread per (point, channel) */
#define MF_INTERP_FWD_SIMPLE_CL 4  /* the same on a channels-last grid */
#define MF_INTERP_BWD_CELLS 5      /* cell-owner gather, deterministic */
#define MF_INTERP_BWD_STREAM 6     /* persistent CTAs, shared-memory atomics */
#define MF_INTERP_BWD_PLANES 7     /* CG channel planes per CTA, shared-memory atomics */
#define MF_INTERP_BWD_ATOMIC 8     /* memset + global atomics */
#define MF_INTERP_BWD_ATOMIC_CL 9  /* the same on a channels-last grid */
#define MF_INTERP_BWD_ZERO 10      /* no points: memset only */
int mf_interpolate_voxel_grid_path(
    int64_t n_points, int batch_size, int channels, int X, int Y, int Z,
    int channels_last, int backward, int n_sm, int* cg);

/* ------------------------------------------------------------------------
 * a3  truncated_distance_function
 *     replaces TruncatedDistanceFunction.forward_gpu / backward_gpu
 *     (morefusion/functions/geometry/truncated_distance_function.py:21-101, :103-166)
 * points [P,3] -> tdf [X,Y,Z] (init = truncation), indices [X,Y,Z] (winning
 * point id, -1 if none; already divided by K as at :177).
 * Winner = lexicographic min of (distance, point id): deterministic.
 * ------------------------------------------------------------------------ */
size_t mf_truncated_distance_function_workspace_bytes(int X, int Y, int Z);
int mf_truncated_distance_function_fwd(
    const float* points, int64_t n_points,
    float pitch, float origin_x, float origin_y, float origin_z,
    int X, int Y, int Z, float truncation,
    float* tdf, int32_t* indices,
    void* workspace, size_t workspace_bytes, void* stream);
int mf_truncated_distance_function_bwd(
    const float* gtdf, const float* points, const int32_t* indices, int64_t n_points,
    float pitch, float origin_x, float origin_y, float origin_z,
    int X, int Y, int Z, float truncation,
    float* gpoints, void* stream);

/* ------------------------------------------------------------------------
 * a4  pseudo_occupancy_voxelization
 *     replaces the function at truncated_distance_function.py:181-213
 * Outputs grid/surface/inside [X,Y,Z]; also tdf, indices, w_surface, w_inside
 * (kept for backward: weights carry no gradient, :196-213).
 * ------------------------------------------------------------------------ */
size_t mf_pseudo_occupancy_voxelization_workspace_bytes(int X, int Y, int Z);
int mf_pseudo_occupancy_voxelization_fwd(
    const float* points, const float* sdf, int64_t n_points,
    float pitch, float origin_x, float origin_y, float origin_z,
    int X, int Y, int Z, float threshold, float sdf_offset,
    float* grid, float* grid_surface, float* grid_inside,
    float* tdf, int32_t* indices, float* w_surface, float* w_inside,
    void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * a2  occupancy_grid_3d
 *     replaces OccupancyGrid3D + the chainer op chain at
 *     morefusion/functions/geometry/occupancy_grid_3d.py:31-85
 * matrix-free: never materialises the [X,Y,Z,P] distance tensors.
 * ------------------------------------------------------------------------ */
int mf_occupancy_grid_3d_fwd(
    const float* points, int64_t n_points,
    float pitch, float origin_x, float origin_y, float origin_z,
    int X, int Y, int Z, float threshold,
    float* grid, float* dmin /* [X,Y,Z], kept for backward */, void* stream);
int mf_occupancy_grid_3d_bwd(
    const float* ggrid, const float* dmin, const float* points, int64_t n_points,
    float pitch, float origin_x, float origin_y, float origin_z,
    int X, int Y, int Z, float threshold,
    float* gpoints /* zero-filled by the call */, void* stream);

/* ------------------------------------------------------------------------
 * a7  rigid-transform operators
 *     quaternion_matrix.py:6-78, compose_transform.py:5-48,
 *     translation_matrix.py:5-39, transformation_matrix.py:5-18,
 *     transform_points.py:6-30
 * ------------------------------------------------------------------------ */
int mf_quaternion_matrix_fwd(const float* q /*[N,4]*/, int64_t n, float* R /*[N,4,4]*/, void* stream);
int mf_quaternion_matrix_bwd(const float* gR /*[N,4,4]*/, const float* q, int64_t n,
                             float* gq /*[N,4]*/, void* stream);
int mf_compose_transform_fwd(const float* R /*[N,3,3]*/, const float* t /*[N,3] or NULL*/,
                             int64_t n, float* T /*[N,4,4]*/, void* stream);
int mf_transform_points_fwd(const float* points /*[P,3]*/, int64_t n_points,
                            const float* T /*[M,4,4]*/, int64_t m,
                            float* out /*[M,P,3]*/, void* stream);
int mf_transform_points_bwd(const float* gout /*[M,P,3]*/, const float* points, int64_t n_points,
                            const float* T, int64_t m,
                            float* gpoints /*[P,3] or NULL*/, float* gT /*[M,4,4] or NULL*/,
                            void* stream);


/* ------------------------------------------------------------------------
 * a10 / a11  3D-CNN section of the singleview_3d pose model
 *     replaces the chainer/cuDNN layers of
 *     morefusion/contrib/singleview_3d/models/model.py:62-91 (layer defs),
 *     :93-141 (_extract), :239-273 (heads + pose assembly)
 * Activations are channels-last bf16, accumulation fp32.  The k4/s2/p1 Conv3Ds run as
 * implicit GEMMs over a space-to-depth ("s2d") layout of the zero-padded input:
 *   X[b][jd][jh][jw][r*C + c] = xpad[b][c][2jd+rd][2jh+rh][2jw+rw],  r = rd<<2|rh<<1|rw,
 * and weights Wg[co][((ad*2+ah)*2+aw)*8C + r*C + ci] = W[co][ci][2ad+rd][2ah+rh][2aw+rw].
 * ------------------------------------------------------------------------ */
#define GEMM_LINEAR 0    /* A[m][k] row-major, leading dimension lda */
#define GEMM_CONV_S2D 1  /* A gathered from an s2d grid: m=(b,od,oh,ow), k=(a, r*C+ci) */
#define OUT_BF16 0       /* out[m*ldo + col_off + n], bf16 */
#define OUT_F32 1        /* out[m*ldo + col_off + n], fp32 */
#define OUT_S2D_BF16 2   /* row m=(b,od,oh,ow) scattered into the s2d layout of the next conv */
/* singleview_pcd (examples/ycb_video/singleview_pcd/contrib/models/model.py:119-121, :299-330):
 * the rows of a GEMM are the points of consecutive objects, Do rows per object. */
#define GEMM_LINEAR_OBJ_BIAS 2  /* GEMM_LINEAR whose bias is per object: bias[(m / Do) * N + n] */
#define OUT_OBJ_SUM_F32 3  /* act(row) summed per object within each 16-row group, no row stored:
                            * out fp32 [ceil(M/16)][2][N], slot s of group g = rows of object
                            * (16 g) / Do + s (slot 1 written only where the group holds two
                            * objects).  Fixed-order sums, no atomics; Do >= 16, GEMM_LINEAR;
                            * ldo / col_off unused.  Finish with mf_posenet_pool. */

typedef struct GemmParams {
  const void* A;      /* bf16 */
  const void* W;      /* bf16 [N][ldw], K-major */
  const float* bias;  /* [N] or NULL */
  void* out;
  int M, N, K;
  int mode;           /* GEMM_* */
  long long lda;      /* GEMM_LINEAR */
  long long ldw;
  int Do;             /* GEMM_CONV_S2D / OUT_S2D_BF16: output grid edge (16 for conv3, 8 for conv4);
                         GEMM_LINEAR_OBJ_BIAS / OUT_OBJ_SUM_F32: rows per object */
  int Ci8;            /* GEMM_CONV_S2D: 8 * input channels */
  int relu;
  int out_mode;       /* OUT_* */
  long long ldo;
  int col_off;
} GemmParams;

/* weights are passed TRANSPOSED ([in][out], k-major): w1_rgb [32,64], w1_pcd [3,8], ... */
int mf_cnn_point_mlp(const float* values /*[B,32,P]*/, const float* points /*[B,3,P] voxel frame*/,
                     const float* w1_rgb, const float* b1_rgb, const float* w1_pcd,
                     const float* b1_pcd, const float* w2_rgb, const float* b2_rgb,
                     const float* w2_pcd, const float* b2_pcd, int B, int P, float center,
                     void* feat_bf16 /*[B*P, ldf], cols 0..215*/, int ldf,
                     float* feat2 /*[B*P,144]*/, void* stream);
/* conv2's output goes to h2 (fp32 [B,V,16]) or, when X != NULL, as bf16 into channels
 * [c_off, c_off+16) of the s2d conv3 input X (row length 8*Ct). */
int mf_cnn_occ_convs(const float* grid_nontarget_empty /*[B,D,D,D]*/, const float* w1,
                     const float* b1, const float* w2, const float* b2, int B, int D,
                     float* h1 /*[B,V,8] scratch*/, float* h2 /*[B,V,16] or NULL*/,
                     void* X /*bf16 s2d or NULL*/, int Ct, int c_off, void* stream);
/* tensor-core variant (D == 32): conv1_occ -> bf16 [B,V,8] scratch, conv2_occ as warp-level
 * mma.sync m16n8k16 (bf16 operands, fp32 accumulate) writing bf16 into X. */
int mf_cnn_occ_convs_tc(const float* grid_nontarget_empty, const float* w1, const float* b1,
                        const float* w2, const float* b2, int B, int D, void* h1_bf16 /*[B,V,8]*/,
                        void* X, int Ct, int c_off, void* stream);
/* same, reading the occupancy grid as bytes (0/1; uint8 or bool storage): saves the cast the
 * reference does inside the model (model.py:115-116) */
int mf_cnn_occ_convs_tc_u8(const uint8_t* grid_nontarget_empty, const float* w1, const float* b1,
                           const float* w2, const float* b2, int B, int D,
                           void* h1_bf16 /*[B,V,8]*/, void* X, int Ct, int c_off, void* stream);
/* conv1_occ + conv2_occ (model.py:69-70,114-125) in ONE kernel (D == 32): each x-slab CTA evaluates
 * conv1_occ for the three slabs its dilated conv2_occ reads, in shared memory, then conv2_occ on
 * mma.sync; no [B,V,8] intermediate in global memory.  Same bits as mf_cnn_occ_convs_tc. */
int mf_cnn_occ_fused(const float* grid_nontarget_empty, const float* w1, const float* b1,
                     const float* w2, const float* b2, int B, int D, void* X, int Ct, int c_off,
                     void* stream);
int mf_cnn_occ_fused_u8(const uint8_t* grid_nontarget_empty, const float* w1, const float* b1,
                        const float* w2, const float* b2, int B, int D, void* X, int Ct, int c_off,
                        void* stream);
/* average_voxelization_3d of model.py:143-164 (origin 0, pitch 1, D^3) fused with the s2d/bf16
 * packing: writes channels [0,C) of X.  prev_keys [2*B*P] int32 (in/out, initialise to -1): the
 * first B*P entries hold the voxel key of every point of the previous call (b*D^3 + voxel, -1 =
 * dropped, bit 30 = shares its voxel) so that only those voxels are re-zeroed; the second B*P
 * entries are scratch (each object's points sorted by voxel, then index). */
int mf_cnn_voxelize_s2d(const float* feat2 /*[B*P,C]*/, const float* points /*[B,3,P]*/, int B,
                        int P, int C, int D, int Ct, int32_t* prev_keys, void* X, void* stream);
/* mf_cnn_point_mlp + phase 1 of mf_cnn_voxelize_s2d_phase (sparse clear of the previous call's
 * voxels + this call's keys / sorted order) in ONE launch: the bookkeeping CTAs are dispatched
 * first and run beside the MLP CTAs.  P <= 4096 (else MF_E_UNSUPPORTED: use the two calls).
 * Follow with mf_cnn_voxelize_s2d_phase(..., phases = 2). */
int mf_cnn_point_mlp_voxkeys(const float* values, const float* points, const float* w1_rgb,
                             const float* b1_rgb, const float* w1_pcd, const float* b1_pcd,
                             const float* w2_rgb, const float* b2_rgb, const float* w2_pcd,
                             const float* b2_pcd, int B, int P, float center, void* feat, int ldf,
                             float* feat2, int C, int D, int Ct, int32_t* prev_keys, void* X,
                             void* stream);
/* the same in two halves so that a caller can overlap the first with the point MLP that produces
 * feat2: phases bit 0 = sparse clear + new keys (feat2 may be NULL), bit 1 = ordered scatter */
int mf_cnn_voxelize_s2d_phase(const float* feat2, const float* points, int B, int P, int C, int D,
                              int Ct, int32_t* prev_keys, void* X, int phases, void* stream);
int mf_cnn_pack_s2d(const float* vox /*[B,C,D,D,D]*/, const float* hocc /*[B,V,Cocc] or NULL*/,
                    int B, int C, int Cocc, int D, void* X /*bf16 s2d, borders pre-zeroed*/,
                    void* stream);
int mf_gemm_bf16_simt(const GemmParams* p, void* stream);
/* up to 3 GEMMs in one launch (the three pose heads); tc variant needs identical M,N,K,mode */
int mf_gemm_bf16_simt_grouped(const GemmParams* p, int n_groups, void* stream);
int mf_gemm_bf16_tc_grouped(const GemmParams* p, int n_groups, void* workspace,
                            size_t workspace_bytes, void* stream);
/* wgmma/TMA kernel; returns MF_E_UNSUPPORTED for shapes it does not cover (N % 32, N < 128,
 * K < 64, unaligned views) -- the caller then uses mf_gemm_bf16_simt.  `workspace` holds fp32
 * [M][N] partial sums when the launch splits K (few output tiles, long K). */
size_t mf_gemm_bf16_tc_workspace_bytes(int M, int N);
int mf_gemm_bf16_tc(const GemmParams* p, void* workspace, size_t workspace_bytes, void* stream);
/* Extended entry.
 *  sync   : NULL, or MF_GEMM_TC_SYNC_INTS int32 words owned by the caller, zeroed ONCE before the
 *           first call (the kernel leaves them zero).  With it, bf16-output GEMMs (grouped or
 *           not) whose tile count would idle > 5 % of the SMs run "stream-K": the
 *           tiles x K-blocks space is cut into one equal range per SM, a CTA that starts inside
 *           a tile parks its fp32 accumulator in `workspace` (one 128 x 256 slot per SM) and the
 *           tile's first CTA adds the slots in CTA order in its epilogue: every SM does the same
 *           number of K blocks and there is no separate reduction launch.  Two launches that
 *           may run concurrently must not share `sync` / `workspace`.
 *  stamps : NULL, or a device buffer of 16*8 int64 receiving clock64 stamps of CTA 0's roles per
 *           work unit (0/1 TMA producer begin/end, 2/3/4 consumer unit start / first operands / main loop
 *           done, 5/6/7 epilogue start / stored / stored).
 *  one_shot : 1 = whole-tile scheduling only (no stream-K) as a baseline; 0 or 2 = stream-K
 *           where it pays (see `sync`). */
#define MF_GEMM_TC_SYNC_INTS 2048
int mf_gemm_bf16_tc_ex(const GemmParams* p, int n_groups, void* workspace, size_t workspace_bytes,
                       int32_t* sync, long long* stamps, int one_shot, void* stream);
/* The launch plan of mf_gemm_bf16_tc_ex, which decides through mf_gemm_bf16_tc_plan.
 *  WHOLE   : every unit is a whole tile (all of K).
 *  STREAMK : the units x K-blocks space cut into one equal range per cluster.  Chosen only when
 *            there are at least as many K blocks as clusters, so that no range is empty and no
 *            tile owner waits on a cluster that runs nothing.
 *  SPLITK  : 2-4 K slices stored as fp32 to the workspace, summed by a second kernel that adds
 *            the bias first.  Declined when a bias is not 16-byte aligned.
 * ReLU keeps NaN on every plan (cvt.rn.relu on bf16 stores; x < 0 ? 0 : x elsewhere), as
 * torch.relu does; -0 may come out as either zero. */
#define MF_GEMM_WHOLE 0
#define MF_GEMM_STREAMK 1
#define MF_GEMM_SPLITK 2
typedef struct MfGemmPlan {
  int cluster;      /* CTAs per cluster: 1, or 2 (CTA pairs sharing the W tile; convolutions) */
  int block_n;      /* N tile: 256 (4 stages) or 128 (6 stages) */
  int stages;
  int schedule;     /* MF_GEMM_* */
  int splitk;       /* K slices (1 unless SPLITK) */
  int staged;       /* bf16 outputs leave through shared memory and TMA stores */
  int grid;         /* CTAs launched */
  int n_units;      /* work units (tile pairs when cluster = 2, times K slices) */
  int kb_total;     /* 64-wide K blocks */
  int max_pieces;   /* most partial sums any output tile is built from (slices or stream-K pieces) */
} MfGemmPlan;
/* Pure host: the plan mf_gemm_bf16_tc_ex would launch on a device of n_sm SMs where n_pairs CTA
 * pairs are co-resident.  workspace_bytes = 0 stands for no workspace.  Returns what the launch
 * returns before it launches: MF_OK, MF_E_UNSUPPORTED (the SIMT kernel covers the shape),
 * MF_E_BADARG (e.g. a row-major output with ldo < col_off + N) or MF_E_WORKSPACE. */
int mf_gemm_bf16_tc_plan(const GemmParams* p, int n_groups, size_t workspace_bytes, int has_sync,
                         int one_shot, int n_sm, int n_pairs, MfGemmPlan* out);
/* CTA pairs of the persistent kernel with an N tile of block_n (256 or 128) co-resident on the
 * current device, as mf_gemm_bf16_tc_ex counts them (cached per device). */
int mf_gemm_bf16_tc_pair_clusters(int block_n, int* n_pairs);
/* Pure host: the stream-K segments of n_units x kb_total K blocks over n_clusters clusters, as the
 * kernel walks them.  Writes up to `cap` rows of 7 ints (cluster, unit, kb0, kb1, partial, peer0,
 * n_peers) and returns the number of segments (more than cap: only cap written), or MF_E_BADARG. */
int mf_gemm_bf16_tc_segments(int n_units, int kb_total, int n_clusters, int* seg, int cap);
/* Layers 1-3 of the three pose heads (model.py:239-254) as ONE persistent launch.  layers[0] =
 * the three first layers side by side (N = 3 x 640), layers[1..3] = conv2_{rot,trans,conf}
 * reading their column block of layer 0's output, layers[4..6] = conv3_* reading layers[1..3]'s
 * outputs; all GEMM_LINEAR, OUT_BF16, same M.  Tiles of later layers start as soon as the
 * 128-row tiles they read are stored (global arrival counters), so the three layers share one
 * wave structure and there are no launch gaps.  sync: MF_HEADS_SYNC_INTS int32 words owned by the
 * caller, zeroed ONCE (never reset afterwards: an epoch word makes the counters monotonic).
 * Runs on CTA pairs; returns MF_E_UNSUPPORTED when pairs cannot cover every SM of the device
 * (the caller then runs the three grouped launches). */
#define MF_HEADS_SYNC_INTS 4096
int mf_cnn_heads_tc(const GemmParams* layers, int n_layers /* 7 */, int32_t* sync, void* stream);
int mf_cnn_interp_cl(const void* grid_bf16, int s2d, const float* points /*[B,3,P]*/, int B,
                     int P, int C, int D, float divisor, void* feat_bf16, int ldf, int col_off,
                     void* stream);
int mf_cnn_pose(const float* out_rot, const float* out_trans, const float* out_conf,
                const float* points, const int32_t* class_id, const float* pitch,
                const float* origin, int B, int P, int n_fg_class, float* rot /*[B,P,4]*/,
                float* trans /*[B,P,3]*/, float* conf /*[B,P]*/, void* stream);
/* last head layer (conv4_{rot,trans,conf}, model.py:249-254) fused with the pose epilogue: only
 * the 4+3+1 output rows of each object's class are evaluated.  hd3 = bf16 [B*P, ld] holding the
 * rot | trans | conf 128-channel blocks; weights bf16 [rows,128] row-major, biases fp32.  class_id
 * is 1-based and must lie in [1, nfg] (as in the reference's indexing, model.py:256-262). */
int mf_cnn_head4_pose(const void* hd3, int ld, const void* w_rot, const float* b_rot,
                      const void* w_trans, const float* b_trans, const void* w_conf,
                      const float* b_conf, const float* points, const int32_t* class_id,
                      const float* pitch, const float* origin, int B, int P, int nfg, float* rot,
                      float* trans, float* conf, void* stream);

/* ------------------------------------------------------------------------
 * PoseNet section of the singleview_pcd ("DenseFusion*") pose model
 *     replaces the chainer layers of
 *     examples/ycb_video/singleview_pcd/contrib/models/model.py:299-330 (PoseNetExtractor),
 *     :115-116 (centring) and the feat3 columns of :119-121 (the heads' first layer)
 * Launch sequence of one forward (csrc/posenet.cu, the GEMMs on conv3d_tc.cu):
 *   mf_posenet_point_mlp -> conv3 GEMM (OUT_BF16) -> conv4 GEMM (OUT_OBJ_SUM_F32) ->
 *   mf_posenet_pool -> mf_posenet_obj_bias -> mf_cnn_heads_tc (layer 1 GEMM_LINEAR_OBJ_BIAS,
 *   K = 384) -> mf_cnn_head4_pose (pitch 1, origin = center, points = the centred pcd).
 * ------------------------------------------------------------------------ */
/* conv1_rgb 32->64, conv1_pcd 3->64, conv2_rgb 64->128, conv2_pcd 64->128, Conv1D k=1 + ReLU
 * (:320-326), weights TRANSPOSED ([in][out]) fp32.  The pcd branch reads pcd - center[b] (center
 * NULL: 0), which is also written to pcd_c.  feat row n (bf16, pitch ldf >= 384):
 * [conv1_rgb | conv1_pcd | conv2_rgb | conv2_pcd] = [feat1 | feat2] of :322,:325. */
int mf_posenet_point_mlp(const float* values /*[B,32,P]*/, const float* pcd /*[B,3,P]*/,
                         const float* center /*[B,3] or NULL*/, const float* w1_rgb,
                         const float* b1_rgb, const float* w1_pcd, const float* b1_pcd,
                         const float* w2_rgb, const float* b2_rgb, const float* w2_pcd,
                         const float* b2_pcd, int B, int P, void* feat, int ldf,
                         float* pcd_c /*[B,3,P]*/, void* stream);
/* the mean over each object's P points (:328, F.average_pooling_1d) from the partial sums of an
 * OUT_OBJ_SUM_F32 GEMM with Do = P (fp32 [ceil(B*P/16)][2][N]), added group by group in ascending
 * order: pooled fp32 [B][N] */
int mf_posenet_pool(const float* partials, int B, int P, int N, float* pooled, void* stream);
/* per-object bias of the heads' first layer: out[b][o] = bias[o] + sum_k W[o][k] pooled[b][k],
 * W bf16 rows of pitch ldw (the feat3 columns of conv1_{rot,trans,conf}.W, K = 1024), fp32
 * accumulation in a fixed order; out fp32 [B][rows] */
int mf_posenet_obj_bias(const void* W, long long ldw, int rows, int K, const float* bias,
                        const float* pooled, int B, float* out, void* stream);
/* Backward (training).  s [B][rows] fp32 = per-object column sums of the heads' layer-1 gradient
 * dZ1 (mf_posenet_obj_colsum): dW (row pitch lddw, the feat3 columns of
 * conv1_*.W) += s^T pooled, db (may be NULL) += sum_b s[b], dpooled [B][K] = s W (overwritten). */
int mf_posenet_obj_bias_bwd(const float* s, const float* pooled, const void* W, long long ldw, int rows,
                            int K, int B, float* dW, long long lddw, float* db, float* dpooled,
                            void* stream);
/* per-object column sums in one launch: out[b][n] += sum_{p<P} x[b P + p][n] for every object b,
 * x bf16 rows of pitch ldx (>= N), out fp32 [B][N].  Each column is summed in mf_train_colsum's
 * order (its 256-row blocks ascending), with no atomics: equal to B mf_train_colsum launches
 * whose atomics land in block order. */
int mf_posenet_obj_colsum(const void* x /*bf16 [B*P, ldx]*/, long long ldx, int B, int P, int N,
                          float* out /*accumulated*/, void* stream);
/* mean-pool + ReLU backward: dz[m][n] = bf16((h4[m][n] > 0) * dpooled[m / P][n] / P) */
int mf_posenet_pool_bwd(const float* dpooled, const void* h4 /*bf16 [B*P,N]*/, int B, int P, int N,
                        void* dz /*bf16 [B*P,N]*/, void* stream);
/* conv1_* / conv2_* backward from dfeat [B*P,384] fp32 (d [feat1|feat2] through the heads) +
 * dfeat2 [B*P,256] fp32 (d feat2 through conv3); weights [out][in] fp32; the activations are
 * recomputed from values and pcd_c (mf_posenet_point_mlp's output).  Weight / bias gradients
 * accumulated; dvalues [B,32,P] overwritten (may be NULL). */
int mf_posenet_point_mlp_bwd(const float* values, const float* pcd_c, const float* w1_rgb,
                             const float* b1_rgb, const float* w1_pcd, const float* b1_pcd,
                             const float* w2_rgb, const float* b2_rgb, const float* w2_pcd,
                             const float* b2_pcd, int B, int P, const float* dfeat,
                             const float* dfeat2, float* dw1_rgb, float* db1_rgb, float* dw1_pcd,
                             float* db1_pcd, float* dw2_rgb, float* db2_rgb, float* dw2_pcd,
                             float* db2_pcd, float* dvalues, void* stream);

/* ------------------------------------------------------------------------
 * a8 / a9  IterativeCollisionCheckLink + its Adam loop, fused
 *     replaces IterativeCollisionCheckLink.forward
 *       (morefusion/contrib/iterative_collision_check_link.py:31-99), chainer's reverse pass
 *       through it and chainer.optimizers.Adam.update as driven by
 *       examples/ycb_video/pose_refinement/check_iterative_collision_check_link.py:44-79
 * One persistent cooperative kernel runs all `n_iter` (<= 128 per call) iterations for a BATCH of
 * independent scenes; scene s owns objects [scene_obj_off[s], scene_obj_off[s+1]) (<= 32 per
 * scene) and `group_size` CTAs.  Points/sdf are concatenated over all objects (obj_pt_off);
 * work tables: 256-point chunks (chunk_obj / chunk_start, grouped by scene via scene_chunk_off),
 * scene_slot_off = prefix sums of N_s * C_s.  All tables are DEVICE int32 arrays.
 *   update == 0 : one forward/backward, parameters untouched (loss_history, grads written)
 *   update == 1 : Chainer-form Adam, m += (1-b1)(g-m); v += (1-b2)(g*g-v);
 *                 p -= eta * alpha_t[it] * m / (sqrt(v) + eps); alpha_t given per iteration by the
 *                 caller (HOST float arrays) for quaternion and translation separately.
 * adam_state: device [m_q(N,4) | m_t(N,3) | v_q(N,4) | v_t(N,3)].  grads: device [N,7] = gq | gt
 * of the last iteration.  loss_history: device [n_scenes, n_iter].
 * ------------------------------------------------------------------------ */
int mf_icc_max_group_size(int n_scenes);
size_t mf_icc_workspace_bytes(int n_objects_total, int voxel_dim, int n_scenes, int group_size,
                              int n_slots);
int mf_icc_run(int n_scenes, int n_objects_total, int voxel_dim, float voxel_threshold,
               float sdf_offset, const int32_t* scene_obj_off, const int32_t* obj_pt_off,
               const int32_t* scene_chunk_off, const int32_t* chunk_obj,
               const int32_t* chunk_start, const int32_t* scene_slot_off,
               const int32_t* obj_chunk_off /*[N+1] first chunk of each object*/, int n_slots,
               const float* points, const float* sdf, const float* pitch, const float* origin,
               const float* grid_target, const float* grid_nontarget_empty, float* quaternion,
               float* translation, float* adam_state, int n_iter, int update,
               const float* alpha_q_host, const float* alpha_t_host, double beta1, double beta2,
               double eps, double eta, float* loss_history, float* grads, int group_size,
               void* workspace, size_t workspace_bytes, void* stream);
/* same, plus phase_ns: device uint64 [n_scenes][n_iter][8] receiving %globaltimer stamps at the
 * phase boundaries of every iteration (profiling aid; NULL = off) */
int mf_icc_run_profiled(int n_scenes, int n_objects_total, int voxel_dim, float voxel_threshold,
               float sdf_offset, const int32_t* scene_obj_off, const int32_t* obj_pt_off,
               const int32_t* scene_chunk_off, const int32_t* chunk_obj,
               const int32_t* chunk_start, const int32_t* scene_slot_off,
               const int32_t* obj_chunk_off, int n_slots,
               const float* points, const float* sdf, const float* pitch, const float* origin,
               const float* grid_target, const float* grid_nontarget_empty, float* quaternion,
               float* translation, float* adam_state, int n_iter, int update,
               const float* alpha_q_host, const float* alpha_t_host, double beta1, double beta2,
               double eps, double eta, float* loss_history, float* grads, int group_size,
               void* workspace, size_t workspace_bytes, unsigned long long* phase_ns, void* stream);
/* same as mf_icc_run_profiled, with the stopping rule of the reference's refinement node
 * (ros/src/morefusion_ros/nodes/collision_based_pose_refinement.py:18-45,184-206) applied per
 * scene inside the kernel.  After each Adam update the iteration's fp32 loss goes to the scene's
 * observer, in float64: delta = |last - loss| enters a window of the last `window` deltas,
 * m = max of the window in Python's order (oldest first, replaced only on a strict '>'),
 * m < threshold counts a pass (NaN resets the count), and `patience` consecutive passes stop the
 * scene.  The update of the stopping iteration stays applied; after it the scene's q, t, Adam state
 * and grads row are left alone and the rest of its loss_history row is NaN.
 *   observer_state: device, mf_icc_observer_state_bytes(n_scenes) bytes, one record per scene.
 *       Zero-filled = a fresh observer.  The records persist across calls like adam_state does: a
 *       scene that has stopped stays stopped (its CTAs return at once, its loss row is all NaN, its
 *       grads row is not written) until the caller zeroes the buffer for a new run.  Words 0 and 1
 *       (int32) of scene s's record are its `stopped` flag and its iteration count since zeroing.
 *   threshold (finite, >= 0), patience (>= 1) and window (1..32) must stay the same between
 *       zeroings.  update must be 1.
 *   n_iter_run: device int32 [n_scenes] out = iterations run since the buffer was zeroed, the
 *       stopping one included. */
size_t mf_icc_observer_state_bytes(int n_scenes);
int mf_icc_run_early_stop(int n_scenes, int n_objects_total, int voxel_dim, float voxel_threshold,
               float sdf_offset, const int32_t* scene_obj_off, const int32_t* obj_pt_off,
               const int32_t* scene_chunk_off, const int32_t* chunk_obj,
               const int32_t* chunk_start, const int32_t* scene_slot_off,
               const int32_t* obj_chunk_off, int n_slots,
               const float* points, const float* sdf, const float* pitch, const float* origin,
               const float* grid_target, const float* grid_nontarget_empty, float* quaternion,
               float* translation, float* adam_state, int n_iter, int update,
               const float* alpha_q_host, const float* alpha_t_host, double beta1, double beta2,
               double eps, double eta, float* loss_history, float* grads, int group_size,
               void* workspace, size_t workspace_bytes, unsigned long long* phase_ns,
               void* observer_state, size_t observer_state_bytes, double threshold, int patience,
               int window, int32_t* n_iter_run, void* stream);

/* ------------------------------------------------------------------------
 * a10 / a11 fp32-class parity mode ("bf16x3"): every GEMM operand is split hi + lo (bf16 each)
 * and A.W is evaluated as A_hi.W_hi + A_lo.W_hi + A_hi.W_lo on the wgmma GEMMs into fp32
 * slices (mf_gemm_bf16_tc with OUT_F32); these helpers split / combine / gather in fp32
 * (csrc/precise.cu).  Same reference lines as the bf16 path (model.py:93-141, :239-273).
 * ------------------------------------------------------------------------ */
int mf_cnn_point_mlp_f32(const float* values, const float* points, const float* w1_rgb,
                         const float* b1_rgb, const float* w1_pcd, const float* b1_pcd,
                         const float* w2_rgb, const float* b2_rgb, const float* w2_pcd,
                         const float* b2_pcd, int B, int P, float center, void* feat_bf16, int ldf,
                         float* feat2 /*[B*P,144]*/, float* feat1 /*[B*P,72]*/, void* stream);
int mf_px_split(const float* src, long long lds, long long M, int N, void* hi, void* lo,
                long long ldd, int col_off, void* stream);
int mf_px_combine(const float* ws /*[n_slices][M][N]*/, int n_slices, long long M, int N,
                  const float* bias, int relu, int out_mode /*OUT_BF16 | OUT_S2D_BF16*/, int Do,
                  void* hi, void* lo, long long ldo, int col_off, void* stream);
int mf_px_pack_s2d(const float* vox, const float* hocc, int B, int C, int Cocc, int D, void* X_hi,
                   void* X_lo, void* stream);
int mf_px_interp(const void* grid_hi, const void* grid_lo, int s2d, const float* points, int B,
                 int P, int C, int D, float divisor, void* feat_hi, void* feat_lo, int ldf,
                 int col_off, void* stream);
int mf_px_head4_pose(const void* hd3_hi, const void* hd3_lo, int ld, const float* w_rot,
                     const float* b_rot, const float* w_trans, const float* b_trans,
                     const float* w_conf, const float* b_conf, const float* points,
                     const int32_t* class_id, const float* pitch, const float* origin, int B, int P,
                     int nfg, float* rot, float* trans, float* conf, void* stream);

/* ------------------------------------------------------------------------
 * a10 / a11 backward: training step of the 3-D section of singleview_3d.Model
 *     replaces chainer's reverse pass through morefusion/contrib/singleview_3d/models/model.py
 *     :93-141 (_extract) and :239-273 (heads, pose) -- cuDNN backward-data / backward-filter,
 *     interpolate_voxel_grid.py:216-268, average_voxelization_3d.py:147-220 -- and the
 *     ChainerMN-side optimizer step (examples/ycb_video/singleview_3d/train.py:342-344).
 * Activations are the forward's channels-last bf16 buffers; gradients that feed a GEMM are bf16,
 * accumulators and parameter gradients fp32.  All outputs named d* that are described as
 * "accumulated" must be zeroed by the caller once per step.
 * ------------------------------------------------------------------------ */
/* forward variant of mf_cnn_head4_pose that also saves the 8 selected pre-activation outputs */
int mf_cnn_head4_pose_train(const void* hd3, int ld, const void* w_rot, const float* b_rot,
                            const void* w_trans, const float* b_trans, const void* w_conf,
                            const float* b_conf, const float* points, const int32_t* class_id,
                            const float* pitch, const float* origin, int B, int P, int nfg,
                            float* rot, float* trans, float* conf, float* raw8 /*[B*P,8]*/,
                            void* stream);
/* wgmma, both operands MN-major: out[g][n, k] (+)= sum_m dZ[m, g*dz_group_cols + n] *
 * X[m, g*x_group_cols + k]   (Conv1D weight gradients; bf16 operands, fp32 output) */
int mf_train_gemm_tn(const void* dZ, long long ldz, const void* X, long long ldx, int m_rows,
                     int n_out, int k_in, float* out, long long ldo, int n_groups,
                     long long dz_group_cols, long long x_group_cols, long long out_group_stride,
                     int accumulate, void* stream);
/* k4 s2 p1 Conv3D weight gradient in the space-to-depth form of the forward: dYp bf16
 * [B, Do+2, Do+2, Do+2, Co] (zero border), Xs2d bf16 [B, Do+1, Do+1, Do+1, C8]; out fp32
 * [Co][8 * C8] in the packed K order of the forward weights (tap-major) */
int mf_train_conv_wgrad(const void* dYp, const void* Xs2d, int batch, int Do, int Co, int C8,
                        float* out, int accumulate, void* stream);
/* k4 s2 p1 Conv3D input gradient: 8 parity GEMMs over the padded dY; Wd bf16 [8][Ci][8*Co]
 * (per parity r: Wd[r][ci][a*Co+co] = W[co][ci][2a+r]).  epilogue 1: added into a channels-last
 * fp32 grid [B,(2Do)^3,ldo]; epilogue 2: bf16 rows [8][B*Do^3][ldo] in parity order */
int mf_train_conv_dgrad(const void* dYp, const void* Wd, int batch, int Do, int Co, int Ci,
                        int epilogue, void* out, long long ldo, long long out_group_stride,
                        void* stream);
int mf_train_head4_bwd(const float* g_rot, const float* g_trans, const float* g_conf,
                       const float* raw8, const void* hd3, int ld, const void* w_rot,
                       const void* w_trans, const void* w_conf, const int32_t* class_id,
                       const float* pitch, int B, int P, int nfg, void* dhd3 /*bf16, masked*/,
                       float* dw_rot, float* db_rot, float* dw_trans, float* db_trans,
                       float* dw_conf, float* db_conf /*accumulated*/, void* stream);
int mf_train_relu_mask(void* x /*bf16 in/out*/, long long ldx, const void* act, long long lda,
                       long long M, int N, void* stream);
int mf_train_colsum(const void* x /*bf16*/, long long ldx, long long M, int N,
                    float* out /*accumulated*/, void* stream);
int mf_train_interp_bwd(const void* g /*bf16 [B*P, ldg]*/, long long ldg, int col_off,
                        const float* points /*[B,3,P]*/, int B, int P, int C, int D,
                        float divisor, float* dgrid /*[B,D^3,C] accumulated*/, void* stream);
int mf_train_mask_pack(const float* dgrid, const void* act, int act_s2d, int B, int D, int C,
                       void* out /*bf16 [B,(D+2)^3,C], interior written*/,
                       float* dbias /*accumulated, may be NULL*/, void* stream);
int mf_train_vox_bwd(const void* dx3 /*bf16 parity rows*/, long long ldp, const int32_t* keys,
                     int B, int P, int C, int D, const void* g_direct, long long ldg, int col_off,
                     float* dfeat2 /*[B*P, C]*/, void* stream);
int mf_train_point_mlp_bwd(const float* values, const float* points, const void* feat,
                           long long ldf, const void* dfeat, long long ldd, const float* feat2,
                           const float* g2, const float* w1r, const float* w1p, const float* w2r,
                           const float* w2p, int B, int P, float center, float* dw1r,
                           float* db1r, float* dw1p, float* db1p, float* dw2r, float* db2r,
                           float* dw2p, float* db2p /*accumulated*/,
                           float* dvalues /*[B,32,P], may be NULL*/, void* stream);
/* fused gradient unscale (x grad_scale, e.g. 1/world after a sum all-reduce) + chainer Adam on
 * flat fp32 buffers */
int mf_train_adam(float* params, const float* grads, float* m, float* v, int64_t n,
                  float alpha_t, double beta1, double beta2, double eps, double eta,
                  float grad_scale, void* stream);

/* ------------------------------------------------------------------------
 * f2  per-frame front end (SURVEY.md 8f-2): replaces the host NumPy helpers
 *     morefusion/geometry/pointcloud_from_depth.py:4-26 and masks_to_bboxes.py:4-38
 * depth [H,W] f32 metres (NaN = invalid) -> pcd [H,W,3]; masks [N,H,W] u8 -> bboxes [N,4] int32
 * (y1, x1, y2, x2), upper bounds exclusive, zeros for an empty mask.
 * ------------------------------------------------------------------------ */
int mf_pointcloud_from_depth(const float* depth, int H, int W, float fx, float fy, float cx,
                             float cy, int euclidean, float* pcd, void* stream);
int mf_masks_to_bboxes(const uint8_t* masks, int N, int H, int W, int32_t* bboxes, void* stream);
/* Per-instance crops of a labelled frame (datasets/rgbd_pose_estimation/base.py:113-161, the ROS
 * pose node's crop): label [H,W] int32, pcd [H,W,3] f32, lut [lut_n] int32 maps label - lut_lo
 * to the instance slot 0..N-1 (-1 = not requested) -- device arrays.
 * mf_label_bboxes: one pass over the label image -> stats [N,6] int32 per slot:
 *     (y1, x1, y2, x2) of label == id (upper bounds exclusive, zeros when empty), n_mask, n_valid
 *     (mask pixels whose point has no NaN).  N <= 1024 (else MF_E_UNSUPPORTED); workspace of
 *     mf_label_bboxes_workspace_bytes(N) bytes, contents irrelevant.
 * mf_instance_crops: rgb [H,W,3] u8, ids [N] int32 (the instance id of each slot), stats from
 *     mf_label_bboxes -> rgb_ins [N,S,S,3] u8 (bilinear, 0 outside the mask and in the padding)
 *     and pcd_ins [N,S,S,3] f32 (nearest, NaN outside the mask and in the padding): imgviz
 *     centerize of the masked crop with OpenCV's resize rules, every element written. */
size_t mf_label_bboxes_workspace_bytes(int N);
int mf_label_bboxes(const int32_t* label, const float* pcd, int H, int W, const int32_t* lut,
                    int lut_lo, int lut_n, int N, int32_t* stats, void* workspace,
                    size_t workspace_bytes, void* stream);
int mf_instance_crops(const uint8_t* rgb, const float* pcd, const int32_t* label, int H, int W,
                      const int32_t* ids, const int32_t* stats, int N, int S, uint8_t* rgb_ins,
                      float* pcd_ins, void* stream);

/* ------------------------------------------------------------------------
 * f1  2-D extractor tail at the sampled pixels only (SURVEY.md 8f-1): replaces the dense
 *     up3 (resize x2 + Conv2D 64->64 3x3 + PReLU), Conv2D 64->32 1x1 and log_softmax of
 *     morefusion/models/dense_fusion/pspnet.py:64-82 followed by the 1000-pixel gather of
 *     contrib/singleview_3d/models/model.py:222.
 * up2_nhwc [B,Hs,Ws,64] f32 channels-last (output of up2), pix [B,P] int64 row-major pixel index
 * into the 2Hs x 2Ws image, w3t [576,64] = W3[co][ci][dy][dx] transposed to [(ci,dy,dx)][co],
 * b3 [64], prelu_slope [1] (device), w1t [64,32] = W1 transposed, b1 [32] -> out [B,32,P] f32.
 * ------------------------------------------------------------------------ */
int mf_psp_tail_sampled(const float* up2_nhwc, const int64_t* pix, int B, int P, int Hs, int Ws,
                        const float* w3t, const float* b3, const float* prelu_slope,
                        const float* w1t, const float* b1, float* out, void* stream);

/* ------------------------------------------------------------------------
 * f3  occupancy-grid producer (SURVEY.md 8f-3): replaces the OctoMap trees behind
 *     morefusion/contrib/multi_instance_octree_mapping.py:16-34 (initialize / integrate / update)
 *     and :35-94 (get_target_grids).  One caller-owned open-addressing hash table holds the cells
 *     of every instance: cells [capacity] 16-byte entries {u64 key, f32 log-odds, u32 scan stamp}
 *     (16-byte aligned; initialised ONCE to key = all ones, rest zero), cnt u32 [capacity] and
 *     counters int32 [8] (zero at allocation; the kernels keep them consistent afterwards).
 *     capacity is a power of two.  counters[0] = live cells, counters[1] = table full (sticky;
 *     updates were dropped).  `instance` is the caller's dense index (order of initialize()).
 * mf_map_integrate: octree.insertPointCloud(points[mask], origin) (:24): points [n,3] f32 (NaN rows
 *     and rows with mask == 0 are skipped; mask may be NULL), sensor origin as floats, OctoMap's
 *     sensor model as float32 log-odds; scan = 1, 2, ... increasing per table.  Two launches, no
 *     scratch memory.
 * mf_map_integrate_labelled: the same for every instance of a labelled frame in ONE scan (what
 *     datasets/rgbd_pose_estimation/base.py:30-50 and the ROS OctomapServer::insertScan,
 *     ros/.../OctomapServer.cpp:286-395, do instance by instance): labels [n] int32; lut [lut_n]
 *     int32 maps label - lut_lo to the dense instance index (-1 = not mapped: pixel skipped);
 *     inst_resolution [n_instances] f64 -- device arrays.  Equal to one mf_map_integrate per
 *     instance with mask = (labels == id), the instances' cells being disjoint.
 * mf_map_update_points: octree.updateNodes(points, True) (:30): points [m,3] f64, update = the
 *     log-odds increment applied once per row.
 * mf_map_query_grids: get_target_grids for T targets in one launch: target_index [T] int32 (dense
 *     instance index of each target), pitch [T] f64, origin [T,3] f64, res_factor [n_instances] f64
 *     (= 1 / resolution) -- device arrays; outputs [T,X,Y,Z] f32, every element written.
 * mf_map_query_node_grids: the grid / grid_noentry pair the ROS occupancy server publishes for
 *     the refinement node (OctomapServer::publishGrids, ros/src/morefusion_ros/src/
 *     OctomapServer.cpp:510-618), for T targets in one launch; target_index / pitch / origin /
 *     res_factor as in mf_map_query_grids.  Voxel centre origin + pitch * i in double, rounded to
 *     float before the key look-up (:566-575).  grid = the target's occupancy where it is > 0.5
 *     (:586); elsewhere grid_noentry = the occupancy of another instance where it is >=
 *     probability_max, or 1 - occupancy where the background (dense index `background`, -1 =
 *     none) is < 0.5 (free_as_noentry, :597-608).  walk [n_instances] int32 lists the dense
 *     indices in reverse map order (the server's std::map, background first, then ascending
 *     instance id): the first that qualifies is the last the server pushes, which is the value the
 *     node's decoding keeps.  Outputs [T,X,Y,Z] f32, every element written.
 * mf_map_query_node_grids_world: the same with origins in the camera frame: each voxel centre,
 *     rounded to float, is moved to the world frame by sensor_to_world (HOST [12] f32, rows 0-2
 *     of the 4x4, row-major) as pcl::transformPointCloud does with a Matrix4f, ((m0 x + m1 y) +
 *     m2 z) + m3 in float (:573-576), before the look-up.  ground_as_noentry != 0: a centre with
 *     world z < 0 gets grid_noentry = probability_max and nothing else (:579-583).
 * mf_map_integrate_server: the ROS occupancy server's scan (OctomapServer::insertScan, :283-448)
 *     of an organised camera-frame cloud points [height*width,3] f32 with labels [height*width]
 *     int32, moved to the world by sensor_to_world (HOST [12] f32 as above; the sensor origin is
 *     its last column).  Pixels of even row and column only; NaN points skipped; label
 *     `uncertain` or a label the lut maps (lut / lut_lo / lut_n / inst_resolution as in
 *     mf_map_integrate_labelled), other labels skipped.  Inside max_range (< 0: no limit) a pixel
 *     casts a free ray in the background's key space (dense index `background`, resolution
 *     background_resolution), is a hit in its own instance unless uncertain, and, unless labelled
 *     background, also frees its end cell in the background; beyond max_range the free ray stops
 *     at max_range and nothing is hit.  Centres: centre_sums [n_instances,4] u64 and centre_first
 *     [n_instances] u32 are zeroed at allocation (the call leaves them so);
 *     an instance whose centre_set [n_instances] int32 is 0 and that pushed at least one point
 *     gets centre_set = 1 and centres [n_instances,3] f32 = the mean of its listed world points of
 *     this scan, range or not, except the lowest pixel index, summed exactly in fixed point
 *     (2^-32 m).  Boxes: boxes [n_instances,6] u32 hold each instance's (min xyz, max xyz) in an
 *     order-preserving encoding of the floats (negative: bits inverted; otherwise the sign bit
 *     set; a zero is +0); OctoMap's default box (0,0,0)-(0,0,0) at allocation.  tree_state
 *     [n_instances] int32: 1 where the instance has a tree in the server's sense, 0 where not yet;
 *     the scan creates the tree of every instance whose id its labels hold on any pixel (odd rows
 *     and columns and NaN points included, unique(label_ins), :290-319) and sets the flag.  Each
 *     instance other than the background that pushed a point widens its box by those points (the
 *     first excluded) as insertScan's setBBXMin/Max do (:404-437); an instance whose tree this
 *     scan created takes the min / max of them instead, (+FLT_MAX, -FLT_MAX) when there are none,
 *     and keeps the default box when it has no listed point.  Five launches, stream-ordered, no
 *     host sync.
 * mf_map_render: the server's render (OctomapServer::render, :193-281) of the map into the
 *     camera of an organised camera-frame cloud points [height*width,3] f32 (sensor_to_world as
 *     above; fx, fy, cx, cy the intrinsics rounded to float).  walk / walk_ids [n_walk] int32:
 *     dense index / instance id of each rendered instance in ascending id order (the background
 *     left out); boxes as above.  Every even pixel casts castRay(origin, point - origin,
 *     ignoreUnknownCells, 1.1 |point - origin|) into each instance whose box holds its world
 *     point, or, with no depth, to the z = 1 point of its ray with no box test; the nearest hit
 *     (the lower id on a tie) writes its distance to depth [height,width] f32 at the pixel and
 *     its id to label [height,width] int32 on rows v-1..v, columns u-1..u; the rest is
 *     `uncertain` / NaN.  zbuf: workspace of ((height+1)/2)*((width+1)/2) u64.  Two launches
 *     and a memset, stream-ordered, no host sync.
 * mf_map_server_grid_params: publishGrids' pitch [T] f64 (the instance's resolution) and origin
 *     [T,3] f64 of T targets (dense indices, device) from their world centres: the centre moved
 *     by world_to_sensor (HOST [12] f32) in float, minus (off_x, off_y, off_z) * pitch in double
 *     (off = dims / 2 - 0.5, :534-551).
 * mf_map_rehash: move every cell of the old table into a larger, freshly initialised one.
 * ------------------------------------------------------------------------ */
int mf_map_integrate(const float* points, const uint8_t* mask, int64_t n, float ox, float oy,
                     float oz, double resolution, int instance, uint32_t scan, float hit,
                     float miss, float lo_min, float lo_max, void* cells, void* cnt,
                     int64_t capacity, int32_t* counters, void* stream);
int mf_map_integrate_labelled(const float* points, const int32_t* labels, int64_t n, float ox,
                              float oy, float oz, const int32_t* lut, int lut_lo, int lut_n,
                              const double* inst_resolution, uint32_t scan, float hit, float miss,
                              float lo_min, float lo_max, void* cells, void* cnt, int64_t capacity,
                              int32_t* counters, void* stream);
int mf_map_update_points(const double* points, int64_t m, double resolution, int instance,
                         float update, float lo_min, float lo_max, void* cells, void* cnt,
                         int64_t capacity, int32_t* counters, void* stream);
int mf_map_query_grids(const int32_t* target_index, const double* pitch, const double* origin,
                       int T, int X, int Y, int Z, const double* res_factor, int n_instances,
                       void* cells, void* cnt, int64_t capacity, int32_t* counters,
                       float* grid_target, float* grid_nontarget, float* grid_empty, void* stream);
int mf_map_query_node_grids(const int32_t* target_index, const double* pitch, const double* origin,
                            int T, int X, int Y, int Z, const double* res_factor,
                            const int32_t* walk, int n_instances, int background,
                            double probability_max, void* cells, void* cnt, int64_t capacity,
                            int32_t* counters, float* grid, float* grid_noentry, void* stream);
int mf_map_query_node_grids_world(const int32_t* target_index, const double* pitch,
                                  const double* origin, int T, int X, int Y, int Z,
                                  const double* res_factor, const int32_t* walk, int n_instances,
                                  int background, double probability_max,
                                  const float* sensor_to_world, int ground_as_noentry, void* cells,
                                  void* cnt, int64_t capacity, int32_t* counters, float* grid,
                                  float* grid_noentry, void* stream);
int mf_map_integrate_server(const float* points, const int32_t* labels, int height, int width,
                            const float* sensor_to_world, double max_range, const int32_t* lut,
                            int lut_lo, int lut_n, const double* inst_resolution, int n_instances,
                            int background, double background_resolution, int uncertain,
                            uint32_t scan, float hit, float miss, float lo_min, float lo_max,
                            void* centre_sums, uint32_t* centre_first, float* centres,
                            int32_t* centre_set, void* cells, void* cnt, int64_t capacity,
                            int32_t* counters, int32_t* tree_state, uint32_t* boxes, void* stream);
int mf_map_render(const float* points, int height, int width, const float* sensor_to_world,
                  float fx, float fy, float cx, float cy, const int32_t* walk,
                  const int32_t* walk_ids, int n_walk, const double* inst_resolution,
                  const uint32_t* boxes, int uncertain, void* zbuf, int32_t* label, float* depth,
                  void* cells, void* cnt, int64_t capacity, int32_t* counters, void* stream);
int mf_map_server_grid_params(const int32_t* target_index, int T, const double* inst_resolution,
                              const float* centres, const float* world_to_sensor, double off_x,
                              double off_y, double off_z, double* pitch, double* origin,
                              void* stream);
int mf_map_rehash(const void* old_cells, int64_t old_capacity, void* cells, void* cnt,
                  int64_t capacity, int32_t* counters, void* stream);

/* ------------------------------------------------------------------------
 * Object mapping: multi-view pose validation of a static scene
 *     replaces ros/src/morefusion_ros/nodes/object_mapping.py:23-84 (Object) and the pose /
 *     remove / reset callbacks of ObjectMapping (:121-133, :152-233)
 * One caller-owned state blob of mf_objmap_state_bytes(capacity) bytes (16-byte aligned,
 * capacity <= 1024 instance slots; 0 for a capacity out of range) holds, per slot, a ring of the
 * last 6 world poses in float64 (queue.deque([], 6), :34), the spawned / removed flags, the
 * frozen pose and the class's symmetric flag and model-point range.  mf_objmap_reset must run
 * once on a fresh blob; no memset is needed anywhere.
 * plan [n_plan, 8] int32 (device), one row per distinct slot of a view in first-appearance
 * order: slot, first, n (the slot's poses are order[first .. first + n), in message order),
 * points offset, points count (>= 1) of the slot's class in `points`, symmetric, removed before
 * first seen (1: the slot is marked removed, :159-168), unused.
 * mf_objmap_append: one view (:183-233).  quaternion [P,4] f32 (w, x, y, z) and translation [P,3]
 *     f32 as the refinement returns them, widened to double; T(q, t) by quaternion_matrix's
 *     formula (functions/geometry/quaternion_matrix.py:68-80, normalisation included);
 *     cam_to_base [12] f64 (device; rows 0-2 of T_cam2base).  Appends T_cam2base @ T(q, t) to each
 *     slot's ring unless it is spawned (:51-53) and marks the slots that need a vote (not spawned,
 *     not removed, >= n_votes poses).
 * mf_objmap_vote: the votes of the marked slots of the same plan (Object.validate, :55-84).  ADD
 *     (mean |T_new x - T_j x|) or, for symmetric classes, ADD-S (mean over x of the distance from
 *     T_new x to the nearest of all T_j y; metrics/average_distance.py:6-19) of the newest pose
 *     against each earlier pose j, over the class's points [*,3] f64, in float64; a slot spawns
 *     and freezes its newest pose when at least n_votes - 1 distances are below 0.02 (ADD) /
 *     0.01 (ADD-S).  max_points >= every plan row's points count; partials [n_partials] f64
 *     scratch of at least n_plan * 5 * ceil(max_points / 256) (else MF_E_WORKSPACE).
 * mf_objmap_remove: marks slots [n] int32 (device) removed (~input/remove, :152-157).
 * mf_objmap_reset: clears every slot's poses and flags (~reset, :121-133), one kernel.
 * ------------------------------------------------------------------------ */
size_t mf_objmap_state_bytes(int capacity);
int mf_objmap_append(void* state, int capacity, const int32_t* plan, int n_plan,
                     const int32_t* order, const float* quaternion, const float* translation,
                     const double* cam_to_base, int n_votes, void* stream);
int mf_objmap_vote(void* state, int capacity, const int32_t* plan, int n_plan, int max_points,
                   const double* points, int n_votes, double* partials, int64_t n_partials,
                   void* stream);
int mf_objmap_remove(void* state, int capacity, const int32_t* slots, int n, void* stream);
int mf_objmap_reset(void* state, int capacity, void* stream);

/* ------------------------------------------------------------------------
 * a12  average_distance (ADD / ADD-S training loss) + nearest neighbour
 *     replaces morefusion/functions/loss/average_distance.py:40-85 and, for symmetric=1,
 *     morefusion/geometry/knn/nn.py:17-48 + cuComputeDistanceGlobal.cu:20-86 (matrix-free here)
 * points [P,3], transform_true [4,4], transforms_pred [M,4,4] -> out [M];
 * nn_indices [M,P] int32 (may be NULL when symmetric == 0) is kept for the backward pass.
 * ------------------------------------------------------------------------ */
int mf_average_distance_fwd(const float* points, int n_points, const float* transform_true,
                            const float* transforms_pred, int n_pred, int symmetric, float* out,
                            int32_t* nn_indices, void* stream);
/* same forward with the query points split over n_parts CTAs per pose (few poses, many points:
 * the evaluation metrics); out_parts [n_pred, n_parts] holds partial means, their sum is the
 * distance */
int mf_average_distance_fwd_parts(const float* points, int n_points, const float* transform_true,
                                  const float* transforms_pred, int n_pred, int symmetric,
                                  int n_parts, float* out_parts, int32_t* nn_indices, void* stream);
int mf_average_distance_bwd(const float* gout, const float* points, int n_points,
                            const float* transform_true, const float* transforms_pred, int n_pred,
                            const int32_t* nn_indices /*NULL: identity*/,
                            float* g_transforms_pred /*[M,4,4]*/, float* g_transform_true /*[4,4]*/,
                            float* workspace /*[n_pred,12] floats*/, void* stream);
/* the same over the B objects of a training batch from one call (model.py:416-431 calls
 * average_distance per object): points [B,n_points,3], transform_true [B,4,4], transforms_pred
 * [B,n_pred,4,4], out [B,n_pred], nn_indices [B,n_pred,n_points]; symmetric = HOST array [B] */
int mf_average_distance_fwd_batched(const float* points, int n_points, const float* transform_true,
                                    const float* transforms_pred, int n_pred, int B,
                                    const int32_t* symmetric_host, float* out, int32_t* nn_indices,
                                    void* stream);
int mf_average_distance_bwd_batched(const float* gout, const float* points, int n_points,
                                    const float* transform_true, const float* transforms_pred,
                                    int n_pred, int B, const int32_t* symmetric_host,
                                    const int32_t* nn_indices, float* g_transforms_pred,
                                    float* g_transform_true, float* workspace /*[B,n_pred,12]*/,
                                    void* stream);

/* ------------------------------------------------------------------------
 * Point-to-point ICP (contrib.ICPRegistration; the pose node's ~icp option)
 *     replaces morefusion/contrib/icp_registration.py:15-44 (Open3D's voxel_down_sample and
 *     registration_icp with TransformationEstimationPointToPoint(False)), called per instance at
 *     ros/src/morefusion_ros/nodes/singleview_3d_pose_estimation.py:246-264.  float64 throughout;
 *     the algorithm is stated in oracle/icp.py.
 * mf_icp_voxel_down_sample (icp_registration.py:22-23): M clouds points [M,N,3] (float32, or
 *     float64 with points_f64 = 1); rows with a non-finite coordinate are skipped (the crops' NaN
 *     rows).  Per cloud: min_bound = min - voxel_size / 2, voxel = floor((p - min_bound) /
 *     voxel_size); writes one row per occupied voxel in ascending (i, j, k) at means[m*N ...]
 *     [*,3] f64 (the mean of its points, summed in row order), keys [*,3] int32, counts [*] int32,
 *     and n_out[m], the number of voxels (<= the cloud's finite rows, so nothing can overflow).
 *     A cloud whose keys reach 2^31 - 1 on an axis is refused, n_out[m] = -1 and no row written,
 *     rather than having voxels merged at the int32 limit; mf_icp_cell_list refuses such a cloud
 *     with a NaN origin, and mf_icp_run gives an instance with a refused source or target NaN
 *     transform, fitness and rmse and 0 iterations.
 *     One CTA per cloud; deterministic.  workspace: mf_icp_sort_workspace_bytes(M, N).
 * mf_icp_cell_list: a uniform cell list of side cell_size over the first *n_points rows of one
 *     float64 cloud [N,3] (the down-sampled CAD cloud): the rows sorted by cell (i, j, k)
 *     (sorted_points [N,3], cells [N,3] int32, index [N] = the row) and origin [3] = min -
 *     cell_size / 2.  workspace: mf_icp_sort_workspace_bytes(1, N).
 * mf_icp_run (icp_registration.py:32-44): every iteration of M instances in one launch.
 *     source [M,N,3] f64 with n_source[M] rows each (mf_icp_voxel_down_sample's output);
 *     targets [M] (device) the cell list each instance registers to; transform_init [M,4,4] f64
 *     (device) with the same values on the host (transform_init_host, checked finite before
 *     launch).  Correspondence = nearest target with d^2 < max_distance^2 (ties to the lowest
 *     index), the Umeyama rotation (Horn's closed form), stop when |d fitness| <
 *     relative_fitness and |d rmse| < relative_rmse or after max_iteration.  Writes transform
 *     [M,4,4] f64, fitness [M], rmse [M] f64 and iterations [M] int32.
 *     workspace: mf_icp_run_workspace_bytes(M, N).
 * ------------------------------------------------------------------------ */
typedef struct {
  const double* points;   /* [n,3] sorted by cell */
  const int32_t* cells;   /* [n,3] */
  const int32_t* index;   /* [n] row in the down-sampled cloud */
  const int32_t* count;   /* n (device) */
  const double* origin;   /* [3] */
  double cell_size;       /* >= the max_distance it is searched with */
} mf_icp_target;
size_t mf_icp_sort_workspace_bytes(int M, int N);
int mf_icp_voxel_down_sample(const void* points, int points_f64, int M, int N, double voxel_size,
                             double* means, int32_t* keys, int32_t* counts, int32_t* n_out,
                             void* workspace, size_t workspace_bytes, void* stream);
int mf_icp_cell_list(const double* points, const int32_t* n_points, int N, double cell_size,
                     double* sorted_points, int32_t* cells, int32_t* index, double* origin,
                     void* workspace, size_t workspace_bytes, void* stream);
size_t mf_icp_run_workspace_bytes(int M, int N);
int mf_icp_run(int M, const double* source, int N, const int32_t* n_source,
               const mf_icp_target* targets, const double* transform_init,
               const double* transform_init_host, double max_distance, int max_iteration,
               double relative_fitness, double relative_rmse, double* transform, double* fitness,
               double* rmse, int32_t* iterations, void* workspace, size_t workspace_bytes,
               void* stream);

/* ------------------------------------------------------------------------
 * Occupancy registration (contrib.occupancy_registration.register_batch; FramePoseEstimator.occupancy)
 *     replaces OccupancyRegistration.register (morefusion/contrib/occupancy_registration.py:62-139,
 *     the link's forward :21-59, chainer Adam with translation alpha x 0.1 :99-101) as
 *     examples/ycb_video/dense_fusion/eval_densefusion_occupancy.py:68-120 calls it per instance.
 * mf_occupancy_registration_run: every iteration of M independent instances in one launch, one
 *     CTA each, no host read between iterations.  points [M,N,3] f32 (rows >= n_points[m]
 *     ignored, non-finite rows contribute nothing); grids [M,C,X,Y,Z] f32 (C = 2: occupied,
 *     unoccupied; C = 3: occupied, then unoccupied = max of the other two); pitch [M], origin
 *     [M,3], q_init [M,4] (w, x, y, z), t_init [M,3], n_points [M] int32: device.  pitch_host
 *     [M]: the same pitches on the host, checked before launch, or NULL (then an instance whose
 *     pitch is not positive and finite gets NaN results).  Writes q_out [M,4], t_out [M,3],
 *     loss_history [M,iteration] (the loss of every iteration, before its Adam step) and, when
 *     grad_last is not NULL, grad_last [M,7] = (d q, d t) of the last iteration evaluated (NaN
 *     when iteration = 0).  q is not renormalised between steps.  Deterministic: no float
 *     atomics, every sum in a fixed order; an instance's result does not depend on M.
 *     Returns MF_E_BADARG for M < 0, C not 2 or 3, iteration < 0, threshold <= 0 (or >= 2^20),
 *     a pitch_host entry <= 0, and MF_E_UNSUPPORTED for X Y Z > 32^3, before any launch; never
 *     synchronises.  workspace: mf_occupancy_registration_workspace_bytes(M, X, Y, Z).
 * ------------------------------------------------------------------------ */
size_t mf_occupancy_registration_workspace_bytes(int M, int X, int Y, int Z);
int mf_occupancy_registration_run(int M, const float* points, int N, const int32_t* n_points,
                                  const float* grids, int C, int X, int Y, int Z,
                                  const float* pitch, const float* origin, const float* pitch_host,
                                  float threshold, const float* q_init, const float* t_init,
                                  int iteration, double alpha, float* q_out, float* t_out,
                                  float* loss_history, float* grad_last, void* workspace,
                                  size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * IterativeClosestPointLink (contrib.IterativeClosestPointLink; contrib.iterative_closest_point_link.
 *     refine_batch)
 *     replaces IterativeClosestPointLink.forward (morefusion/contrib/iterative_closest_point_link.py:
 *     26-44), its reverse pass and chainer Adam (translation alpha x 0.1) as
 *     examples/ycb_video/pose_refinement/check_iterative_closest_point_link.py drives them.
 * mf_icp_link_run: `iteration` steps of M independent instances in one launch, one cluster of
 *     CTAs each, no host read between iterations.  sources [M,N,3] (CAD points; rows >= n_sources[m]
 *     ignored), targets [M,K,3] (depth points; rows >= n_targets[m] ignored), n_sources [M],
 *     n_targets [M] int32, q_init [M,4] (w, x, y, z), t_init [M,3]: device.  Per step, with
 *     s_j = T(q, t) [p_j, 1]: every target takes its first nearest source j(i) by fp32 squared
 *     distance d2 (a NaN d2 counts as the smallest, the first NaN wins: numpy's argmin), is kept when
 *     d2 < float32(0.02) (a NaN row is dropped), loss = sum of the kept d2, and (d q, d t) flow
 *     through s_{j(i)} only.  update = 1: one Chainer-Adam step per iteration with alpha_t of q and
 *     of t from step_alpha [iteration,2] (device float32) and moments adam_state [M,14] = (m_q, m_t,
 *     v_q, v_t), read and written back; update = 0: the parameters do not move (the forward: pass
 *     iteration = 1; step_alpha and adam_state may be NULL).  Writes q_out [M,4], t_out [M,3],
 *     loss_history [M,iteration] (each iteration's loss, before its step), grad_last [M,7] =
 *     (d q, d t) of the last iteration (NaN when iteration = 0) when not NULL, and match [M,K], when
 *     not NULL, of the last iteration: j(i) for a kept target, -1 - j(i) for a dropped one (rows
 *     >= n_targets[m] untouched).  Deterministic: targets are summed in fixed chunks in an order
 *     that depends only on the instance's n_targets, so results do not depend on M, the batch's
 *     order or cluster_size (0 = chosen from K, mf_icp_link_cluster_size; 1..8 forces it).
 *     Returns MF_E_BADARG for M, N, K or iteration < 0 or cluster_size outside [0, 8], and
 *     MF_E_UNSUPPORTED for N > MF_ICP_LINK_MAX_SOURCES (the transformed sources live in shared
 *     memory, 16 B each), before any launch; never synchronises.
 *     workspace: mf_icp_link_workspace_bytes(M, K).
 * ------------------------------------------------------------------------ */
#define MF_ICP_LINK_MAX_SOURCES 12288
size_t mf_icp_link_workspace_bytes(int M, int K);
int mf_icp_link_cluster_size(int K);
int mf_icp_link_run(int M, const float* sources, int N, const int32_t* n_sources,
                    const float* targets, int K, const int32_t* n_targets, const float* q_init,
                    const float* t_init, int iteration, int update, const float* step_alpha,
                    float* adam_state, float* q_out, float* t_out, float* loss_history,
                    float* grad_last, int32_t* match, int cluster_size, void* workspace,
                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Validation metric: float64 ADD / ADD-S of M pose pairs (metrics.average_distance_batch)
 *     replaces morefusion/metrics/average_distance.py:6-19 (trimesh.transform_points in float64,
 *     a float64 KD-tree over the second transform's points), batched over instances.
 * mf_pose_metrics: points [Ntot,3] f64, the CAD points of every class back to back; offsets
 *     [S+1] int64, segment s is points[offsets[s] .. offsets[s+1]) (every segment non-empty);
 *     seg [M] int32, the segment of each instance; transform1, transform2 [M,4,4] f64 row-major;
 *     translate = 0 drops column 3 of both.  units [n_units,2] int32 (instance, chunk): every
 *     instance's ceil(n/256) chunks, consecutive and in chunk order.  All device.  Writes out
 *     [M,2] f64 = (ADD, ADD-S): with p1 = T1 x and p2 = T2 x, ADD = mean |p1 - p2|, ADD-S = mean
 *     over p1 of the distance to the nearest p2.  Two launches (chunk sums, then each instance's
 *     sum in chunk order), no host read; an instance's result does not depend on M or on the
 *     other instances.  M = 0 returns MF_OK without a launch; MF_E_BADARG for n_units < M.
 *     workspace: mf_pose_metrics_workspace_bytes(n_units) bytes, no initial contents.
 * ------------------------------------------------------------------------ */
size_t mf_pose_metrics_workspace_bytes(int n_units);
int mf_pose_metrics(int M, const double* points, const int64_t* offsets, const int32_t* seg,
                    const double* transform1, const double* transform2, int translate,
                    const int32_t* units, int n_units, void* workspace, size_t workspace_bytes,
                    double* out, void* stream);

/* ------------------------------------------------------------------------
 * Training examples (datasets.RGBDPoseEstimationDatasetBase.get_example and
 * contrib.singleview_3d.Transform): replaces _get_grid_full of
 *     morefusion/datasets/rgbd_pose_estimation/base.py:52-76, :179-195 and the grid part of
 *     examples/ycb_video/singleview_3d/train.py:27-140 (Transform.__call__).  Every grid is
 *     [., 32, 32, 32], C order (i, j, k).
 * mf_training_full_grids: the full grids of M kept instances of one frame (M <= 64, else
 *     MF_E_UNSUPPORTED).  points [Ntot,3] f64, the solid points of every class back to back;
 *     offsets [S+1] int64, segment s is points[offsets[s] .. offsets[s+1]); seg [M] int32, the
 *     segment of each instance; max_points >= the largest of its instances' segment lengths;
 *     Rt [M,3,4] f64 row-major, the ground-truth cad->camera transform; origin [M,3] f32, pitch
 *     [M] f64, each instance's grid.  All device.  p' = ((r0 x + r1 y) + r2 z) + t (f64, no
 *     FMA), index = rint((p' - origin) / pitch), kept when inside the grid.  Writes
 *     target_full[i] = 1 where instance i's own points land, nontarget_full[i] = the largest
 *     rank + 1 of the other instances landing there (rank = j for j < i, j - 1 for j > i), 0
 *     elsewhere; both are zeroed by the call.  Two launches, no host read.
 * mf_training_nontarget_present: present [B] u64, bit v - 1 set when value v in 1..64 occurs in
 *     nontarget_full[b] (the values mf_training_full_grids writes; others are ignored here and
 *     count as not selected in mf_training_transform).  One launch.
 * mf_training_transform: from the map's grid_target / grid_nontarget / grid_empty [B,...] f32
 *     and the full grids, writes grid_target_out = grid_target > 0.5 and grid_nontarget_empty_out
 *     (uint8 0/1) for case_code [B] int32 (0 none, 1 empty, 2 nontarget, 3 empty+nontarget,
 *     4 nontarget_full, 5 empty+nontarget_full, 6 other_full, 7 nontarget_full+other_full,
 *     8 empty+nontarget_full+other_full) and selected [B] u64 (bit v - 1: nontarget value v is
 *     chosen).  One launch; MF_E_UNSUPPORTED when B * 128 exceeds 2^31 - 1.
 * ------------------------------------------------------------------------ */
#define MF_TRAINING_MAX_INSTANCES 64
int mf_training_full_grids(int M, const double* points, const int64_t* offsets, const int32_t* seg,
                           int max_points, const double* Rt, const float* origin,
                           const double* pitch, int32_t* target_full, int32_t* nontarget_full,
                           void* stream);
int mf_training_nontarget_present(int B, const int32_t* nontarget_full, uint64_t* present,
                                  void* stream);
int mf_training_transform(int B, const float* grid_target, const float* grid_nontarget,
                          const float* grid_empty, const int32_t* target_full,
                          const int32_t* nontarget_full, const int32_t* case_code,
                          const uint64_t* selected, uint8_t* grid_target_out,
                          uint8_t* grid_nontarget_empty_out, void* stream);

/* ------------------------------------------------------------------------
 * CAD render (geometry.render_cad; the masks and depth of extra/_pybullet.py:215-288
 * render_cad, each pose rendered alone; oracle/render_cad.py states the rules).
 * mf_render_cad: N poses of S meshes packed back to back.  vertices [V,3] f64 and faces [F,3]
 *     int32 (indices into vertices) on the device; offsets [S+1] int64 on the HOST, mesh s is
 *     faces[offsets[s] .. offsets[s+1]) (offsets[0] = 0, non-decreasing, offsets[S] = F,
 *     1 <= S <= MF_RENDER_CAD_MAX_MESHES); mesh [N] int32 and Ts_cad2cam [N,4,4] f64 row-major
 *     on the device.  f = (height / 2) / tan(fovy / 2) in pixels, principal point at the image
 *     centre.  Writes depth [N,height,width] f32 (NaN where nothing covers), mask [N,height,width]
 *     u8 0/1 and count [N] int32 (mask pixels).  A face with a vertex index outside [0, V) is
 *     dropped (the binding rejects such faces on the host before upload); a pose whose mesh index
 *     is outside [0, S) renders nothing.  Three launches, no host read, no memset; outputs are
 *     bitwise identical between runs.  MF_E_BADARG, before any launch, for height or width <= 0,
 *     height * width >= 2^30, N, F or V < 0, bad offsets, f not finite and positive, or a NULL
 *     pointer the call needs; N = 0 returns MF_OK without a launch.  workspace:
 *     mf_render_cad_workspace_bytes(N, F, height, width) bytes, no initial contents.
 * ------------------------------------------------------------------------ */
#define MF_RENDER_CAD_MAX_MESHES 64
size_t mf_render_cad_workspace_bytes(int N, int F, int height, int width);
int mf_render_cad(const double* vertices, int V, const int32_t* faces, int F,
                  const int64_t* offsets, int S, const int32_t* mesh, const double* Ts_cad2cam,
                  int N, double f, int height, int width, float* depth, uint8_t* mask,
                  int32_t* count, void* workspace, size_t workspace_bytes, void* stream);

/* mf_render_scene (geometry.render_instances; the depth and instance image of the picking-order
 *     node's _render_object_pose_array, ros/.../select_picking_order.py:129-190): N posed objects
 *     rendered together into one camera.  Meshes, mesh [N], Ts_cad2cam [N,4,4], f and the
 *     argument checks are those of mf_render_cad, and each object's coverage and depth are the
 *     bits mf_render_cad gives it alone.  instance_ids [N] int32 on the device.  The visible
 *     object of a pixel is the one of smallest float32 depth; an exact tie goes to the lower
 *     index.  Writes depth [height,width] f32 (NaN where nothing covers), ins [height,width]
 *     int32 (instance_ids of the visible object, -1 where nothing covers), whole [N] int32 (the
 *     pixels each object covers alone, = mf_render_cad's count) and occluded [N,N] int32
 *     (occluded[i][j]: pixels object i covers where object j is visible; zero diagonal).  Four
 *     launches, no host read, no memset; outputs are bitwise identical between runs.
 *     N > MF_RENDER_SCENE_MAX_OBJECTS returns MF_E_UNSUPPORTED before any launch.  N = 0 writes
 *     the empty image (NaN / -1) in one launch; mesh, Ts_cad2cam, instance_ids, whole, occluded
 *     and workspace may then be NULL.  workspace: mf_render_cad_workspace_bytes(N, F, height,
 *     width) bytes, no initial contents. */
#define MF_RENDER_SCENE_MAX_OBJECTS 64
int mf_render_scene(const double* vertices, int V, const int32_t* faces, int F,
                    const int64_t* offsets, int S, const int32_t* mesh, const double* Ts_cad2cam,
                    const int32_t* instance_ids, int N, double f, int height, int width,
                    float* depth, int32_t* ins, int32_t* whole, int32_t* occluded,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Model data from CAD meshes (datasets.MeshModels; what YCBVideoModels derives with binvox and
 * trimesh, datasets/ycb_video/models.py:56-115; oracle/mesh_models.py states the rules).
 * Meshes are packed as for mf_render_cad: vertices [V,3] f64 and faces [F,3] int32 on the
 * device, offsets [S+1] int64 on the HOST (1 <= S <= MF_MESH_MODELS_MAX_MESHES).  Face indices
 * must lie in [0, V) (the binding checks them on the host).
 * mf_mesh_voxelize_solid: the D^3 solid grid of every mesh (1 <= D <= MF_MESH_MODELS_MAX_DIM):
 *     translate [S,3], scale [S] (largest extent of the referenced vertices) and pitch [S]
 *     (scale / D); matrix [S,D,D,D] u8 0/1 (i along x), filled when a face overlaps the voxel's
 *     closed box or the voxel centre is inside by +z ray parity; counts [S] int32; points
 *     [S,D^3,3] f64, mesh s's filled centres in ascending (i, j, k) in its first counts[s] rows
 *     and NaN in the rest.  A mesh without faces, or with a zero or non-finite extent, has pitch
 *     0 and an empty grid.  Seven launches, no host read; outputs are bitwise identical between
 *     runs.  workspace: mf_mesh_voxelize_workspace_bytes(S, D) bytes, no initial contents.
 * mf_mesh_signed_distance: points [P,3] f64 and mesh [P] int32 on the device.  Writes sdf [P] f64
 *     (the distance to the nearest face of the point's mesh, positive inside by the +z parity
 *     rule) and face [P] int32 (that face, the lowest index on a tie).  A point whose mesh is
 *     outside [0, S), or that has a non-finite coordinate, gets NaN and -1.  Two launches, no
 *     host read; bitwise identical between runs and to per-mesh calls.  workspace:
 *     mf_mesh_signed_distance_workspace_bytes(P, f_max) bytes (f_max: the largest mesh's face
 *     count), no initial contents.
 * Both return MF_E_BADARG, before any launch, for bad offsets, sizes or NULL pointers.
 * ------------------------------------------------------------------------ */
#define MF_MESH_MODELS_MAX_MESHES 64
#define MF_MESH_MODELS_MAX_DIM 128
size_t mf_mesh_voxelize_workspace_bytes(int S, int D);
int mf_mesh_voxelize_solid(const double* vertices, int V, const int32_t* faces, int F,
                           const int64_t* offsets, int S, int D, uint8_t* matrix, int32_t* counts,
                           double* points, double* translate, double* scale, double* pitch,
                           void* workspace, size_t workspace_bytes, void* stream);
size_t mf_mesh_signed_distance_workspace_bytes(int P, int f_max);
int mf_mesh_signed_distance(const double* vertices, int V, const int32_t* faces, int F,
                            const int64_t* offsets, int S, const double* points,
                            const int32_t* mesh, int P, double* sdf, int32_t* face,
                            void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MOREFUSION_B200_H_ */
