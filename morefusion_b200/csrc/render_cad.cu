// Masks and depth of posed CAD meshes, each pose rendered alone (extra/_pybullet.py:215-288,
// render_cad): the rules of oracle/render_cad.py, bit for bit.
//
// k_rc_init    one thread per pose: the pose's pixel box opens empty and count[pose] = 0, so the
//              sequence needs no memset.
// k_rc_setup   one thread per (pose, face of the pose's mesh): the three vertices transformed as
//              ((r0 x + r1 y) + r2 z) + t in float64, projected u = (f X) / Z + W / 2,
//              v = (f Y) / Z + H / 2 and snapped to 1/256 pixel with rint.  A face with a vertex
//              at Z < near, a non-finite vertex, a snapped coordinate beyond +-2^30, a vertex index
//              outside [0, V) or zero area is dropped (empty pixel box).  The kept face is
//              oriented to positive area and written as a record: its pixel box (the pixels whose
//              centre lies in the face's snapped bounding box, clipped to the image) and its
//              geometry (snapped vertices, top-left flags, 1/Z of each vertex, twice the area).
//              Non-empty boxes fold into the pose's box with integer atomics.
// k_rc_raster  one CTA per (16x16 tile, pose), a thread per pixel.  A tile outside the pose's
//              box writes NaN / 0 and stops.  Otherwise the pose's face boxes stream through in
//              chunks of 256; the faces whose box meets the tile are gathered into shared memory
//              and each pixel tests them (rc_cover), keeping its covered flag and minimum depth in
//              registers.  __syncthreads_count gives the tile's covered count, which one integer
//              atomic adds to count[pose].
//
// Union and minimum do not depend on order, and count is an integer sum, so every output is
// bitwise identical between runs.  Built with -fmad=false; the float64 expressions also use the
// _rn intrinsics so their order and rounding are explicit.
//
// Coverage is exact integer arithmetic on the snapped coordinates (1/256 pixel).  With every
// coordinate in [-2^30, 2^30] and the pixel centre inside the face's bounding box, each edge
// function is below 2^63 in magnitude, so int64 cannot overflow.
#include <math.h>

#ifdef MF_HOST_EMU
// tests/emu/render_cad_emu.cpp runs these kernels' per-thread code serially on the host against
// oracle/render_cad.py in the CPU test suite; the stubs supply the CUDA spellings used below.
#include "mapping_emu_stubs.h"
#include "render_cad_emu_stubs.h"
#include "../../include/morefusion_b200.h"
#else
#include "common.cuh"
#endif

namespace mf {

constexpr int RC_TILE = 16;
constexpr int RC_THREADS = RC_TILE * RC_TILE;
constexpr int RC_SNAP = 256;                     // subpixel steps per pixel
constexpr long long RC_LIMIT = 1LL << 30;        // largest |snapped coordinate| kept
constexpr double RC_NEAR = 0.01;                 // get_camera_image's near plane (_pybullet.py:229)
constexpr int RC_EMPTY_LO = 0x7fffffff;          // an empty box: lo = INT_MAX, hi = -1

// pixel box of a face: columns x0..x1, rows y0..y1 (inclusive); empty when x0 > x1
struct RcBox {
  int x0, y0, x1, y1;
};

struct __align__(16) RcGeom {
  int ax, ay, bx, by, cx, cy;  // snapped vertices, positive orientation
  int tl;                      // bit k: edge k (0 = b->c, 1 = c->a, 2 = a->b) is top or left
  int pad;
  double iza, izb, izc;        // 1 / Z of each vertex
  double area2;                // twice the snapped area, > 0
};

struct RcParams {
  const double* v;
  const int32_t* faces;
  const int32_t* mesh;         // [N] mesh of each pose
  const double* T;             // [N,4,4]
  int V, F, N, S, H, W, f_max;
  double f;
  int off[MF_RENDER_CAD_MAX_MESHES + 1];
};

__device__ __forceinline__ long long rc_floor256(long long a) { return a >> 8; }
__device__ __forceinline__ long long rc_ceil256(long long a) { return -((-a) >> 8); }

// top or left edge from a to a + (dx, dy), for a triangle of positive area in y-down pixel
// coordinates: the interior lies below a horizontal edge running +x, right of an edge running -y
__device__ __forceinline__ int rc_top_left(long long dx, long long dy) {
  return (dy < 0 || (dy == 0 && dx > 0)) ? 1 : 0;
}

// e(a, b; p) = (bx - ax)(py - ay) - (by - ay)(px - ax)
__device__ __forceinline__ long long rc_edge(long long ax, long long ay, long long bx, long long by,
                                             long long px, long long py) {
  return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}

// camera-frame point of CAD vertex i under the row-major 4x4 T; ((r0 x + r1 y) + r2 z) + t
__device__ __forceinline__ void rc_xform(const double* T, const double* p, double& X, double& Y,
                                         double& Z) {
  const double x = p[0], y = p[1], z = p[2];
  X = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[1], y)), __dmul_rn(T[2], z)), T[3]);
  Y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], x), __dmul_rn(T[5], y)), __dmul_rn(T[6], z)), T[7]);
  Z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], x), __dmul_rn(T[9], y)), __dmul_rn(T[10], z)), T[11]);
}

// snapped pixel coordinate rint(256 ((f c) / Z + half)); false when it must drop the face
__device__ __forceinline__ bool rc_snap(double f, double c, double Z, double half, long long& s) {
  const double u = __dmul_rn(__dadd_rn(__ddiv_rn(__dmul_rn(f, c), Z), half), (double)RC_SNAP);
  const double r = rint(u);
  if (!(fabs(r) <= (double)RC_LIMIT)) return false;   // also NaN and inf
  s = (long long)r;
  return true;
}

// The record of face `face` (global index) under pose n; returns false (box empty) when dropped.
__device__ __forceinline__ bool rc_face(const RcParams& p, int n, int face, RcBox& box,
                                        RcGeom& g) {
  box.x0 = box.y0 = RC_EMPTY_LO;
  box.x1 = box.y1 = -1;
  const double* T = p.T + (size_t)n * 16;
  long long sx[3], sy[3];
  double iz[3];
  for (int k = 0; k < 3; ++k) {
    const int vi = p.faces[3 * (size_t)face + k];
    if (vi < 0 || vi >= p.V) return false;
    double X, Y, Z;
    rc_xform(T, p.v + 3 * (size_t)vi, X, Y, Z);
    if (!(Z >= RC_NEAR) || !isfinite(X) || !isfinite(Y) || !isfinite(Z)) return false;
    if (!rc_snap(p.f, X, Z, 0.5 * p.W, sx[k]) || !rc_snap(p.f, Y, Z, 0.5 * p.H, sy[k])) return false;
    iz[k] = __ddiv_rn(1.0, Z);
  }
  long long a2 = rc_edge(sx[0], sy[0], sx[1], sy[1], sx[2], sy[2]);
  if (a2 == 0) return false;
  if (a2 < 0) {                                     // no culling: orient to positive area
    long long t = sx[1]; sx[1] = sx[2]; sx[2] = t;
    t = sy[1]; sy[1] = sy[2]; sy[2] = t;
    const double d = iz[1]; iz[1] = iz[2]; iz[2] = d;
    a2 = -a2;
  }
  const long long lx = min(min(sx[0], sx[1]), sx[2]), hx = max(max(sx[0], sx[1]), sx[2]);
  const long long ly = min(min(sy[0], sy[1]), sy[2]), hy = max(max(sy[0], sy[1]), sy[2]);
  // pixel c has its centre at 256 c + 128
  const long long c0 = max(rc_ceil256(lx - RC_SNAP / 2), 0LL);
  const long long c1 = min(rc_floor256(hx - RC_SNAP / 2), (long long)p.W - 1);
  const long long r0 = max(rc_ceil256(ly - RC_SNAP / 2), 0LL);
  const long long r1 = min(rc_floor256(hy - RC_SNAP / 2), (long long)p.H - 1);
  if (c0 > c1 || r0 > r1) return false;
  g.ax = (int)sx[0]; g.ay = (int)sy[0];
  g.bx = (int)sx[1]; g.by = (int)sy[1];
  g.cx = (int)sx[2]; g.cy = (int)sy[2];
  g.tl = rc_top_left(sx[2] - sx[1], sy[2] - sy[1]) | (rc_top_left(sx[0] - sx[2], sy[0] - sy[2]) << 1)
         | (rc_top_left(sx[1] - sx[0], sy[1] - sy[0]) << 2);
  g.pad = 0;
  g.iza = iz[0]; g.izb = iz[1]; g.izc = iz[2];
  g.area2 = (double)a2;
  box.x0 = (int)c0; box.x1 = (int)c1; box.y0 = (int)r0; box.y1 = (int)r1;
  return true;
}

// Does the face cover the centre of pixel (col, row)?  If so, lower zmin to its depth there:
// with w_a = e(b, c; p), w_b = e(c, a; p), w_c = e(a, b; p),
//   z = area2 / ((w_a / Z_a + w_b / Z_b) + w_c / Z_c)   (float64, each w converted first)
// rounded to float32.  The pixel must lie in the face's box.
__device__ __forceinline__ void rc_cover(const RcGeom& g, int col, int row, bool& hit, float& zmin) {
  const long long px = (long long)col * RC_SNAP + RC_SNAP / 2;
  const long long py = (long long)row * RC_SNAP + RC_SNAP / 2;
  const long long wa = rc_edge(g.bx, g.by, g.cx, g.cy, px, py);
  const long long wb = rc_edge(g.cx, g.cy, g.ax, g.ay, px, py);
  const long long wc = rc_edge(g.ax, g.ay, g.bx, g.by, px, py);
  const bool in = (wa > 0 || (wa == 0 && (g.tl & 1))) && (wb > 0 || (wb == 0 && (g.tl & 2)))
                  && (wc > 0 || (wc == 0 && (g.tl & 4)));
  if (!in) return;
  const double s = __dadd_rn(__dadd_rn(__dmul_rn((double)wa, g.iza), __dmul_rn((double)wb, g.izb)),
                             __dmul_rn((double)wc, g.izc));
  const float z = __double2float_rn(__ddiv_rn(g.area2, s));
  zmin = hit ? fminf(zmin, z) : z;
  hit = true;
}

__device__ __forceinline__ bool rc_pose_mesh(const RcParams& p, int n, int& lo, int& hi) {
  const int m = p.mesh[n];
  if (m < 0 || m >= p.S) return false;
  lo = p.off[m];
  hi = p.off[m + 1];
  return true;
}

__global__ void k_rc_init(int N, int4* __restrict__ pose_box, int32_t* __restrict__ count) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  pose_box[n] = make_int4(RC_EMPTY_LO, RC_EMPTY_LO, -1, -1);
  count[n] = 0;
}

__global__ void __launch_bounds__(RC_THREADS) k_rc_setup(RcParams p, RcBox* __restrict__ boxes,
                                                          RcGeom* __restrict__ geom,
                                                          int4* __restrict__ pose_box) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.N * p.f_max) return;
  const int n = (int)(i / p.f_max);
  const int j = (int)(i - (long long)n * p.f_max);
  int lo, hi;
  if (!rc_pose_mesh(p, n, lo, hi) || lo + j >= hi) return;
  const size_t r = (size_t)n * p.F + lo + j;
  RcBox b;
  RcGeom g;
  if (rc_face(p, n, lo + j, b, g)) {
    geom[r] = g;
    atomicMin(&pose_box[n].x, b.x0);
    atomicMin(&pose_box[n].y, b.y0);
    atomicMax(&pose_box[n].z, b.x1);
    atomicMax(&pose_box[n].w, b.y1);
  }
  boxes[r] = b;
}

#ifndef MF_HOST_EMU

__global__ void __launch_bounds__(RC_THREADS) k_rc_raster(RcParams p, const RcBox* __restrict__ boxes,
                                                           const RcGeom* __restrict__ geom,
                                                           const int4* __restrict__ pose_box,
                                                           float* __restrict__ depth,
                                                           uint8_t* __restrict__ mask,
                                                           int32_t* __restrict__ count) {
  __shared__ RcGeom s_geom[RC_THREADS];
  __shared__ RcBox s_box[RC_THREADS];
  __shared__ int s_n;
  const int tiles_x = (p.W + RC_TILE - 1) / RC_TILE;
  const int tx0 = (blockIdx.x % tiles_x) * RC_TILE, ty0 = (blockIdx.x / tiles_x) * RC_TILE;
  const int col = tx0 + (threadIdx.x % RC_TILE), row = ty0 + (threadIdx.x / RC_TILE);
  const bool on_image = col < p.W && row < p.H;
  const int tx1 = tx0 + RC_TILE - 1, ty1 = ty0 + RC_TILE - 1;
  for (int n = blockIdx.y; n < p.N; n += gridDim.y) {
    const int4 pb = pose_box[n];
    bool hit = false;
    float zmin = 0.0f;
    int lo, hi;
    if (pb.x <= tx1 && pb.z >= tx0 && pb.y <= ty1 && pb.w >= ty0 && rc_pose_mesh(p, n, lo, hi)) {
      const RcBox* bn = boxes + (size_t)n * p.F;
      const RcGeom* gn = geom + (size_t)n * p.F;
      for (int base = lo; base < hi; base += RC_THREADS) {
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        const int k = base + threadIdx.x;
        if (k < hi) {
          const RcBox b = bn[k];
          if (b.x0 <= tx1 && b.x1 >= tx0 && b.y0 <= ty1 && b.y1 >= ty0) {
            const int slot = atomicAdd(&s_n, 1);      // slot order is free: union and min commute
            s_box[slot] = b;
            s_geom[slot] = gn[k];
          }
        }
        __syncthreads();
        const int m = s_n;
        if (on_image)
          for (int q = 0; q < m; ++q) {
            const RcBox& b = s_box[q];
            if (col >= b.x0 && col <= b.x1 && row >= b.y0 && row <= b.y1)
              rc_cover(s_geom[q], col, row, hit, zmin);
          }
        __syncthreads();
      }
    }
    if (on_image) {
      const size_t o = ((size_t)n * p.H + row) * p.W + col;
      depth[o] = hit ? zmin : __int_as_float(0x7fc00000);
      mask[o] = hit ? 1 : 0;
    }
    const int c = __syncthreads_count(hit);
    if (threadIdx.x == 0 && c > 0) atomicAdd(count + n, c);
  }
}

// ------------------------------------------------------------------------------------------
// One scene of N <= 64 posed objects rendered together (mf_render_scene).  k_rc_init and
// k_rc_setup build the same records as mf_render_cad; k_rs_zero clears occluded [N,N].
// k_rs_raster  one CTA per 16x16 tile, a thread per pixel.  The objects are taken in input order;
//              one whose box misses the tile is skipped.  Each object's faces stream through
//              shared memory as in k_rc_raster, so rc_cover gives the pixel exactly the coverage
//              and depth that object has rendered alone.  The pixel keeps a 64-bit cover mask,
//              the best depth and the best object; only a strict < replaces the best, so an exact
//              tie goes to the lower index (GL_LESS with the objects drawn in input order).
//              __syncthreads_count adds each object's covered pixels to whole[n] (= mf_render_cad's
//              count).  For a pixel whose visible object is j, every other covering object i adds
//              1 to the tile's occ[i][j] in shared memory; the non-zero entries go to
//              occluded [N,N] with integer atomics.
// Every output is a min, a union or an integer sum, so every output is bitwise identical between
// runs.
// ------------------------------------------------------------------------------------------
__global__ void k_rs_zero(int n, int32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = 0;
}

__global__ void __launch_bounds__(RC_THREADS) k_rs_raster(RcParams p, const RcBox* __restrict__ boxes,
                                                           const RcGeom* __restrict__ geom,
                                                           const int4* __restrict__ pose_box,
                                                           const int32_t* __restrict__ instance_ids,
                                                           float* __restrict__ depth,
                                                           int32_t* __restrict__ ins,
                                                           int32_t* __restrict__ whole,
                                                           int32_t* __restrict__ occluded) {
  __shared__ RcGeom s_geom[RC_THREADS];
  __shared__ RcBox s_box[RC_THREADS];
  __shared__ int s_occ[MF_RENDER_SCENE_MAX_OBJECTS * MF_RENDER_SCENE_MAX_OBJECTS];
  __shared__ int s_n;
  const int tiles_x = (p.W + RC_TILE - 1) / RC_TILE;
  const int tx0 = (blockIdx.x % tiles_x) * RC_TILE, ty0 = (blockIdx.x / tiles_x) * RC_TILE;
  const int col = tx0 + (threadIdx.x % RC_TILE), row = ty0 + (threadIdx.x / RC_TILE);
  const bool on_image = col < p.W && row < p.H;
  const int tx1 = tx0 + RC_TILE - 1, ty1 = ty0 + RC_TILE - 1;
  const int NN = p.N * p.N;
  for (int i = threadIdx.x; i < NN; i += RC_THREADS) s_occ[i] = 0;
  unsigned long long cover = 0ull;
  float best = 0.0f;
  int best_n = -1;
  for (int n = 0; n < p.N; ++n) {
    const int4 pb = pose_box[n];
    int lo, hi;
    if (!(pb.x <= tx1 && pb.z >= tx0 && pb.y <= ty1 && pb.w >= ty0) || !rc_pose_mesh(p, n, lo, hi))
      continue;                                      // uniform over the CTA
    bool hit = false;
    float zmin = 0.0f;
    const RcBox* bn = boxes + (size_t)n * p.F;
    const RcGeom* gn = geom + (size_t)n * p.F;
    for (int base = lo; base < hi; base += RC_THREADS) {
      if (threadIdx.x == 0) s_n = 0;
      __syncthreads();
      const int k = base + threadIdx.x;
      if (k < hi) {
        const RcBox b = bn[k];
        if (b.x0 <= tx1 && b.x1 >= tx0 && b.y0 <= ty1 && b.y1 >= ty0) {
          const int slot = atomicAdd(&s_n, 1);        // slot order is free: union and min commute
          s_box[slot] = b;
          s_geom[slot] = gn[k];
        }
      }
      __syncthreads();
      const int m = s_n;
      if (on_image)
        for (int q = 0; q < m; ++q) {
          const RcBox& b = s_box[q];
          if (col >= b.x0 && col <= b.x1 && row >= b.y0 && row <= b.y1)
            rc_cover(s_geom[q], col, row, hit, zmin);
        }
      __syncthreads();
    }
    if (hit) {
      cover |= 1ull << n;
      if (best_n < 0 || zmin < best) {
        best = zmin;
        best_n = n;
      }
    }
    const int c = __syncthreads_count(hit);
    if (threadIdx.x == 0 && c > 0) atomicAdd(whole + n, c);
  }
  if (on_image) {
    const size_t o = (size_t)row * p.W + col;
    depth[o] = best_n >= 0 ? best : __int_as_float(0x7fc00000);
    ins[o] = best_n >= 0 ? instance_ids[best_n] : -1;
  }
  __syncthreads();                                   // s_occ cleared (also when no object ran)
  if (best_n >= 0) {
    unsigned long long rest = cover & ~(1ull << best_n);
    while (rest) {
      const int i = __ffsll((long long)rest) - 1;
      rest &= rest - 1;
      atomicAdd(&s_occ[i * p.N + best_n], 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NN; i += RC_THREADS)
    if (s_occ[i]) atomicAdd(occluded + i, s_occ[i]);
}

#endif  // !MF_HOST_EMU

}  // namespace mf

#ifndef MF_HOST_EMU
using namespace mf;

static size_t rc_align(size_t b) { return (b + 255) & ~(size_t)255; }

extern "C" size_t mf_render_cad_workspace_bytes(int N, int F, int H, int W) {
  if (N <= 0 || F < 0 || H <= 0 || W <= 0) return 0;
  const size_t rec = (size_t)N * F;
  return rc_align(rec * sizeof(RcBox)) + rc_align(rec * sizeof(RcGeom)) + rc_align((size_t)N * sizeof(int4));
}

extern "C" int mf_render_cad(const double* vertices, int V, const int32_t* faces, int F,
                             const int64_t* offsets, int S, const int32_t* mesh,
                             const double* Ts_cad2cam, int N, double f, int height, int width,
                             float* depth, uint8_t* mask, int32_t* count, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  if (height <= 0 || width <= 0 || (long long)height * width >= (1LL << 30)) return MF_E_BADARG;
  if (N < 0 || F < 0 || V < 0 || S < 1 || S > MF_RENDER_CAD_MAX_MESHES || !offsets)
    return MF_E_BADARG;
  if (!(f > 0.0) || !isfinite(f)) return MF_E_BADARG;
  if (offsets[0] != 0 || offsets[S] != F) return MF_E_BADARG;
  int f_max = 0;
  for (int s = 0; s < S; ++s) {
    if (offsets[s + 1] < offsets[s]) return MF_E_BADARG;
    if (offsets[s + 1] - offsets[s] > f_max) f_max = (int)(offsets[s + 1] - offsets[s]);
  }
  if (F > 0 && (!vertices || !faces || V == 0)) return MF_E_BADARG;
  if (N == 0) return MF_OK;
  if (!mesh || !Ts_cad2cam || !depth || !mask || !count || !workspace) return MF_E_BADARG;
  if (workspace_bytes < mf_render_cad_workspace_bytes(N, F, height, width)) return MF_E_WORKSPACE;
  if ((long long)N * f_max > (long long)RC_THREADS * 0x7fffffffLL) return MF_E_UNSUPPORTED;
  RcParams p;
  p.v = vertices; p.faces = faces; p.mesh = mesh; p.T = Ts_cad2cam;
  p.V = V; p.F = F; p.N = N; p.S = S; p.H = height; p.W = width; p.f_max = f_max; p.f = f;
  for (int s = 0; s <= S; ++s) p.off[s] = (int)offsets[s];
  const size_t rec = (size_t)N * F;
  char* ws = (char*)workspace;
  RcBox* boxes = (RcBox*)ws;
  RcGeom* geom = (RcGeom*)(ws + rc_align(rec * sizeof(RcBox)));
  int4* pose_box = (int4*)(ws + rc_align(rec * sizeof(RcBox)) + rc_align(rec * sizeof(RcGeom)));
  cudaStream_t st = (cudaStream_t)stream_;
  k_rc_init<<<div_up(N, 128), 128, 0, st>>>(N, pose_box, count);
  MF_LAUNCH_CHECK();
  if (f_max > 0) {
    k_rc_setup<<<div_up((long long)N * f_max, RC_THREADS), RC_THREADS, 0, st>>>(p, boxes, geom, pose_box);
    MF_LAUNCH_CHECK();
  }
  const long long tiles = (long long)div_up(width, RC_TILE) * div_up(height, RC_TILE);
  k_rc_raster<<<dim3((unsigned)tiles, (unsigned)(N < 65535 ? N : 65535)), RC_THREADS, 0, st>>>(
      p, boxes, geom, pose_box, depth, mask, count);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_render_scene(const double* vertices, int V, const int32_t* faces, int F,
                               const int64_t* offsets, int S, const int32_t* mesh,
                               const double* Ts_cad2cam, const int32_t* instance_ids, int N,
                               double f, int height, int width, float* depth, int32_t* ins,
                               int32_t* whole, int32_t* occluded, void* workspace,
                               size_t workspace_bytes, void* stream_) {
  if (height <= 0 || width <= 0 || (long long)height * width >= (1LL << 30)) return MF_E_BADARG;
  if (N < 0 || F < 0 || V < 0 || S < 1 || S > MF_RENDER_CAD_MAX_MESHES || !offsets)
    return MF_E_BADARG;
  if (N > MF_RENDER_SCENE_MAX_OBJECTS) return MF_E_UNSUPPORTED;
  if (!(f > 0.0) || !isfinite(f)) return MF_E_BADARG;
  if (offsets[0] != 0 || offsets[S] != F) return MF_E_BADARG;
  int f_max = 0;
  for (int s = 0; s < S; ++s) {
    if (offsets[s + 1] < offsets[s]) return MF_E_BADARG;
    if (offsets[s + 1] - offsets[s] > f_max) f_max = (int)(offsets[s + 1] - offsets[s]);
  }
  if (F > 0 && (!vertices || !faces || V == 0)) return MF_E_BADARG;
  if (!depth || !ins) return MF_E_BADARG;
  if (N > 0) {
    if (!mesh || !Ts_cad2cam || !instance_ids || !whole || !occluded || !workspace)
      return MF_E_BADARG;
    if (workspace_bytes < mf_render_cad_workspace_bytes(N, F, height, width)) return MF_E_WORKSPACE;
  }
  RcParams p;
  p.v = vertices; p.faces = faces; p.mesh = mesh; p.T = Ts_cad2cam;
  p.V = V; p.F = F; p.N = N; p.S = S; p.H = height; p.W = width; p.f_max = f_max; p.f = f;
  for (int s = 0; s <= S; ++s) p.off[s] = (int)offsets[s];
  const size_t rec = (size_t)N * F;
  char* ws = (char*)workspace;
  RcBox* boxes = (RcBox*)ws;
  RcGeom* geom = (RcGeom*)(ws + rc_align(rec * sizeof(RcBox)));
  int4* pose_box = (int4*)(ws + rc_align(rec * sizeof(RcBox)) + rc_align(rec * sizeof(RcGeom)));
  cudaStream_t st = (cudaStream_t)stream_;
  if (N > 0) {
    k_rc_init<<<div_up(N, 128), 128, 0, st>>>(N, pose_box, whole);
    MF_LAUNCH_CHECK();
    k_rs_zero<<<div_up(N * N, 256), 256, 0, st>>>(N * N, occluded);
    MF_LAUNCH_CHECK();
    if (f_max > 0) {
      k_rc_setup<<<div_up((long long)N * f_max, RC_THREADS), RC_THREADS, 0, st>>>(p, boxes, geom,
                                                                                 pose_box);
      MF_LAUNCH_CHECK();
    }
  }
  const long long tiles = (long long)div_up(width, RC_TILE) * div_up(height, RC_TILE);
  k_rs_raster<<<(unsigned)tiles, RC_THREADS, 0, st>>>(p, boxes, geom, pose_box, instance_ids,
                                                      depth, ins, whole, occluded);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
#endif  // !MF_HOST_EMU
