// Per-class model data from CAD meshes (datasets.MeshModels; what YCBVideoModels derives with
// binvox and trimesh, morefusion/datasets/ycb_video/models.py:56-115): the solid voxel grid and
// the signed distance of points to a mesh.  The rules are oracle/mesh_models.py's, bit for bit.
//
// mf_mesh_voxelize_solid, S meshes packed back to back, seven launches:
//   k_mm_bounds   one CTA per mesh: translate (the minimum of the referenced vertices), scale (the
//                 largest extent) and the step s = scale / D.  min and max are exact in any order.
//   k_mm_zero     clears the surface and parity bit planes ([S,D,D] columns of D bits).
//   k_mm_surface  one warp per face: the lanes walk the face's candidate voxels and atomicOr the
//                 surface bit of each voxel the separating-axis test accepts (mm_tri_box).
//   k_mm_parity   one warp per face: the lanes walk the face's candidate columns; where the +z
//                 ray of a column's centre crosses the face (mm_crossing), the parity bits of the
//                 n centres below the crossing (mm_count_below) are flipped with atomicXor.
//                 XOR commutes, so the bits do not depend on thread order, and no column needs a
//                 list of its crossings: nothing is capped.
//   k_mm_plane    one CTA per (mesh, x plane i): matrix[s,i] = surface | parity, and the plane's
//                 filled count.
//   k_mm_scan     one thread per mesh: exclusive scan of the plane counts, counts[s].
//   k_mm_points   one CTA per (mesh, plane): the filled centres of the plane in ascending (j, k)
//                 at points[s, plane offset + rank], and NaN in its share of the rows past
//                 counts[s].
// mf_mesh_signed_distance, two launches:
//   k_mm_sdf      a point per thread, CTAs of 128 points times C chunks of the faces.  The CTA's
//                 faces (those of the meshes its points belong to, cut into C equal chunks) go
//                 through shared memory in tiles of 128, each canonically ordered once; a thread
//                 keeps the smallest d^2 (first on a tie) and the crossing parity over the faces of
//                 its own mesh.  Per (chunk, point) it writes d^2, the face and the parity.
//   k_mm_sdf_fin  a thread per point: the chunks in order (strict <, so a tie keeps the lower
//                 face), parity XORed; sdf = +-sqrt(d^2).
// Everything is a min, a max, an OR, an XOR, an integer sum or an ordered scan, so every output is
// bitwise identical between runs and does not depend on which meshes share a call.  Built with
// -fmad=false; tests/emu/mesh_models_emu.cpp runs the per-face and per-pair code on the host.
#include <math.h>

#ifdef MF_HOST_EMU
#include "mapping_emu_stubs.h"
#include "mesh_models_emu_stubs.h"
#include "../../include/morefusion_b200.h"
#else
#include "common.cuh"
#endif

namespace mf {

constexpr int MM_SDF_THREADS = 128;           // points per CTA and faces per shared tile
constexpr int MM_MAX_CHUNKS = 64;
constexpr int MM_WARPS = 8;                   // warps per CTA of the per-face kernels

struct MmMeshes {
  const double* v;
  const int32_t* faces;
  int V, F, S;
  int off[MF_MESH_MODELS_MAX_MESHES + 1];
};

struct MmTri {
  double a[3], b[3], c[3];                    // vertices in canonical order (indices sorted)
};

// the mesh of face f (offsets are non-decreasing; empty meshes are skipped)
__device__ __forceinline__ int mm_mesh_of_face(const MmMeshes& m, int f) {
  int s = 0;
  while (s + 1 < m.S && m.off[s + 1] <= f) ++s;
  return s;
}

__device__ __forceinline__ void mm_load_tri(const MmMeshes& m, int f, MmTri& t) {
  int i0 = m.faces[3 * (size_t)f], i1 = m.faces[3 * (size_t)f + 1], i2 = m.faces[3 * (size_t)f + 2];
  int x;
  if (i1 < i0) { x = i0; i0 = i1; i1 = x; }
  if (i2 < i1) { x = i1; i1 = i2; i2 = x; }
  if (i1 < i0) { x = i0; i0 = i1; i1 = x; }
  for (int q = 0; q < 3; ++q) {
    t.a[q] = m.v[3 * (size_t)i0 + q];
    t.b[q] = m.v[3 * (size_t)i1 + q];
    t.c[q] = m.v[3 * (size_t)i2 + q];
  }
}

// ------------------------------------------------------------------------------------------------
// separating axes (Akenine-Moller): does the face overlap the closed box of centre c, half-size h?
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool mm_axis_sep(double p0, double p1, double p2, double rad) {
  const double lo = fmin(fmin(p0, p1), p2), hi = fmax(fmax(p0, p1), p2);
  return lo > rad || hi < -rad;
}

__device__ __forceinline__ bool mm_tri_box(const MmTri& t, const double c[3], double h) {
  double v0[3], v1[3], v2[3];
  for (int q = 0; q < 3; ++q) {
    v0[q] = t.a[q] - c[q];
    v1[q] = t.b[q] - c[q];
    v2[q] = t.c[q] - c[q];
  }
  double e[3][3];
  for (int q = 0; q < 3; ++q) {
    e[0][q] = v1[q] - v0[q];
    e[1][q] = v2[q] - v1[q];
    e[2][q] = v0[q] - v2[q];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double ex = e[k][0], ey = e[k][1], ez = e[k][2];
    const double fx = fabs(ex), fy = fabs(ey), fz = fabs(ez);
    if (mm_axis_sep(ez * v0[1] - ey * v0[2], ez * v1[1] - ey * v1[2], ez * v2[1] - ey * v2[2],
                    (fz + fy) * h))
      return false;
    if (mm_axis_sep(ex * v0[2] - ez * v0[0], ex * v1[2] - ez * v1[0], ex * v2[2] - ez * v2[0],
                    (fx + fz) * h))
      return false;
    if (mm_axis_sep(ey * v0[0] - ex * v0[1], ey * v1[0] - ex * v1[1], ey * v2[0] - ex * v2[1],
                    (fy + fx) * h))
      return false;
  }
  for (int q = 0; q < 3; ++q)
    if (mm_axis_sep(v0[q], v1[q], v2[q], h)) return false;
  const double n0 = e[0][1] * e[1][2] - e[0][2] * e[1][1];
  const double n1 = e[0][2] * e[1][0] - e[0][0] * e[1][2];
  const double n2 = e[0][0] * e[1][1] - e[0][1] * e[1][0];
  const double n[3] = {n0, n1, n2};
  double vmin[3], vmax[3];
  for (int q = 0; q < 3; ++q) {
    if (n[q] > 0) { vmin[q] = -h - v0[q]; vmax[q] = h - v0[q]; }
    else { vmin[q] = h - v0[q]; vmax[q] = -h - v0[q]; }
  }
  const double dmin = (n0 * vmin[0] + n1 * vmin[1]) + n2 * vmin[2];
  const double dmax = (n0 * vmax[0] + n1 * vmax[1]) + n2 * vmax[2];
  return !(dmin > 0) && dmax >= 0;
}

// ------------------------------------------------------------------------------------------------
// +z ray parity: does the vertical line through (px, py) cross the face, and at which z?
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double mm_edge(double ux, double uy, double vx, double vy, double px,
                                          double py) {
  return (vx - ux) * (py - uy) - (vy - uy) * (px - ux);
}

__device__ __forceinline__ bool mm_top_left(double dx, double dy) {
  return dy < 0 || (dy == 0 && dx < 0);
}

__device__ __forceinline__ bool mm_side(double w, double dx, double dy) {
  return w > 0 || (w == 0 && mm_top_left(dx, dy));
}

__device__ __forceinline__ bool mm_crossing(const MmTri& t, double px, double py, double& z) {
  const double ax = t.a[0], ay = t.a[1], bx = t.b[0], by = t.b[1], cx = t.c[0], cy = t.c[1];
  const double area2 = mm_edge(ax, ay, bx, by, cx, cy);
  if (area2 == 0) return false;
  const double sg = area2 < 0 ? -1.0 : 1.0;
  const double w0 = sg * mm_edge(bx, by, cx, cy, px, py);
  const double w1 = sg * -mm_edge(ax, ay, cx, cy, px, py);
  const double w2 = sg * mm_edge(ax, ay, bx, by, px, py);
  if (!mm_side(w0, sg * (cx - bx), sg * (cy - by))) return false;
  if (!mm_side(w1, sg * -(cx - ax), sg * -(cy - ay))) return false;
  if (!mm_side(w2, sg * (bx - ax), sg * (by - ay))) return false;
  z = ((w0 * t.a[2] + w1 * t.b[2]) + w2 * t.c[2]) / ((w0 + w1) + w2);
  return true;
}

// #{k in [0, D) : t + (k + 0.5) s < z}; the centres are non-decreasing in k
__device__ __forceinline__ int mm_count_below(double t, double s, int D, double z) {
  double g = floor((z - t) / s);
  g = fmin(fmax(g, 0.0), (double)D);
  int n = (int)g;
  while (n > 0 && !(t + ((double)(n - 1) + 0.5) * s < z)) --n;
  while (n < D && t + ((double)n + 0.5) * s < z) ++n;
  return n;
}

// the candidate index range of an extent [lo, hi] along one axis: floor((x - t) / s - shift) -+ 1
__device__ __forceinline__ void mm_range(double lo, double hi, double t, double s, int D,
                                         double shift, int& i0, int& i1) {
  const double a = floor((lo - t) / s - shift) - 1.0;
  const double b = floor((hi - t) / s - shift) + 1.0;
  i0 = (int)fmin(fmax(a, 0.0), (double)(D - 1));
  i1 = (int)fmin(fmax(b, 0.0), (double)(D - 1));
}

__device__ __forceinline__ double mm_centre(double t, double s, int i) {
  return t + ((double)i + 0.5) * s;
}

// the words of one column's bits: [S][D][D][W]
__device__ __forceinline__ size_t mm_col(int s, int i, int j, int D, int W) {
  return (((size_t)s * D + i) * D + j) * W;
}

// Surface bits of face f: candidate voxels lane, lane + nlanes, ...
__device__ __forceinline__ void mm_surface_face(const MmMeshes& m, int f, int D, int W,
                                                const double* translate, const double* pitch,
                                                uint32_t* bits, int lane, int nlanes) {
  const int s = mm_mesh_of_face(m, f);
  const double st = pitch[s];
  if (!(st > 0)) return;
  const double* t = translate + 3 * s;
  MmTri tri;
  mm_load_tri(m, f, tri);
  int lo[3], hi[3];
  for (int q = 0; q < 3; ++q)
    mm_range(fmin(fmin(tri.a[q], tri.b[q]), tri.c[q]), fmax(fmax(tri.a[q], tri.b[q]), tri.c[q]),
             t[q], st, D, 0.0, lo[q], hi[q]);
  const int ni = hi[0] - lo[0] + 1, nj = hi[1] - lo[1] + 1, nk = hi[2] - lo[2] + 1;
  const long long n = (long long)ni * nj * nk;
  const double h = 0.5 * st;
  for (long long r = lane; r < n; r += nlanes) {
    const int k = lo[2] + (int)(r % nk);
    const int j = lo[1] + (int)((r / nk) % nj);
    const int i = lo[0] + (int)(r / ((long long)nk * nj));
    const double c[3] = {mm_centre(t[0], st, i), mm_centre(t[1], st, j), mm_centre(t[2], st, k)};
    if (mm_tri_box(tri, c, h)) atomicOr(bits + mm_col(s, i, j, D, W) + (k >> 5), 1u << (k & 31));
  }
}

// Parity bits of face f: candidate columns lane, lane + nlanes, ...
__device__ __forceinline__ void mm_parity_face(const MmMeshes& m, int f, int D, int W,
                                               const double* translate, const double* pitch,
                                               uint32_t* bits, int lane, int nlanes) {
  const int s = mm_mesh_of_face(m, f);
  const double st = pitch[s];
  if (!(st > 0)) return;
  const double* t = translate + 3 * s;
  MmTri tri;
  mm_load_tri(m, f, tri);
  int lo[2], hi[2];
  for (int q = 0; q < 2; ++q)
    mm_range(fmin(fmin(tri.a[q], tri.b[q]), tri.c[q]), fmax(fmax(tri.a[q], tri.b[q]), tri.c[q]),
             t[q], st, D, 0.5, lo[q], hi[q]);
  const int ni = hi[0] - lo[0] + 1, nj = hi[1] - lo[1] + 1;
  for (int r = lane; r < ni * nj; r += nlanes) {
    const int i = lo[0] + r / nj, j = lo[1] + r % nj;
    double z;
    if (!mm_crossing(tri, mm_centre(t[0], st, i), mm_centre(t[1], st, j), z)) continue;
    const int nb = mm_count_below(t[2], st, D, z);
    uint32_t* col = bits + mm_col(s, i, j, D, W);
    for (int w = 0; w * 32 < nb; ++w) {
      const int left = nb - w * 32;
      atomicXor(col + w, left >= 32 ? 0xffffffffu : ((1u << left) - 1u));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// closest point on a face (Ericson, Real-Time Collision Detection 5.1.5)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double mm_dot(double ux, double uy, double uz, double vx, double vy,
                                         double vz) {
  return (ux * vx + uy * vy) + uz * vz;
}

__device__ __forceinline__ double mm_seg_d2(const double p[3], const double u[3], const double v[3]) {
  const double dx = v[0] - u[0], dy = v[1] - u[1], dz = v[2] - u[2];
  const double dd = mm_dot(dx, dy, dz, dx, dy, dz);
  double tt = dd > 0 ? mm_dot(p[0] - u[0], p[1] - u[1], p[2] - u[2], dx, dy, dz) / dd : 0.0;
  tt = fmin(fmax(tt, 0.0), 1.0);
  const double rx = p[0] - (u[0] + tt * dx), ry = p[1] - (u[1] + tt * dy),
               rz = p[2] - (u[2] + tt * dz);
  return mm_dot(rx, ry, rz, rx, ry, rz);
}

__device__ __forceinline__ double mm_closest_d2(const MmTri& t, const double p[3]) {
  const double* a = t.a;
  const double* b = t.b;
  const double* c = t.c;
  const double abx = b[0] - a[0], aby = b[1] - a[1], abz = b[2] - a[2];
  const double acx = c[0] - a[0], acy = c[1] - a[1], acz = c[2] - a[2];
  const double n0 = aby * acz - abz * acy, n1 = abz * acx - abx * acz, n2 = abx * acy - aby * acx;
  if (n0 == 0 && n1 == 0 && n2 == 0) {
    double d = mm_seg_d2(p, a, b);
    const double d_bc = mm_seg_d2(p, b, c);
    if (d_bc < d) d = d_bc;
    const double d_ca = mm_seg_d2(p, c, a);
    if (d_ca < d) d = d_ca;
    return d;
  }
  double q0, q1, q2;
  const double d1 = mm_dot(abx, aby, abz, p[0] - a[0], p[1] - a[1], p[2] - a[2]);
  const double d2 = mm_dot(acx, acy, acz, p[0] - a[0], p[1] - a[1], p[2] - a[2]);
  const double bpx = p[0] - b[0], bpy = p[1] - b[1], bpz = p[2] - b[2];
  const double d3 = mm_dot(abx, aby, abz, bpx, bpy, bpz);
  const double d4 = mm_dot(acx, acy, acz, bpx, bpy, bpz);
  const double vc = d1 * d4 - d3 * d2;
  const double cpx = p[0] - c[0], cpy = p[1] - c[1], cpz = p[2] - c[2];
  const double d5 = mm_dot(abx, aby, abz, cpx, cpy, cpz);
  const double d6 = mm_dot(acx, acy, acz, cpx, cpy, cpz);
  const double vb = d5 * d2 - d1 * d6;
  const double va = d3 * d6 - d5 * d4;
  if (d1 <= 0 && d2 <= 0) {
    q0 = a[0]; q1 = a[1]; q2 = a[2];
  } else if (d3 >= 0 && d4 <= d3) {
    q0 = b[0]; q1 = b[1]; q2 = b[2];
  } else if (vc <= 0 && d1 >= 0 && d3 <= 0) {
    const double v = d1 / (d1 - d3);
    q0 = a[0] + v * abx; q1 = a[1] + v * aby; q2 = a[2] + v * abz;
  } else if (d6 >= 0 && d5 <= d6) {
    q0 = c[0]; q1 = c[1]; q2 = c[2];
  } else if (vb <= 0 && d2 >= 0 && d6 <= 0) {
    const double w = d2 / (d2 - d6);
    q0 = a[0] + w * acx; q1 = a[1] + w * acy; q2 = a[2] + w * acz;
  } else if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) {
    const double w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    q0 = b[0] + w * (c[0] - b[0]); q1 = b[1] + w * (c[1] - b[1]); q2 = b[2] + w * (c[2] - b[2]);
  } else {
    const double denom = 1.0 / ((va + vb) + vc);
    const double v = vb * denom, w = vc * denom;
    q0 = (a[0] + abx * v) + acx * w;
    q1 = (a[1] + aby * v) + acy * w;
    q2 = (a[2] + abz * v) + acz * w;
  }
  const double rx = p[0] - q0, ry = p[1] - q1, rz = p[2] - q2;
  return mm_dot(rx, ry, rz, rx, ry, rz);
}

// one (point, face) pair: lower (best, arg) on a strictly smaller d^2, flip odd on a crossing
__device__ __forceinline__ void mm_sdf_pair(const MmTri& t, int f, const double p[3], double& best,
                                            int& arg, int& odd) {
  const double d2 = mm_closest_d2(t, p);
  if (d2 < best) {
    best = d2;
    arg = f;
  }
  double z;
  if (mm_crossing(t, p[0], p[1], z) && z > p[2]) odd ^= 1;
}

__device__ __forceinline__ double mm_signed(double best, int odd) {
  const double d = sqrt(best);
  return odd ? d : -d;
}

__device__ __forceinline__ void mm_chunk(int lo, int hi, int C, int c, int& c0, int& c1) {
  const int len = (hi - lo + C - 1) / C;
  c0 = min(hi, lo + c * len);
  c1 = min(hi, c0 + len);
}

#ifndef MF_HOST_EMU

__global__ void __launch_bounds__(256) k_mm_bounds(MmMeshes m, int D, double* __restrict__ translate,
                                                   double* __restrict__ scale,
                                                   double* __restrict__ pitch) {
  __shared__ double s_lo[3][256], s_hi[3][256];
  const int s = blockIdx.x;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int r = m.off[s] * 3 + threadIdx.x; r < m.off[s + 1] * 3; r += blockDim.x) {
    const double* p = m.v + 3 * (size_t)m.faces[r];
    for (int q = 0; q < 3; ++q) {
      lo[q] = fmin(lo[q], p[q]);
      hi[q] = fmax(hi[q], p[q]);
    }
  }
  for (int q = 0; q < 3; ++q) {
    s_lo[q][threadIdx.x] = lo[q];
    s_hi[q][threadIdx.x] = hi[q];
  }
  __syncthreads();
  for (int w = blockDim.x / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
      for (int q = 0; q < 3; ++q) {
        s_lo[q][threadIdx.x] = fmin(s_lo[q][threadIdx.x], s_lo[q][threadIdx.x + w]);
        s_hi[q][threadIdx.x] = fmax(s_hi[q][threadIdx.x], s_hi[q][threadIdx.x + w]);
      }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const bool any = m.off[s + 1] > m.off[s];
    double sc = 0.0;
    for (int q = 0; q < 3; ++q) {
      translate[3 * s + q] = any ? s_lo[0 + q][0] : 0.0;
      const double ext = s_hi[q][0] - s_lo[q][0];
      sc = q == 0 ? ext : fmax(sc, ext);
    }
    if (!any || !isfinite(sc)) sc = 0.0;
    scale[s] = sc;
    pitch[s] = sc / D;
  }
}

__global__ void k_mm_zero(size_t n, uint32_t* __restrict__ a) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    a[i] = 0u;
}

__global__ void __launch_bounds__(MM_WARPS * 32) k_mm_surface(MmMeshes m, int D, int W,
                                                              const double* __restrict__ translate,
                                                              const double* __restrict__ pitch,
                                                              uint32_t* __restrict__ bits) {
  const int f = blockIdx.x * MM_WARPS + threadIdx.x / 32;
  if (f >= m.F) return;
  mm_surface_face(m, f, D, W, translate, pitch, bits, threadIdx.x & 31, 32);
}

__global__ void __launch_bounds__(MM_WARPS * 32) k_mm_parity(MmMeshes m, int D, int W,
                                                             const double* __restrict__ translate,
                                                             const double* __restrict__ pitch,
                                                             uint32_t* __restrict__ bits) {
  const int f = blockIdx.x * MM_WARPS + threadIdx.x / 32;
  if (f >= m.F) return;
  mm_parity_face(m, f, D, W, translate, pitch, bits, threadIdx.x & 31, 32);
}

// the filled bits of a column word: surface | parity, only voxels k < D
__device__ __forceinline__ uint32_t mm_filled(const uint32_t* surf, const uint32_t* par, size_t o,
                                              int w, int D) {
  uint32_t b = surf[o + w] | par[o + w];
  const int left = D - w * 32;
  if (left < 32) b &= (1u << left) - 1u;
  return b;
}

__global__ void __launch_bounds__(128) k_mm_plane(int D, int W, const uint32_t* __restrict__ surf,
                                                  const uint32_t* __restrict__ par,
                                                  uint8_t* __restrict__ matrix,
                                                  int32_t* __restrict__ plane_count) {
  const int s = blockIdx.x / D, i = blockIdx.x % D;
  int cnt = 0;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const size_t o = mm_col(s, i, j, D, W);
    uint8_t* row = matrix + (((size_t)s * D + i) * D + j) * D;
    for (int w = 0; w < W; ++w) {
      const uint32_t b = mm_filled(surf, par, o, w, D);
      cnt += __popc(b);
      for (int k = w * 32; k < min(D, w * 32 + 32); ++k) row[k] = (b >> (k - w * 32)) & 1u;
    }
  }
  __shared__ int s_sum;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  if (cnt) atomicAdd(&s_sum, cnt);
  __syncthreads();
  if (threadIdx.x == 0) plane_count[blockIdx.x] = s_sum;
}

__global__ void k_mm_scan(int S, int D, const int32_t* __restrict__ plane_count,
                          int32_t* __restrict__ plane_off, int32_t* __restrict__ counts) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  int acc = 0;
  for (int i = 0; i < D; ++i) {
    plane_off[s * D + i] = acc;
    acc += plane_count[s * D + i];
  }
  counts[s] = acc;
}

__global__ void __launch_bounds__(128) k_mm_points(int D, int W, const uint32_t* __restrict__ surf,
                                                   const uint32_t* __restrict__ par,
                                                   const double* __restrict__ translate,
                                                   const double* __restrict__ pitch,
                                                   const int32_t* __restrict__ plane_off,
                                                   const int32_t* __restrict__ counts,
                                                   double* __restrict__ points) {
  __shared__ int s_cnt[MF_MESH_MODELS_MAX_DIM];
  const int s = blockIdx.x / D, i = blockIdx.x % D;
  const long long D3 = (long long)D * D * D;
  const int j = threadIdx.x;                      // blockDim.x == D rounded up to a warp
  const size_t o = j < D ? mm_col(s, i, j, D, W) : 0;
  int c = 0;
  if (j < D)
    for (int w = 0; w < W; ++w) c += __popc(mm_filled(surf, par, o, w, D));
  if (j < D) s_cnt[j] = c;
  __syncthreads();
  if (j < D) {
    int base = plane_off[blockIdx.x];
    for (int q = 0; q < j; ++q) base += s_cnt[q];
    const double st = pitch[s];
    const double* t = translate + 3 * s;
    double* out = points + (size_t)s * D3 * 3;
    const double x = mm_centre(t[0], st, i), y = mm_centre(t[1], st, j);
    for (int w = 0; w < W; ++w) {
      uint32_t b = mm_filled(surf, par, o, w, D);
      while (b) {
        const int k = w * 32 + __ffs(b) - 1;
        b &= b - 1;
        double* r = out + 3 * (size_t)base++;
        r[0] = x;
        r[1] = y;
        r[2] = mm_centre(t[2], st, k);
      }
    }
  }
  // this plane's share of the rows past counts[s]: [n + i D^2, n + (i + 1) D^2) within [n, D^3)
  const long long n = counts[s];
  const long long r0 = n + (long long)i * D * D, r1 = min(D3, r0 + (long long)D * D);
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (long long r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
    double* row = points + ((size_t)s * D3 + r) * 3;
    row[0] = nan;
    row[1] = nan;
    row[2] = nan;
  }
}

__global__ void __launch_bounds__(MM_SDF_THREADS) k_mm_sdf(MmMeshes m, const double* __restrict__ pts,
                                                           const int32_t* __restrict__ mesh, int P,
                                                           int C, double* __restrict__ part_d2,
                                                           int32_t* __restrict__ part_arg,
                                                           uint8_t* __restrict__ part_odd) {
  __shared__ MmTri s_tri[MM_SDF_THREADS];
  __shared__ int s_mlo, s_mhi;
  const int r = blockIdx.x * MM_SDF_THREADS + threadIdx.x;
  const int c = blockIdx.y;
  int ms = -1;
  double p[3] = {0.0, 0.0, 0.0};
  if (r < P) {
    ms = mesh[r];
    if (ms < 0 || ms >= m.S) ms = -1;
    for (int q = 0; q < 3; ++q) p[q] = pts[3 * (size_t)r + q];
  }
  if (threadIdx.x == 0) {
    s_mlo = 0x7fffffff;
    s_mhi = -1;
  }
  __syncthreads();
  if (ms >= 0) {
    atomicMin(&s_mlo, ms);
    atomicMax(&s_mhi, ms);
  }
  __syncthreads();
  double best = INFINITY;
  int arg = -1, odd = 0;
  if (s_mhi >= 0) {                               // uniform over the CTA
    int f0, f1;
    mm_chunk(m.off[s_mlo], m.off[s_mhi + 1], C, c, f0, f1);
    const int lo = ms >= 0 ? max(m.off[ms], f0) : 0, hi = ms >= 0 ? min(m.off[ms + 1], f1) : 0;
    for (int base = f0; base < f1; base += MM_SDF_THREADS) {
      const int f = base + threadIdx.x;
      if (f < f1) mm_load_tri(m, f, s_tri[threadIdx.x]);
      __syncthreads();
      const int q0 = max(lo, base), q1 = min(hi, min(f1, base + MM_SDF_THREADS));
      for (int q = q0; q < q1; ++q) mm_sdf_pair(s_tri[q - base], q, p, best, arg, odd);
      __syncthreads();
    }
  }
  if (r < P) {
    const size_t o = (size_t)c * P + r;
    part_d2[o] = best;
    part_arg[o] = arg;
    part_odd[o] = (uint8_t)odd;
  }
}

__global__ void k_mm_sdf_fin(int P, int C, const int32_t* __restrict__ mesh, int S,
                             const double* __restrict__ part_d2, const int32_t* __restrict__ part_arg,
                             const uint8_t* __restrict__ part_odd, double* __restrict__ sdf,
                             int32_t* __restrict__ face) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P) return;
  double best = INFINITY;
  int arg = -1, odd = 0;
  for (int c = 0; c < C; ++c) {
    const size_t o = (size_t)c * P + r;
    if (part_d2[o] < best) {
      best = part_d2[o];
      arg = part_arg[o];
    }
    odd ^= part_odd[o];
  }
  const int ms = mesh[r];
  const bool ok = ms >= 0 && ms < S && arg >= 0;
  sdf[r] = ok ? mm_signed(best, odd) : __longlong_as_double(0x7ff8000000000000LL);
  face[r] = ok ? arg : -1;
}

#endif  // !MF_HOST_EMU

}  // namespace mf

#ifndef MF_HOST_EMU
using namespace mf;

static size_t mm_align(size_t b) { return (b + 255) & ~(size_t)255; }

static int mm_meshes(const double* vertices, int V, const int32_t* faces, int F,
                     const int64_t* offsets, int S, MmMeshes& m, int& f_max) {
  if (V < 0 || F < 0 || S < 1 || S > MF_MESH_MODELS_MAX_MESHES || !offsets) return MF_E_BADARG;
  if (offsets[0] != 0 || offsets[S] != F) return MF_E_BADARG;
  f_max = 0;
  for (int s = 0; s < S; ++s) {
    if (offsets[s + 1] < offsets[s]) return MF_E_BADARG;
    if (offsets[s + 1] - offsets[s] > f_max) f_max = (int)(offsets[s + 1] - offsets[s]);
  }
  if (F > 0 && (!vertices || !faces || V == 0)) return MF_E_BADARG;
  m.v = vertices; m.faces = faces; m.V = V; m.F = F; m.S = S;
  for (int s = 0; s <= MF_MESH_MODELS_MAX_MESHES; ++s) m.off[s] = s <= S ? (int)offsets[s] : F;
  return MF_OK;
}

extern "C" size_t mf_mesh_voxelize_workspace_bytes(int S, int D) {
  if (S <= 0 || D <= 0) return 0;
  const size_t W = (size_t)(D + 31) / 32;
  const size_t words = (size_t)S * D * D * W;
  return 2 * mm_align(words * 4) + 2 * mm_align((size_t)S * D * 4);
}

extern "C" int mf_mesh_voxelize_solid(const double* vertices, int V, const int32_t* faces, int F,
                                      const int64_t* offsets, int S, int D, uint8_t* matrix,
                                      int32_t* counts, double* points, double* translate,
                                      double* scale, double* pitch, void* workspace,
                                      size_t workspace_bytes, void* stream_) {
  MmMeshes m;
  int f_max;
  const int rc = mm_meshes(vertices, V, faces, F, offsets, S, m, f_max);
  if (rc != MF_OK) return rc;
  if (D < 1 || D > MF_MESH_MODELS_MAX_DIM) return MF_E_BADARG;
  if (!matrix || !counts || !points || !translate || !scale || !pitch || !workspace)
    return MF_E_BADARG;
  if (workspace_bytes < mf_mesh_voxelize_workspace_bytes(S, D)) return MF_E_WORKSPACE;
  const int W = (D + 31) / 32;
  const size_t words = (size_t)S * D * D * W;
  char* ws = (char*)workspace;
  uint32_t* surf = (uint32_t*)ws;
  uint32_t* par = (uint32_t*)(ws + mm_align(words * 4));
  int32_t* plane_count = (int32_t*)(ws + 2 * mm_align(words * 4));
  int32_t* plane_off = (int32_t*)(ws + 2 * mm_align(words * 4) + mm_align((size_t)S * D * 4));
  cudaStream_t st = (cudaStream_t)stream_;
  k_mm_bounds<<<S, 256, 0, st>>>(m, D, translate, scale, pitch);
  MF_LAUNCH_CHECK();
  k_mm_zero<<<(unsigned)min((size_t)4096, (2 * words + 255) / 256 + 1), 256, 0, st>>>(
      (size_t)(par - surf) + words, surf);        // both bit planes (and the gap between them)
  MF_LAUNCH_CHECK();
  if (F > 0) {
    k_mm_surface<<<div_up(F, MM_WARPS), MM_WARPS * 32, 0, st>>>(m, D, W, translate, pitch, surf);
    MF_LAUNCH_CHECK();
    k_mm_parity<<<div_up(F, MM_WARPS), MM_WARPS * 32, 0, st>>>(m, D, W, translate, pitch, par);
    MF_LAUNCH_CHECK();
  }
  k_mm_plane<<<S * D, 128, 0, st>>>(D, W, surf, par, matrix, plane_count);
  MF_LAUNCH_CHECK();
  k_mm_scan<<<div_up(S, 64), 64, 0, st>>>(S, D, plane_count, plane_off, counts);
  MF_LAUNCH_CHECK();
  k_mm_points<<<S * D, (D + 31) / 32 * 32, 0, st>>>(D, W, surf, par, translate, pitch, plane_off,
                                                    counts, points);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

// face chunks per CTA of points: enough CTAs for about four per SM, at most one chunk per tile
static int mm_sdf_chunks(int P, int f_max) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess)
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long blocks = (P + MM_SDF_THREADS - 1) / MM_SDF_THREADS;
  long long C = blocks > 0 ? (4LL * sms + blocks - 1) / blocks : 1;
  const long long tiles = (f_max + MM_SDF_THREADS - 1) / MM_SDF_THREADS;
  if (C > tiles) C = tiles;
  if (C > MM_MAX_CHUNKS) C = MM_MAX_CHUNKS;
  return C < 1 ? 1 : (int)C;
}

extern "C" size_t mf_mesh_signed_distance_workspace_bytes(int P, int f_max) {
  if (P <= 0) return 0;
  const size_t C = (size_t)mm_sdf_chunks(P, f_max);
  return mm_align(C * P * 8) + mm_align(C * P * 4) + mm_align(C * P);
}

extern "C" int mf_mesh_signed_distance(const double* vertices, int V, const int32_t* faces, int F,
                                       const int64_t* offsets, int S, const double* points,
                                       const int32_t* mesh, int P, double* sdf, int32_t* face,
                                       void* workspace, size_t workspace_bytes, void* stream_) {
  MmMeshes m;
  int f_max;
  const int rc = mm_meshes(vertices, V, faces, F, offsets, S, m, f_max);
  if (rc != MF_OK) return rc;
  if (P < 0) return MF_E_BADARG;
  if (P == 0) return MF_OK;
  if (!points || !mesh || !sdf || !face || !workspace) return MF_E_BADARG;
  if (workspace_bytes < mf_mesh_signed_distance_workspace_bytes(P, f_max)) return MF_E_WORKSPACE;
  const int C = mm_sdf_chunks(P, f_max);
  char* ws = (char*)workspace;
  double* part_d2 = (double*)ws;
  int32_t* part_arg = (int32_t*)(ws + mm_align((size_t)C * P * 8));
  uint8_t* part_odd = (uint8_t*)(ws + mm_align((size_t)C * P * 8) + mm_align((size_t)C * P * 4));
  cudaStream_t st = (cudaStream_t)stream_;
  k_mm_sdf<<<dim3(div_up(P, MM_SDF_THREADS), C), MM_SDF_THREADS, 0, st>>>(m, points, mesh, P, C,
                                                                         part_d2, part_arg, part_odd);
  MF_LAUNCH_CHECK();
  k_mm_sdf_fin<<<div_up(P, 256), 256, 0, st>>>(P, C, mesh, S, part_d2, part_arg, part_odd, sdf, face);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
#endif  // !MF_HOST_EMU
