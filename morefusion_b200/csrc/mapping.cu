// Occupancy-grid producer (SURVEY.md 8f-3): the map behind
//   morefusion/contrib/multi_instance_octree_mapping.py:7-94   (OcTree per instance, get_target_grids)
// as a device-resident hashed log-odds voxel map.  The reference delegates to OctoMap (octomap-python,
// absent from the reference tree); the semantics kept here are OctoMap 1.9's, as restated and cited
// in oracle/octomap.py: 16-bit keys per axis, float32 log-odds with clamping, the Amanatides & Woo
// key ray of OcTreeBaseImpl::computeRayKeys in the library's float/double mix, "every cell updated
// at most once per scan, end points win over free cells" (OccupancyOcTreeBase::computeUpdate).
//
// GPU design.  A pruned octree is, for search(depth=0), a flat key -> log-odds map: ONE open-
// addressing hash table in HBM holds every instance's cells as 16-byte entries
// {key = instance:16 | kx:16 | ky:16 | kz:16, float log-odds, u32 scan stamp}: a probe is one
// 16-byte L2 access that brings the key, the value and the stamp together.  A scan is two launches,
// the three 32^3 grids of all targets are one launch:
//   k_map_scan_hits   one thread per pixel: end-point ("hit") update.
//   k_map_scan_free   one thread per pixel walks its ray (the DDA is sequential double arithmetic:
//                     tMax accumulates rounding exactly as the library's does).  The 32 lanes of a
//                     warp are 32 neighbouring pixels; at a 1 cm cell and <1.7 mm between rays they
//                     sit in the same one to five cells at every step, so the lanes of a step are
//                     grouped by key (__match_any_sync) and only one lane per distinct cell probes
//                     the table; a cell already stamped by this scan costs that one read
//                     (test-before-atomic), the first toucher applies the miss update.  No key
//                     buffer: the first version wrote every (ray, cell) key to HBM and applied them
//                     in a second kernel (profiles/r02_mapping_history.md: 39 M keys, 310 MB written
//                     and read back, 130 visits per distinct cell).
//   k_map_query_grids one thread per (target, voxel): looks the voxel centre up in every instance,
//                     in insertion order, and writes grid_target / grid_nontarget / grid_empty with
//                     the reference's overwrite rules (multi_instance_octree_mapping.py:85-92).
//   k_map_query_node_grids  the same work split for the refinement node's grid / grid_noentry
//                     pair, with the occupancy server's rules (OctomapServer.cpp:510-618);
//                     k_map_query_node_grids_world the same with camera-frame origins.
//   k_map_server_hits / k_map_scan_free<ServerScanParams> / k_map_server_centres  the server's
//                     scan of a moving camera's frame in the world frame (insertScan, :283-448);
//                     k_map_server_boxes the instance boxes that scan keeps (:404-437).
//   k_map_render_rays / k_map_render_write  the server's render of the map into the camera
//                     (:193-281): castRay per (even pixel, instance), a per-pixel z-buffer.
// A cell is updated by exactly one thread per scan, so results do not depend on thread order:
// bit-identical to the serial oracle.  -fmad=false: the double expressions must not contract.
#include <math.h>

#ifdef MF_HOST_EMU
// tests/emu/mapping_emu.cpp runs the kernels of this file serially on the host (one-lane "warps")
// against oracle/octomap.py in the CPU test suite; it supplies the CUDA spellings used below.
#include "mapping_emu_stubs.h"
#include "mapping_render_emu_stubs.h"
#else
#include "common.cuh"
#endif

namespace mf {

typedef unsigned long long u64;
static constexpr u64 MAP_EMPTY = ~0ull;
static constexpr int TREE_MAX_VAL = 32768;

struct __align__(16) MapCell {
  u64 key;          // MAP_EMPTY = free slot
  float lo;         // log-odds, 0 for a slot that has never been updated
  unsigned stamp;   // 2*scan (missed in scan) / 2*scan+1 (hit in scan), monotonic
};

struct MapTable {
  MapCell* cells;   // [cap]
  unsigned* cnt;    // [cap]   pending updateNodes() multiplicity (0 between calls)
  unsigned mask;    // cap - 1 (cap is a power of two)
  int* counters;    // [0] live entries  [1] table full (sticky; updates were dropped)
};

__device__ __forceinline__ unsigned map_hash(u64 k) {
  k *= 0x9E3779B97F4A7C15ull;
  k ^= k >> 29;
  k *= 0xBF58476D1CE4E5B9ull;
  return (unsigned)(k >> 32);
}

// one 16-byte L2 access (other SMs update cells during a scan: never through the incoherent L1)
__device__ __forceinline__ MapCell map_load(const MapCell* c) {
  const ulonglong2 v = __ldcg(reinterpret_cast<const ulonglong2*>(c));
  MapCell r;
  r.key = v.x;
  r.lo = __uint_as_float((unsigned)(v.y & 0xffffffffull));
  r.stamp = (unsigned)(v.y >> 32);
  return r;
}

// slot of `key`, inserting it when absent; -1 when the table is full (overflow flag raised).
// *seen = the cell as loaded (stamp 0 for a cell this call inserted or lost the race for: a stale
// stamp only costs a redundant atomicMax, never an update).
// Probe sequences are bounded (MAP_MAX_PROBES): a table that is (nearly) full reports overflow
// instead of walking millions of slots per thread.
static constexpr unsigned MAP_MAX_PROBES = 4096;
__device__ __forceinline__ int map_find_or_insert(const MapTable& t, u64 key, MapCell* seen) {
  unsigned s = map_hash(key) & t.mask;
  const unsigned limit = t.mask < MAP_MAX_PROBES ? t.mask : MAP_MAX_PROBES;
  for (unsigned n = 0; n <= limit; ++n) {
    const MapCell c = map_load(t.cells + s);
    if (c.key == key) { *seen = c; return (int)s; }
    if (c.key == MAP_EMPTY) {
      const u64 old = atomicCAS(&t.cells[s].key, MAP_EMPTY, key);
      if (old == MAP_EMPTY || old == key) {
        if (old == MAP_EMPTY) atomicAdd(t.counters, 1);
        seen->key = key; seen->lo = 0.f; seen->stamp = 0u;
        return (int)s;
      }
    }
    s = (s + 1) & t.mask;
  }
  t.counters[1] = 1;
  return -1;
}

__device__ __forceinline__ int map_find(const MapTable& t, u64 key, MapCell* seen) {
  unsigned s = map_hash(key) & t.mask;
  const unsigned limit = t.mask < MAP_MAX_PROBES ? t.mask : MAP_MAX_PROBES;
  for (unsigned n = 0; n <= limit; ++n) {
    const MapCell c = map_load(t.cells + s);
    if (c.key == key) { *seen = c; return (int)s; }
    if (c.key == MAP_EMPTY) return -1;
    s = (s + 1) & t.mask;
  }
  return -1;
}

__device__ __forceinline__ float map_clamped_add(float v, float upd, float lo_min, float lo_max) {
  v = __fadd_rn(v, upd);                      // OccupancyOcTreeBase::updateNodeLogOdds
  if (v < lo_min) v = lo_min;
  if (v > lo_max) v = lo_max;
  return v;
}

// the once-per-scan update of a cell: the thread whose atomicMax raises the stamp to `want` owns it
__device__ __forceinline__ void map_scan_update(const MapTable& t, int s, const MapCell& seen,
                                                unsigned want, float upd, float lo_min, float lo_max) {
  if (seen.stamp >= want) return;                                  // already done in this scan
  if (atomicMax(&t.cells[s].stamp, want) < want) {
    // nobody else writes lo in this launch; the value is from an earlier launch (or 0)
    const float v = __ldcg(&t.cells[s].lo);
    t.cells[s].lo = map_clamped_add(v, upd, lo_min, lo_max);
  }
}

// OcTreeBaseImpl::coordToKeyChecked for one axis: floor(coord / resolution) + 32768, -1 if outside
__device__ __forceinline__ int coord_to_key(double c, double res_factor) {
  const double f = floor(res_factor * c) + (double)TREE_MAX_VAL;     // exact: |floor| < 2^52
  return (f >= 0.0 && f < (double)(2 * TREE_MAX_VAL)) ? (int)f : -1;  // NaN / inf fail both tests
}

__device__ __forceinline__ u64 pack_key(int inst, int kx, int ky, int kz) {
  return ((u64)(unsigned)inst << 48) | ((u64)(unsigned)kx << 32) | ((u64)(unsigned)ky << 16) |
         (u64)(unsigned)kz;
}

struct ScanParams {
  const float* points;        // [n,3]
  const unsigned char* mask;  // [n] or null          (single-instance scan)
  const int* labels;          // [n] or null          (labelled frame: every instance in one scan)
  const int* lut;             // [lut_n] label - lut_lo -> dense instance index, -1 = not mapped
  const double* inst_res;     // [n_inst] resolution of each instance (labelled frame)
  int lut_lo, lut_n;
  int n;
  float ox, oy, oz;           // sensor origin (point3d: floats)
  double res;                 // single-instance scan
  int inst;
  unsigned scan;
  float hit, miss, lo_min, lo_max;
};

// The occupancy server's scan (OctomapServer::insertScan, ros/src/morefusion_ros/src/
// OctomapServer.cpp:283-448; oracle/octomap_server_multiview.py::insert_scan restates it rule by rule): an
// organised camera-frame cloud moved to the world frame, every second pixel of every second row,
// free rays in the background's key space only, end points as hits in their instance's key space.
struct ServerScanParams {
  const float* points;        // [n,3] camera frame, row-major H x W
  const int* labels;          // [n]
  const int* lut;             // [lut_n] label - lut_lo -> dense instance index, -1 = skipped
  const double* inst_res;     // [n_inst] resolution of each instance
  u64* csum;                  // [n_inst,4] this scan's centre sums (fixed point) and point counts
  unsigned* cfirst;           // [n_inst] ~(this scan's lowest listed pixel index); 0 = none
  int lut_lo, lut_n;
  int n, width;
  int bg;                     // dense index of the background
  int uncertain;              // label of uncertain pixels (-2 in the server)
  float m[12];                // rows 0-2 of sensorToWorld as an Eigen::Matrix4f
  float ox, oy, oz;           // sensor origin (point3d: floats)
  double max_range;           // < 0: no limit
  double res;                 // background resolution: the key space of every ray
  unsigned scan;
  float hit, miss, lo_min, lo_max;
};

// pcl::transformPointCloud with a Matrix4f (OctomapServer.cpp:111-119), PCL's generic path:
// ((m0 x + m1 y) + m2 z) + m3 per row in float, no contraction
__device__ __forceinline__ void xform_f32(const float* m, float x, float y, float z, float w[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    w[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4 * r], x), __fmul_rn(m[4 * r + 1], y)),
                               __fmul_rn(m[4 * r + 2], z)), m[4 * r + 3]);
}

// a kept pixel of the server's scan: its world point and its dense instance index (-1 for an
// uncertain pixel); false for odd rows / columns (:329-333), NaN points (:334-338) and labels that
// are neither listed nor uncertain (the server aborts the scan there, :302-304)
__device__ __forceinline__ bool server_point(const ServerScanParams& p, int i, float w[3], int* q) {
  w[0] = w[1] = w[2] = 0.f;
  *q = -1;
  if (i >= p.n) return false;
  const int row = i / p.width, col = i - row * p.width;
  if ((row | col) & 1) return false;
  xform_f32(p.m, p.points[3 * (size_t)i], p.points[3 * (size_t)i + 1], p.points[3 * (size_t)i + 2],
            w);
  if (isnan(w[0]) || isnan(w[1]) || isnan(w[2])) return false;
  const int lab = p.labels[i];
  if (lab == p.uncertain) return true;
  const int l = lab - p.lut_lo;
  *q = (l >= 0 && l < p.lut_n) ? p.lut[l] : -1;
  return *q >= 0;
}

// (point - origin): the float difference and its point3d::norm(), sqrt of the float norm_sq
__device__ __forceinline__ double point_diff_norm(const float w[3], float ox, float oy, float oz,
                                                  float d[3]) {
  d[0] = __fsub_rn(w[0], ox);
  d[1] = __fsub_rn(w[1], oy);
  d[2] = __fsub_rn(w[2], oz);
  const float nsq = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])),
                              __fmul_rn(d[2], d[2]));
  return sqrt((double)nsq);
}

__device__ __forceinline__ double server_ray(const ServerScanParams& p, const float w[3], float d[3]) {
  return point_diff_norm(w, p.ox, p.oy, p.oz, d);
}

// pcl::compute3DCentroid's sum in a fixed point of 2^-32 m: integer sums do not depend on the
// order of the atomics, so the centre is reproducible
__device__ __forceinline__ long long centre_fix(float v) {
  return llrint((double)v * 4294967296.0);                   // to nearest, ties to even
}

// a pixel's end point, its instance / resolution and the keys of both ends; false for masked,
// unmapped and NaN pixels.  end_free is the server's (below); never set here
__device__ __forceinline__ bool scan_pixel(const ScanParams& p, int i, float e[3], int ko[3],
                                           int ke[3], bool* ok_o, bool* ok_e, int* inst,
                                           double* res, bool* end_free) {
  bool valid = i < p.n;
  e[0] = e[1] = e[2] = 0.f;
  *inst = p.inst;
  *res = p.res;
  if (valid) {
    e[0] = p.points[3 * (size_t)i];
    e[1] = p.points[3 * (size_t)i + 1];
    e[2] = p.points[3 * (size_t)i + 2];
    valid = !(isnan(e[0]) || isnan(e[1]) || isnan(e[2])) && (!p.mask || p.mask[i]);
    if (valid && p.labels) {
      const int l = p.labels[i] - p.lut_lo;
      const int q = (l >= 0 && l < p.lut_n) ? p.lut[l] : -1;
      valid = q >= 0;
      if (valid) { *inst = q; *res = p.inst_res[q]; }
    }
  }
  const double res_factor = 1.0 / *res;
  const float o[3] = {p.ox, p.oy, p.oz};
  *ok_o = *ok_e = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ko[a] = coord_to_key((double)o[a], res_factor);
    ke[a] = coord_to_key((double)e[a], res_factor);
    *ok_o &= ko[a] >= 0;
    *ok_e &= ke[a] >= 0;
  }
  return valid;
}

// The server's free ray of a pixel, in the background's key space: to the point inside max_range
// (:352-358), to o + normalized(p - o) * max_range in float beyond it (:375-383; Vector3::normalized
// divides by the float norm).  end_free: the end point of a pixel inside max_range that is not
// labelled background is free in the background too (:367-372); uncertain pixels included.
__device__ __forceinline__ bool scan_pixel(const ServerScanParams& p, int i, float e[3], int ko[3],
                                           int ke[3], bool* ok_o, bool* ok_e, int* inst,
                                           double* res, bool* end_free) {
  int q;
  const bool valid = server_point(p, i, e, &q);
  *inst = p.bg;
  *res = p.res;
  const float o[3] = {p.ox, p.oy, p.oz};
  bool in_range = false;
  if (valid) {
    float d[3];
    const double len = server_ray(p, e, d);
    in_range = p.max_range < 0.0 || len <= p.max_range;
    if (!in_range) {
      const float fl = (float)len, mr = (float)p.max_range;
#pragma unroll
      for (int a = 0; a < 3; ++a) e[a] = __fadd_rn(o[a], __fmul_rn(__fdiv_rn(d[a], fl), mr));
    }
  }
  const double res_factor = 1.0 / p.res;
  *ok_o = *ok_e = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ko[a] = coord_to_key((double)o[a], res_factor);
    ke[a] = coord_to_key((double)e[a], res_factor);
    *ok_o &= ko[a] >= 0;
    *ok_e &= ke[a] >= 0;
  }
  *end_free = valid && in_range && q != p.bg && *ok_e;
  return valid;
}

__global__ void __launch_bounds__(256)
k_map_scan_hits(ScanParams p, MapTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float e[3];
  int ko[3], ke[3], inst;
  double res;
  bool ok_o, ok_e, end_free;
  if (!scan_pixel(p, i, e, ko, ke, &ok_o, &ok_e, &inst, &res, &end_free) || !ok_e) return;
  MapCell seen;
  const int s = map_find_or_insert(t, pack_key(inst, ke[0], ke[1], ke[2]), &seen);
  if (s >= 0) map_scan_update(t, s, seen, 2u * p.scan + 1u, p.hit, p.lo_min, p.lo_max);
}

// The server's hits (:361-366): a listed pixel inside max_range is a hit in its own instance's
// key space.  Every listed pixel, inside max_range or not (the push precedes the range check,
// :340-349), adds its world point to its instance's centre sums; the background's centre is never
// read (publishGrids skips it, :530-532), so it is not summed.
__global__ void __launch_bounds__(256)
k_map_server_hits(ServerScanParams p, MapTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float w[3], d[3];
  int q;
  if (!server_point(p, i, w, &q) || q < 0) return;
  if (q != p.bg) {
#pragma unroll
    for (int a = 0; a < 3; ++a) atomicAdd(p.csum + 4 * q + a, (u64)centre_fix(w[a]));
    atomicAdd(p.csum + 4 * q + 3, 1ull);
    atomicMax(p.cfirst + q, ~(unsigned)i);
  }
  const double len = server_ray(p, w, d);
  if (!(p.max_range < 0.0 || len <= p.max_range)) return;
  const double rf = 1.0 / p.inst_res[q];
  const int kx = coord_to_key((double)w[0], rf), ky = coord_to_key((double)w[1], rf),
            kz = coord_to_key((double)w[2], rf);
  if (kx < 0 || ky < 0 || kz < 0) return;
  MapCell seen;
  const int s = map_find_or_insert(t, pack_key(q, kx, ky, kz), &seen);
  if (s >= 0) map_scan_update(t, s, seen, 2u * p.scan + 1u, p.hit, p.lo_min, p.lo_max);
}

// The centres (:404-447), one thread per instance, after k_map_server_hits.  The server does not
// push an instance's first point of a scan (:345-349): of a parallel scan that is the lowest kept
// pixel index, whose point is taken back out of the sums.  centers_.insert never overwrites, so a
// centre is set by the first scan that pushed a point and stays.  (With no point pushed the server
// reads an uninitialised centroid; here the instance has no centre yet.)  The sums are reset for
// the next scan.
__global__ void __launch_bounds__(256)
k_map_server_centres(ServerScanParams p, int n_inst, float* __restrict__ centres,
                     int* __restrict__ centre_set) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_inst) return;
  u64* acc = p.csum + 4 * q;
  const u64 cnt = acc[3];
  if (!centre_set[q] && cnt >= 2) {
    float w[3];
    int qq;
    server_point(p, (int)~p.cfirst[q], w, &qq);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const long long s = (long long)(acc[a] - (u64)centre_fix(w[a]));
      centres[3 * q + a] = (float)((double)s * (1.0 / 4294967296.0) / (double)(cnt - 1));
    }
    centre_set[q] = 1;
  }
  acc[0] = acc[1] = acc[2] = acc[3] = 0ull;
  p.cfirst[q] = 0u;
}

// An instance box as [6] u32: box_enc of (min x, y, z, max x, y, z).  box_enc orders like the
// floats it encodes (non-NaN), so atomicMin / atomicMax on it give the exact float min / max in
// any order of the atomics.  A zero is encoded as +0: the server's sign of a zero bound depends
// on its OpenMP order, and inBBX does not see it.
__device__ __forceinline__ unsigned box_enc(float f) {
  const unsigned b = __float_as_uint(f == 0.f ? 0.f : f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float box_dec(unsigned e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

// The server creates an instance's tree in the first scan whose label image holds its id on any
// pixel -- odd rows and columns and NaN points included -- (unique(label_ins), :290-319), and in
// that scan its box is set to, not widened by, the min / max of the points it pushes (:425-432).
// tree [n_inst] int32: 0 = no tree yet, 1 = a tree, 2 = created by this scan (until
// k_map_server_boxes).  One thread per pixel, before k_map_server_boxes: the thread that creates
// a tree opens its box at pcl::getMinMax3D of no point, (+FLT_MAX, -FLT_MAX).
__global__ void __launch_bounds__(256)
k_map_server_trees(ServerScanParams p, int* __restrict__ tree, unsigned* __restrict__ box) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int l = p.labels[i] - p.lut_lo;
  const int q = (l >= 0 && l < p.lut_n) ? p.lut[l] : -1;
  if (q < 0 || q == p.bg || tree[q] != 0 || atomicCAS(tree + q, 0, 2) != 0) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    box[6 * q + a] = box_enc(3.402823466e38f);
    box[6 * q + 3 + a] = box_enc(-3.402823466e38f);
  }
}

// The boxes (:404-437), after k_map_server_hits (which leaves each instance's point count in
// csum and its first pixel in cfirst) and before k_map_server_centres (which resets both).  Every
// point the server pushes -- a listed point of an instance other than the background, range or
// not, except the instance's first of the scan -- widens its instance's box.  An instance with
// exactly one point pushes none and gets no widening: one whose tree this scan created keeps
// the empty box, an older one its box.  An instance whose tree this scan created with no listed
// point (its id only on odd rows / columns or NaN points) is not boxed by the server and keeps
// OctoMap's default box (0,0,0)-(0,0,0); thread q (< n_inst) restores it and marks the tree as
// existing.
__global__ void __launch_bounds__(256)
k_map_server_boxes(ServerScanParams p, int n_inst, int* __restrict__ tree,
                   unsigned* __restrict__ box) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_inst && tree[i] == 2) {
    if (p.csum[4 * i + 3] == 0ull) {
#pragma unroll
      for (int a = 0; a < 6; ++a) box[6 * i + a] = box_enc(0.f);
    }
    tree[i] = 1;
  }
  float w[3];
  int q;
  const bool push = server_point(p, i, w, &q) && q >= 0 && q != p.bg &&
                    (unsigned)i != ~p.cfirst[q];
  // the pushing lanes of a warp (neighbouring pixels of one row) mostly share an instance: each
  // instance's lanes reduce first, and one of them issues the atomics
  const unsigned act = __ballot_sync(0xffffffffu, push);
  if (!push) return;
  const unsigned peers = __match_any_sync(act, q);
  const bool lead = (__ffs(peers) - 1) == (int)(threadIdx.x & 31);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const unsigned lo = __reduce_min_sync(peers, box_enc(w[a]));
    const unsigned hi = __reduce_max_sync(peers, box_enc(w[a]));
    if (lead) {
      atomicMin(box + 6 * q + a, lo);
      atomicMax(box + 6 * q + 3 + a, hi);
    }
  }
}

// The key ray of computeRayKeys (oracle/octomap.py::OcTree.computeRayKeys has the line-by-line
// commentary): first cell included, end cell excluded; every cell of the ray that this scan has not
// hit gets the miss update.  Runs after k_map_scan_hits / k_map_server_hits of the same scan
// (stream order).  P = ScanParams (OctoMap's insertPointCloud) or ServerScanParams (the server's
// background rays, plus the end-point cell of end_free pixels).
template <class P>
__global__ void __launch_bounds__(256, 5)
k_map_scan_free(P p, MapTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  float e[3];
  int ko[3], ke[3], inst;
  double res;
  bool ok_o, ok_e, end_free = false;
  const bool valid = scan_pixel(p, i, e, ko, ke, &ok_o, &ok_e, &inst, &res, &end_free);
  if (end_free) {
    MapCell seen;
    const int s = map_find_or_insert(t, pack_key(inst, ke[0], ke[1], ke[2]), &seen);
    if (s >= 0) map_scan_update(t, s, seen, 2u * p.scan, p.miss, p.lo_min, p.lo_max);
  }
  bool act = valid && ok_o && ok_e && !(ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]);
  const float o[3] = {p.ox, p.oy, p.oz};
  int step0 = 0, step1 = 0, step2 = 0, cur0 = ko[0], cur1 = ko[1], cur2 = ko[2];
  double tmax0 = 0.0, tmax1 = 0.0, tmax2 = 0.0, td0 = 0.0, td1 = 0.0, td2 = 0.0, flen = 0.0;
  if (act) {
    float d[3] = {__fsub_rn(e[0], o[0]), __fsub_rn(e[1], o[1]), __fsub_rn(e[2], o[2])};
    const float nsq = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])),
                                __fmul_rn(d[2], d[2]));
    const float length = (float)sqrt((double)nsq);
    flen = (double)length;
    int step[3];
    double tmax[3], tdelta[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      d[a] = __fdiv_rn(d[a], length);
      step[a] = d[a] > 0.f ? 1 : (d[a] < 0.f ? -1 : 0);
      if (step[a] != 0) {
        double border = ((double)(ko[a] - TREE_MAX_VAL) + 0.5) * res;
        border += (double)(float)((double)step[a] * res * 0.5);
        tmax[a] = (border - (double)o[a]) / (double)d[a];
        tdelta[a] = res / fabs((double)d[a]);
      } else {
        tmax[a] = 1.7976931348623157e308;
        tdelta[a] = 1.7976931348623157e308;
      }
    }
    step0 = step[0]; step1 = step[1]; step2 = step[2];
    tmax0 = tmax[0]; tmax1 = tmax[1]; tmax2 = tmax[2];
    td0 = tdelta[0]; td1 = tdelta[1]; td2 = tdelta[2];
  }
  const unsigned want = 2u * p.scan;
  u64 key = pack_key(inst, cur0, cur1, cur2);
  for (;;) {
    const unsigned bal = __ballot_sync(0xffffffffu, act);
    if (!bal) break;
    if (act) {
      // lanes of this step that stand in the same cell: the lowest one does the table work.  Its
      // 16-byte probe is issued here and looked at after the DDA advance below (ALU work that
      // does not depend on it), which hides most of the L2 latency.
      const unsigned peers = __match_any_sync(bal, key);
      const bool lead = (__ffs(peers) - 1) == lane;
      const unsigned s0 = map_hash(key) & t.mask;
      MapCell c;
      c.key = 0; c.lo = 0.f; c.stamp = 0u;
      if (lead) c = map_load(t.cells + s0);
      const u64 kcur = key;
      // advance to the next cell.  The library's selection
      //   if (tMax0 < tMax1) dim = tMax0 < tMax2 ? 0 : 2;  else dim = tMax1 < tMax2 ? 1 : 2;
      // as predicates (no divergence); "min(tMax) > length" <=> every tMax > length
      const bool lt01 = tmax0 < tmax1, lt02 = tmax0 < tmax2, lt12 = tmax1 < tmax2;
      const bool a0 = lt01 && lt02, a1 = !lt01 && lt12;
      const bool a2 = !(a0 || a1);
      const double n0 = tmax0 + td0, n1 = tmax1 + td1, n2 = tmax2 + td2;
      tmax0 = a0 ? n0 : tmax0;
      tmax1 = a1 ? n1 : tmax1;
      tmax2 = a2 ? n2 : tmax2;
      cur0 += a0 ? step0 : 0;
      cur1 += a1 ? step1 : 0;
      cur2 += a2 ? step2 : 0;
      const int cc = a0 ? cur0 : (a1 ? cur1 : cur2);
      const bool at_end = cur0 == ke[0] && cur1 == ke[1] && cur2 == ke[2];
      const bool over = tmax0 > flen && tmax1 > flen && tmax2 > flen;
      act = !(at_end || over || cc < 0 || cc >= 2 * TREE_MAX_VAL);
      key = pack_key(inst, cur0, cur1, cur2);
      // the probe: the common case is "first slot holds the key and is already stamped"
      if (lead) {
        if (c.key == kcur) {
          map_scan_update(t, (int)s0, c, want, p.miss, p.lo_min, p.lo_max);
        } else {
          MapCell seen;
          const int s = map_find_or_insert(t, kcur, &seen);
          if (s >= 0) map_scan_update(t, s, seen, want, p.miss, p.lo_min, p.lo_max);
        }
      }
    }
  }
}

// octomap-python updateNodes(points, occupied): one updateNode per row (double coordinates, no
// de-duplication): count the rows per cell, then the thread that collects a cell's count applies
// the update that many times (the update sequence of a cell is the same value k times, so the
// result depends on k only).
__global__ void __launch_bounds__(256)
k_map_update_count(const double* __restrict__ pts, int m, double res_factor, int inst, MapTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int kx = coord_to_key(pts[3 * (size_t)i], res_factor);
  const int ky = coord_to_key(pts[3 * (size_t)i + 1], res_factor);
  const int kz = coord_to_key(pts[3 * (size_t)i + 2], res_factor);
  if (kx < 0 || ky < 0 || kz < 0) return;       // NaN rows land here too
  MapCell seen;
  const int s = map_find_or_insert(t, pack_key(inst, kx, ky, kz), &seen);
  if (s >= 0) atomicAdd(t.cnt + s, 1u);
}

__global__ void __launch_bounds__(256)
k_map_update_apply(const double* __restrict__ pts, int m, double res_factor, int inst, float upd,
                   float lo_min, float lo_max, MapTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int kx = coord_to_key(pts[3 * (size_t)i], res_factor);
  const int ky = coord_to_key(pts[3 * (size_t)i + 1], res_factor);
  const int kz = coord_to_key(pts[3 * (size_t)i + 2], res_factor);
  if (kx < 0 || ky < 0 || kz < 0) return;
  MapCell seen;
  const int s = map_find(t, pack_key(inst, kx, ky, kz), &seen);
  if (s < 0) return;
  unsigned k = atomicExch(t.cnt + s, 0u);
  if (!k) return;
  float v = seen.lo;                            // written by an earlier launch only
  for (; k; --k) v = map_clamped_add(v, upd, lo_min, lo_max);
  t.cells[s].lo = v;
}

// get_target_grids for T targets at once (multi_instance_octree_mapping.py:35-94)
__global__ void __launch_bounds__(256)
k_map_query_grids(const int* __restrict__ target_index, const double* __restrict__ pitch,
                  const double* __restrict__ origin, int T, int X, int Y, int Z,
                  const double* __restrict__ res_factor, int n_inst, MapTable t,
                  float* __restrict__ g_target, float* __restrict__ g_nontarget,
                  float* __restrict__ g_empty) {
  const long long V = (long long)X * Y * Z;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= V * T) return;
  const int tg = (int)(gid / V);
  const int v = (int)(gid - (long long)tg * V);
  const int k = v % Z, j = (v / Z) % Y, i = v / (Z * Y);
  const double pt = pitch[tg];
  // trimesh matrix_to_points: indices * pitch + origin (float64)
  const double cx = (double)i * pt + origin[3 * tg];
  const double cy = (double)j * pt + origin[3 * tg + 1];
  const double cz = (double)k * pt + origin[3 * tg + 2];
  const int tin = target_index[tg];
  float gt = 0.f, gn = 0.f, ge = 0.f;
  for (int q = 0; q < n_inst; ++q) {
    const double rf = res_factor[q];
    const int kx = coord_to_key(cx, rf), ky = coord_to_key(cy, rf), kz = coord_to_key(cz, rf);
    if (kx < 0 || ky < 0 || kz < 0) continue;
    MapCell c;
    if (map_find(t, pack_key(q, kx, ky, kz), &c) < 0) continue;
    const double occ = 1.0 - (1.0 / (1.0 + exp((double)c.lo)));      // octomap::probability
    if (occ >= 0.5) {
      if (q == tin) gt = (float)occ; else gn = (float)occ;
    } else if (occ >= 0.0) {
      ge = (float)(1.0 - occ);
    }
  }
  g_target[gid] = gt;
  g_nontarget[gid] = gn;
  g_empty[gid] = ge;
}

// The refinement node's grid / grid_noentry pair (OctomapServer::publishGrids,
// ros/src/morefusion_ros/src/OctomapServer.cpp:510-618; oracle/octomap_server.py restates it rule
// by rule) for T targets at once, one thread per (target, voxel).  The server pushes an (index,
// value) pair for every qualifying instance and the node decodes them with a NumPy fancy
// assignment, so the last qualifying instance in map order wins; `walk` lists the dense indices
// in REVERSE map order and the first one that qualifies is taken.
// kWorld: origins are in the camera frame and every voxel centre is moved to the world frame
// with `x` (sensorToWorld) before the look-up (:573-576); x.ground: a centre below world z = 0
// is no-entry at probability_max and nothing else is looked at (ground_as_noentry, :579-583).
struct NodeXform {
  float m[12];                // rows 0-2 of sensorToWorld as an Eigen::Matrix4f
  int ground;
};

template <bool kWorld>
__device__ __forceinline__ void
node_grids(const int* __restrict__ target_index, const double* __restrict__ pitch,
           const double* __restrict__ origin, int T, int X, int Y, int Z,
           const double* __restrict__ res_factor, const int* __restrict__ walk, int n_inst,
           int background, double probability_max, const MapTable& t, float* __restrict__ g_grid,
           float* __restrict__ g_noentry, const NodeXform& x) {
  const long long V = (long long)X * Y * Z;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= V * T) return;
  const int tg = (int)(gid / V);
  const int v = (int)(gid - (long long)tg * V);
  const int k = v % Z, j = (v / Z) % Y, i = v / (Z * Y);
  const double pt = pitch[tg];
  // :566-575 the centre in double, then a float PCLPoint; search() takes it back as double
  double cx = (double)(float)(origin[3 * tg] + pt * (double)i);
  double cy = (double)(float)(origin[3 * tg + 1] + pt * (double)j);
  double cz = (double)(float)(origin[3 * tg + 2] + pt * (double)k);
  if constexpr (kWorld) {
    float w[3];
    xform_f32(x.m, (float)cx, (float)cy, (float)cz, w);
    if (x.ground && w[2] < 0.f) {
      g_grid[gid] = 0.f;
      g_noentry[gid] = (float)probability_max;
      return;
    }
    cx = (double)w[0];
    cy = (double)w[1];
    cz = (double)w[2];
  }
  const int tin = target_index[tg];
  float gg = 0.f, gne = 0.f;
  bool occupied = false;
  {
    const double rf = res_factor[tin];
    const int kx = coord_to_key(cx, rf), ky = coord_to_key(cy, rf), kz = coord_to_key(cz, rf);
    MapCell c;
    if (kx >= 0 && ky >= 0 && kz >= 0 && map_find(t, pack_key(tin, kx, ky, kz), &c) >= 0) {
      const double occ = 1.0 - (1.0 / (1.0 + exp((double)c.lo)));
      if (occ > 0.5) { gg = (float)occ; occupied = true; }                         // :586-589
    }
  }
  for (int w = 0; w < n_inst && !occupied; ++w) {                                  // :591-610
    const int q = walk[w];
    if (q == tin) continue;
    const double rf = res_factor[q];
    const int kx = coord_to_key(cx, rf), ky = coord_to_key(cy, rf), kz = coord_to_key(cz, rf);
    if (kx < 0 || ky < 0 || kz < 0) continue;
    MapCell c;
    if (map_find(t, pack_key(q, kx, ky, kz), &c) < 0) continue;
    const double occ = 1.0 - (1.0 / (1.0 + exp((double)c.lo)));
    if (q == background && occ < 0.5) { gne = (float)(1.0 - occ); break; }          // free_as_noentry
    if (occ >= probability_max) { gne = (float)occ; break; }
  }
  g_grid[gid] = gg;
  g_noentry[gid] = gne;
}

__global__ void __launch_bounds__(256)
k_map_query_node_grids(const int* __restrict__ target_index, const double* __restrict__ pitch,
                       const double* __restrict__ origin, int T, int X, int Y, int Z,
                       const double* __restrict__ res_factor, const int* __restrict__ walk,
                       int n_inst, int background, double probability_max, MapTable t,
                       float* __restrict__ g_grid, float* __restrict__ g_noentry) {
  node_grids<false>(target_index, pitch, origin, T, X, Y, Z, res_factor, walk, n_inst, background,
                    probability_max, t, g_grid, g_noentry, NodeXform{});
}

__global__ void __launch_bounds__(256)
k_map_query_node_grids_world(const int* __restrict__ target_index,
                             const double* __restrict__ pitch, const double* __restrict__ origin,
                             int T, int X, int Y, int Z, const double* __restrict__ res_factor,
                             const int* __restrict__ walk, int n_inst, int background,
                             double probability_max, MapTable t, float* __restrict__ g_grid,
                             float* __restrict__ g_noentry, NodeXform x) {
  node_grids<true>(target_index, pitch, origin, T, X, Y, Z, res_factor, walk, n_inst, background,
                   probability_max, t, g_grid, g_noentry, x);
}

// publishGrids' per-target pitch and origin (:534-551): the world centre moved to the camera
// frame in float by `inv` (world -> sensor), origin = centre - (dims / 2 - 0.5) * pitch in double
__global__ void __launch_bounds__(256)
k_map_server_grid_params(const int* __restrict__ target_index, int T,
                         const double* __restrict__ inst_res, const float* __restrict__ centres,
                         NodeXform inv, double off_x, double off_y, double off_z,
                         double* __restrict__ pitch, double* __restrict__ origin) {
  const int tg = blockIdx.x * blockDim.x + threadIdx.x;
  if (tg >= T) return;
  const int q = target_index[tg];
  float c[3];
  xform_f32(inv.m, centres[3 * q], centres[3 * q + 1], centres[3 * q + 2], c);
  const double pt = inst_res[q];
  pitch[tg] = pt;
  origin[3 * tg] = (double)c[0] - off_x * pt;
  origin[3 * tg + 1] = (double)c[1] - off_y * pt;
  origin[3 * tg + 2] = (double)c[2] - off_z * pt;
}

// OccupancyOcTreeBase::castRay(origin, dir, end, ignoreUnknownCells = true, max_range) in
// instance q's key space; oracle/octomap_server_render.py::cast_ray restates it line by line.
// True with `end` = the centre of the first occupied cell (isNodeOccupied: log-odds >= 0) on the
// ray, the origin's own cell included; unknown and free cells are passed.  False when the origin
// is outside the key range, the direction is zero, a key would leave the range, or a cell centre
// lies beyond max_range (> 0; otherwise no limit).  Every DDA step is taken: tMax accumulates
// its rounding in sequence, as the library's does.
__device__ __forceinline__ bool cast_ray(const MapTable& t, int q, double res, const float o[3],
                                         const float dir[3], double max_range, float end[3]) {
  const double rf = 1.0 / res;
  int cur[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    cur[a] = coord_to_key((double)o[a], rf);
    if (cur[a] < 0) return false;
  }
  MapCell c;
#pragma unroll
  for (int a = 0; a < 3; ++a) end[a] = (float)(((double)(cur[a] - TREE_MAX_VAL) + 0.5) * res);
  if (map_find(t, pack_key(q, cur[0], cur[1], cur[2]), &c) >= 0 && c.lo >= 0.f) return true;
  // direction.normalized(): divided by the float of point3d::norm() when that is > 0
  float dn[3];
  const double len = point_diff_norm(dir, 0.f, 0.f, 0.f, dn);
#pragma unroll
  for (int a = 0; a < 3; ++a) dn[a] = len > 0.0 ? __fdiv_rn(dir[a], (float)len) : dir[a];
  int step[3];
  double tmax[3], tdelta[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    step[a] = dn[a] > 0.f ? 1 : (dn[a] < 0.f ? -1 : 0);
    if (step[a] != 0) {
      // castRay keeps the half step in double (computeRayKeys rounds it to float)
      double border = ((double)(cur[a] - TREE_MAX_VAL) + 0.5) * res;
      border += (double)step[a] * res * 0.5;
      tmax[a] = (border - (double)o[a]) / (double)dn[a];
      tdelta[a] = res / fabs((double)dn[a]);
    } else {
      tmax[a] = 1.7976931348623157e308;
      tdelta[a] = 1.7976931348623157e308;
    }
  }
  if (step[0] == 0 && step[1] == 0 && step[2] == 0) return false;
  const bool range_set = max_range > 0.0;
  const double range_sq = max_range * max_range;
  for (;;) {
    const int dim = tmax[0] < tmax[1] ? (tmax[0] < tmax[2] ? 0 : 2) : (tmax[1] < tmax[2] ? 1 : 2);
    bool out = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (a != dim) continue;
      out = (step[a] < 0 && cur[a] == 0) || (step[a] > 0 && cur[a] == 2 * TREE_MAX_VAL - 1);
      cur[a] += step[a];
      tmax[a] += tdelta[a];
    }
    if (out) return false;
    double dsq = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      end[a] = (float)(((double)(cur[a] - TREE_MAX_VAL) + 0.5) * res);
      const float e = __fsub_rn(end[a], o[a]);
      dsq += (double)__fmul_rn(e, e);
    }
    if (range_set && dsq > range_sq) return false;
    if (map_find(t, pack_key(q, cur[0], cur[1], cur[2]), &c) >= 0 && c.lo >= 0.f) return true;
  }
}

// The server's render (OctomapServer::render, :193-281; oracle/octomap_server_render.py::render)
struct RenderParams {
  const float* points;        // [height*width,3] camera frame, NaN = no depth
  const int* walk;            // [n_walk] dense indices of the rendered instances, ascending id
  const double* inst_res;     // [n_inst] resolution of each instance
  const unsigned* box;        // [n_inst,6] box_enc (k_map_server_boxes)
  int height, width, n_walk;
  float m[12];                // rows 0-2 of sensorToWorld as an Eigen::Matrix4f
  float ox, oy, oz;           // sensor origin (point3d: floats)
  float fx, fy, cx, cy;       // camera_info K rounded to float (:224-227)
};

// One thread per (rendered instance w, even pixel e), w-major: a warp is 32 neighbouring rays of
// one instance.  A pixel with depth casts to its world point, and only into instances whose box
// holds that point (inBBX, :245); a NaN pixel casts to the z = 1 point of its ray with no box
// test (:221-237).  maxRange = 1.1 |point - origin|.  The hit distance, a positive float whose
// bits order like its value, and w pack into one u64 per even pixel: atomicMin keeps the nearest
// hit, and of exact ties the lowest w, i.e. the lowest instance id (the server on one thread:
// std::map order and a strict <).
__global__ void __launch_bounds__(256)
k_map_render_rays(RenderParams p, MapTable t, u64* __restrict__ zbuf) {
  const int we = (p.width + 1) >> 1;
  const long long n_even = (long long)((p.height + 1) >> 1) * we;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_even * p.n_walk) return;
  const int w = (int)(g / n_even);
  const int e = (int)(g - (long long)w * n_even);
  const int v = 2 * (e / we), u = 2 * (e - (e / we) * we);
  const size_t i = (size_t)v * p.width + u;
  const int q = p.walk[w];
  float pt[3];
  xform_f32(p.m, p.points[3 * i], p.points[3 * i + 1], p.points[3 * i + 2], pt);
  if (isnan(pt[0]) || isnan(pt[1]) || isnan(pt[2])) {
    xform_f32(p.m, __fdiv_rn(__fsub_rn((float)u, p.cx), p.fx),
              __fdiv_rn(__fsub_rn((float)v, p.cy), p.fy), 1.f, pt);
  } else {
    const unsigned* b = p.box + 6 * q;
#pragma unroll
    for (int a = 0; a < 3; ++a)
      if (!(pt[a] >= box_dec(b[a]) && pt[a] <= box_dec(b[3 + a]))) return;
  }
  const float o[3] = {p.ox, p.oy, p.oz};
  float dir[3], end[3], de[3];
  const double range = point_diff_norm(pt, p.ox, p.oy, p.oz, dir) * 1.1;
  if (!cast_ray(t, q, p.inst_res[q], o, dir, range, end)) return;
  const float d = (float)point_diff_norm(end, p.ox, p.oy, p.oz, de);
  atomicMin(zbuf + e, ((u64)__float_as_uint(d) << 32) | (u64)(unsigned)w);
}

// One thread per pixel: the nearest instance of the even pixel (v, u) labels rows v-1..v and
// columns u-1..u (the dj, di in {-1, 0} loop, :268-276) and its distance is the depth at (v, u);
// everything else is `uncertain` / NaN.
__global__ void __launch_bounds__(256)
k_map_render_write(const u64* __restrict__ zbuf, const int* __restrict__ walk_ids, int height,
                   int width, int uncertain, int* __restrict__ label, float* __restrict__ depth) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)height * width) return;
  const int r = (int)(i / width), c = (int)(i - (long long)r * width);
  const int v = r + (r & 1), u = c + (c & 1);
  int lab = uncertain;
  float d = __uint_as_float(0x7fc00000u);
  if (v < height && u < width) {
    const u64 z = zbuf[(size_t)(v >> 1) * ((width + 1) >> 1) + (u >> 1)];
    if (z != ~0ull) {
      lab = walk_ids[(unsigned)(z & 0xffffffffull)];
      if (v == r && u == c) d = __uint_as_float((unsigned)(z >> 32));
    }
  }
  label[i] = lab;
  depth[i] = d;
}

__global__ void __launch_bounds__(256)
k_map_rehash(const MapCell* __restrict__ old, unsigned old_cap, MapTable t) {
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < old_cap; i += gridDim.x * blockDim.x) {
    const MapCell c = map_load(old + i);
    if (c.key == MAP_EMPTY) continue;
    MapCell seen;
    const int s = map_find_or_insert(t, c.key, &seen);
    if (s >= 0) { t.cells[s].lo = c.lo; t.cells[s].stamp = c.stamp; }
  }
}

}  // namespace mf

#ifndef MF_HOST_EMU
using namespace mf;

static bool table_ok(const void* cells, const void* cnt, long long cap, const void* counters) {
  return cells && cnt && counters && cap >= 64 && cap <= (1LL << 31) && (cap & (cap - 1)) == 0 &&
         ((uintptr_t)cells & 15) == 0;
}

static MapTable make_table(void* cells, void* cnt, long long cap, void* counters) {
  MapTable t;
  t.cells = (MapCell*)cells; t.cnt = (unsigned*)cnt; t.mask = (unsigned)(cap - 1);
  t.counters = (int*)counters;
  return t;
}

extern "C" int mf_map_integrate(const float* points, const uint8_t* mask, int64_t n, float ox,
                                float oy, float oz, double resolution, int instance,
                                uint32_t scan, float hit, float miss, float lo_min, float lo_max,
                                void* cells, void* cnt, int64_t capacity, int32_t* counters,
                                void* stream_) {
  if (!points || n <= 0 || n >= (1LL << 31) || !(resolution > 0.0) || instance < 0 ||
      instance >= 0xFFFF || scan == 0 || scan >= (1u << 31) ||
      !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  MapTable t = make_table(cells, cnt, capacity, counters);
  ScanParams p;
  p.points = points; p.mask = mask; p.labels = nullptr; p.lut = nullptr; p.inst_res = nullptr;
  p.lut_lo = 0; p.lut_n = 0; p.n = (int)n; p.ox = ox; p.oy = oy; p.oz = oz;
  p.res = resolution; p.inst = instance; p.scan = scan;
  p.hit = hit; p.miss = miss; p.lo_min = lo_min; p.lo_max = lo_max;
  k_map_scan_hits<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  k_map_scan_free<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_integrate_labelled(const float* points, const int32_t* labels, int64_t n,
                                         float ox, float oy, float oz, const int32_t* lut,
                                         int lut_lo, int lut_n, const double* inst_resolution,
                                         uint32_t scan, float hit, float miss, float lo_min,
                                         float lo_max, void* cells, void* cnt, int64_t capacity,
                                         int32_t* counters, void* stream_) {
  if (!points || !labels || !lut || lut_n <= 0 || !inst_resolution || n <= 0 || n >= (1LL << 31) ||
      scan == 0 || scan >= (1u << 31) || !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  MapTable t = make_table(cells, cnt, capacity, counters);
  ScanParams p;
  p.points = points; p.mask = nullptr; p.labels = labels; p.lut = lut; p.inst_res = inst_resolution;
  p.lut_lo = lut_lo; p.lut_n = lut_n; p.n = (int)n; p.ox = ox; p.oy = oy; p.oz = oz;
  p.res = 1.0; p.inst = 0; p.scan = scan;
  p.hit = hit; p.miss = miss; p.lo_min = lo_min; p.lo_max = lo_max;
  k_map_scan_hits<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  k_map_scan_free<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_update_points(const double* points, int64_t m, double resolution,
                                    int instance, float update, float lo_min, float lo_max,
                                    void* cells, void* cnt, int64_t capacity, int32_t* counters,
                                    void* stream_) {
  if (!points || m <= 0 || m >= (1LL << 31) || !(resolution > 0.0) || instance < 0 ||
      instance >= 0xFFFF || !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  MapTable t = make_table(cells, cnt, capacity, counters);
  k_map_update_count<<<div_up(m, 256), 256, 0, st>>>(points, (int)m, 1.0 / resolution, instance, t);
  MF_LAUNCH_CHECK();
  k_map_update_apply<<<div_up(m, 256), 256, 0, st>>>(points, (int)m, 1.0 / resolution, instance,
                                                     update, lo_min, lo_max, t);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_query_grids(const int32_t* target_index, const double* pitch,
                                  const double* origin, int T, int X, int Y, int Z,
                                  const double* res_factor, int n_instances, void* cells,
                                  void* cnt, int64_t capacity, int32_t* counters,
                                  float* grid_target, float* grid_nontarget, float* grid_empty,
                                  void* stream_) {
  if (!target_index || !pitch || !origin || T <= 0 || X <= 0 || Y <= 0 || Z <= 0 || !res_factor ||
      n_instances < 0 || !grid_target || !grid_nontarget || !grid_empty ||
      (long long)T * X * Y * Z >= (1LL << 40) || !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  MapTable t = make_table(cells, cnt, capacity, counters);
  const long long total = (long long)T * X * Y * Z;
  k_map_query_grids<<<div_up(total, 256), 256, 0, (cudaStream_t)stream_>>>(
      target_index, pitch, origin, T, X, Y, Z, res_factor, n_instances, t, grid_target,
      grid_nontarget, grid_empty);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_query_node_grids(const int32_t* target_index, const double* pitch,
                                       const double* origin, int T, int X, int Y, int Z,
                                       const double* res_factor, const int32_t* walk,
                                       int n_instances, int background, double probability_max,
                                       void* cells, void* cnt, int64_t capacity,
                                       int32_t* counters, float* grid, float* grid_noentry,
                                       void* stream_) {
  if (!target_index || !pitch || !origin || T <= 0 || X <= 0 || Y <= 0 || Z <= 0 || !res_factor ||
      n_instances <= 0 || !walk || background < -1 ||
      background >= n_instances || !grid || !grid_noentry ||
      (long long)T * X * Y * Z >= (1LL << 40) || !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  MapTable t = make_table(cells, cnt, capacity, counters);
  const long long total = (long long)T * X * Y * Z;
  k_map_query_node_grids<<<div_up(total, 256), 256, 0, (cudaStream_t)stream_>>>(
      target_index, pitch, origin, T, X, Y, Z, res_factor, walk, n_instances, background,
      probability_max, t, grid, grid_noentry);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

static bool xform_ok(const float* m) {
  if (!m) return false;
  for (int a = 0; a < 12; ++a)
    if (!isfinite(m[a])) return false;
  return true;
}

static NodeXform make_xform(const float* m, int ground) {
  NodeXform x;
  for (int a = 0; a < 12; ++a) x.m[a] = m[a];
  x.ground = ground;
  return x;
}

extern "C" int mf_map_query_node_grids_world(const int32_t* target_index, const double* pitch,
                                             const double* origin, int T, int X, int Y, int Z,
                                             const double* res_factor, const int32_t* walk,
                                             int n_instances, int background,
                                             double probability_max, const float* sensor_to_world,
                                             int ground_as_noentry, void* cells, void* cnt,
                                             int64_t capacity, int32_t* counters, float* grid,
                                             float* grid_noentry, void* stream_) {
  if (!target_index || !pitch || !origin || T <= 0 || X <= 0 || Y <= 0 || Z <= 0 || !res_factor ||
      n_instances <= 0 || !walk || background < -1 || background >= n_instances || !grid ||
      !grid_noentry || !xform_ok(sensor_to_world) || (long long)T * X * Y * Z >= (1LL << 40) ||
      !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  MapTable t = make_table(cells, cnt, capacity, counters);
  const long long total = (long long)T * X * Y * Z;
  k_map_query_node_grids_world<<<div_up(total, 256), 256, 0, (cudaStream_t)stream_>>>(
      target_index, pitch, origin, T, X, Y, Z, res_factor, walk, n_instances, background,
      probability_max, t, grid, grid_noentry, make_xform(sensor_to_world, ground_as_noentry != 0));
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_integrate_server(const float* points, const int32_t* labels, int height,
                                       int width, const float* sensor_to_world, double max_range,
                                       const int32_t* lut, int lut_lo, int lut_n,
                                       const double* inst_resolution, int n_instances,
                                       int background, double background_resolution,
                                       int uncertain, uint32_t scan, float hit, float miss,
                                       float lo_min, float lo_max, void* centre_sums,
                                       uint32_t* centre_first, float* centres,
                                       int32_t* centre_set, void* cells, void* cnt,
                                       int64_t capacity, int32_t* counters,
                                       int32_t* tree_state, uint32_t* boxes, void* stream_) {
  const long long n = (long long)height * width;
  if (!points || !labels || !lut || lut_n <= 0 || !inst_resolution || height <= 0 || width <= 0 ||
      n >= (1LL << 31) || n_instances <= 0 || background < 0 || background >= n_instances ||
      !(background_resolution > 0.0) || !xform_ok(sensor_to_world) || isnan(max_range) ||
      !centre_sums || !centre_first || !centres || !centre_set || scan == 0 ||
      scan >= (1u << 31) || !table_ok(cells, cnt, capacity, counters) || !tree_state || !boxes)
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  MapTable t = make_table(cells, cnt, capacity, counters);
  ServerScanParams p;
  p.points = points; p.labels = labels; p.lut = lut; p.inst_res = inst_resolution;
  p.csum = (u64*)centre_sums; p.cfirst = centre_first;
  p.lut_lo = lut_lo; p.lut_n = lut_n; p.n = (int)n; p.width = width;
  p.bg = background; p.uncertain = uncertain;
  for (int a = 0; a < 12; ++a) p.m[a] = sensor_to_world[a];
  p.ox = sensor_to_world[3]; p.oy = sensor_to_world[7]; p.oz = sensor_to_world[11];
  p.max_range = max_range; p.res = background_resolution; p.scan = scan;
  p.hit = hit; p.miss = miss; p.lo_min = lo_min; p.lo_max = lo_max;
  k_map_server_trees<<<div_up(n, 256), 256, 0, st>>>(p, tree_state, boxes);
  MF_LAUNCH_CHECK();
  k_map_server_hits<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  k_map_server_boxes<<<div_up(n > n_instances ? n : n_instances, 256), 256, 0, st>>>(
      p, n_instances, tree_state, boxes);
  MF_LAUNCH_CHECK();
  k_map_scan_free<<<div_up(n, 256), 256, 0, st>>>(p, t);
  MF_LAUNCH_CHECK();
  k_map_server_centres<<<div_up(n_instances, 256), 256, 0, st>>>(p, n_instances, centres,
                                                                  centre_set);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_server_grid_params(const int32_t* target_index, int T,
                                         const double* inst_resolution, const float* centres,
                                         const float* world_to_sensor, double off_x, double off_y,
                                         double off_z, double* pitch, double* origin,
                                         void* stream_) {
  if (!target_index || T <= 0 || !inst_resolution || !centres || !xform_ok(world_to_sensor) ||
      !pitch || !origin)
    return MF_E_BADARG;
  k_map_server_grid_params<<<div_up(T, 256), 256, 0, (cudaStream_t)stream_>>>(
      target_index, T, inst_resolution, centres, make_xform(world_to_sensor, 0), off_x, off_y,
      off_z, pitch, origin);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_map_render(const float* points, int height, int width,
                             const float* sensor_to_world, float fx, float fy, float cx, float cy,
                             const int32_t* walk, const int32_t* walk_ids, int n_walk,
                             const double* inst_resolution, const uint32_t* boxes, int uncertain,
                             void* zbuf, int32_t* label, float* depth, void* cells, void* cnt,
                             int64_t capacity, int32_t* counters, void* stream_) {
  const long long n = (long long)height * width;
  if (!points || height <= 0 || width <= 0 || n >= (1LL << 31) || !xform_ok(sensor_to_world) ||
      !isfinite(fx) || !isfinite(fy) || !isfinite(cx) || !isfinite(cy) || n_walk < 0 ||
      n_walk >= 0xFFFF || (n_walk > 0 && (!walk || !walk_ids || !inst_resolution || !boxes)) ||
      !zbuf || !label || !depth || !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  const long long n_even = (long long)((height + 1) / 2) * ((width + 1) / 2);
  MF_CUDA_TRY(cudaMemsetAsync(zbuf, 0xFF, (size_t)n_even * sizeof(u64), st));
  if (n_walk > 0) {
    RenderParams p;
    p.points = points; p.walk = walk; p.inst_res = inst_resolution; p.box = boxes;
    p.height = height; p.width = width; p.n_walk = n_walk;
    for (int a = 0; a < 12; ++a) p.m[a] = sensor_to_world[a];
    p.ox = sensor_to_world[3]; p.oy = sensor_to_world[7]; p.oz = sensor_to_world[11];
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy;
    k_map_render_rays<<<div_up(n_even * n_walk, 256), 256, 0, st>>>(
        p, make_table(cells, cnt, capacity, counters), (u64*)zbuf);
    MF_LAUNCH_CHECK();
  }
  k_map_render_write<<<div_up(n, 256), 256, 0, st>>>((const u64*)zbuf, walk_ids, height, width,
                                                     uncertain, label, depth);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

// growth (rare, never on the per-frame path): `counters` restarts from the re-inserted cells
extern "C" int mf_map_rehash(const void* old_cells, int64_t old_capacity, void* cells, void* cnt,
                             int64_t capacity, int32_t* counters, void* stream_) {
  if (!old_cells || old_capacity <= 0 || old_capacity > (1LL << 31) || capacity < old_capacity ||
      !table_ok(cells, cnt, capacity, counters))
    return MF_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream_;
  MapTable t = make_table(cells, cnt, capacity, counters);
  MF_CUDA_TRY(cudaMemsetAsync(counters, 0, 2 * sizeof(int32_t), st));
  int dev = 0, n_sm = 0;
  MF_CUDA_TRY(cudaGetDevice(&dev));
  MF_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
  k_map_rehash<<<n_sm * 8, 256, 0, st>>>((const MapCell*)old_cells, (unsigned)old_capacity, t);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
#endif  // MF_HOST_EMU
