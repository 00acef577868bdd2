// TEST INFRASTRUCTURE: serial host execution of morefusion_b200/csrc/mesh_models.cu (built by
// tests/test_mesh_models_emu.py with g++ -DMF_HOST_EMU).  The per-face surface and parity code
// (mm_surface_face, mm_parity_face) runs as one lane per face, in face order, and the per-pair
// distance code (mm_sdf_pair) over every face of the point's mesh in index order: the kernels'
// warps, tiles and chunks only change which thread does a piece of work, and OR, XOR, min with
// the first index kept and ordered compaction do not depend on that.  The bounds, the matrix and
// the compaction are restated here serially.
#define MF_HOST_EMU 1
#include <string.h>

#include <vector>

#include "../../morefusion_b200/csrc/mesh_models.cu"

using namespace mf;

static void emu_meshes(const double* v, int V, const int32_t* faces, int F, const int64_t* offsets,
                       int S, MmMeshes& m) {
  m.v = v; m.faces = faces; m.V = V; m.F = F; m.S = S;
  for (int s = 0; s <= MF_MESH_MODELS_MAX_MESHES; ++s) m.off[s] = s <= S ? (int)offsets[s] : F;
}

// Same outputs as mf_mesh_voxelize_solid, without the workspace and the stream.
extern "C" int emu_voxelize_solid(const double* v, int V, const int32_t* faces, int F,
                                  const int64_t* offsets, int S, int D, uint8_t* matrix,
                                  int32_t* counts, double* points, double* translate, double* scale,
                                  double* pitch) {
  MmMeshes m;
  emu_meshes(v, V, faces, F, offsets, S, m);
  const int W = (D + 31) / 32;
  for (int s = 0; s < S; ++s) {
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int r = m.off[s] * 3; r < m.off[s + 1] * 3; ++r)
      for (int q = 0; q < 3; ++q) {
        lo[q] = fmin(lo[q], v[3 * (size_t)faces[r] + q]);
        hi[q] = fmax(hi[q], v[3 * (size_t)faces[r] + q]);
      }
    const bool any = m.off[s + 1] > m.off[s];
    double sc = 0.0;
    for (int q = 0; q < 3; ++q) {
      translate[3 * s + q] = any ? lo[q] : 0.0;
      sc = q == 0 ? hi[q] - lo[q] : fmax(sc, hi[q] - lo[q]);
    }
    if (!any || !isfinite(sc)) sc = 0.0;
    scale[s] = sc;
    pitch[s] = sc / D;
  }
  std::vector<uint32_t> surf((size_t)S * D * D * W), par((size_t)S * D * D * W);
  for (int f = 0; f < F; ++f) {
    mm_surface_face(m, f, D, W, translate, pitch, surf.data(), 0, 1);
    mm_parity_face(m, f, D, W, translate, pitch, par.data(), 0, 1);
  }
  const size_t D3 = (size_t)D * D * D;
  for (int s = 0; s < S; ++s) {
    int n = 0;
    for (int i = 0; i < D; ++i)
      for (int j = 0; j < D; ++j)
        for (int k = 0; k < D; ++k) {
          const size_t w = mm_col(s, i, j, D, W) + (k >> 5);
          const int b = ((surf[w] | par[w]) >> (k & 31)) & 1;
          matrix[s * D3 + ((size_t)i * D + j) * D + k] = (uint8_t)b;
          if (b) {
            double* r = points + (s * D3 + n) * 3;
            r[0] = mm_centre(translate[3 * s], pitch[s], i);
            r[1] = mm_centre(translate[3 * s + 1], pitch[s], j);
            r[2] = mm_centre(translate[3 * s + 2], pitch[s], k);
            ++n;
          }
        }
    counts[s] = n;
    for (size_t r = n; r < D3; ++r)
      for (int q = 0; q < 3; ++q) points[(s * D3 + r) * 3 + q] = NAN;
  }
  return 0;
}

// Same outputs as mf_mesh_signed_distance.
extern "C" int emu_signed_distance(const double* v, int V, const int32_t* faces, int F,
                                   const int64_t* offsets, int S, const double* pts,
                                   const int32_t* mesh, int P, double* sdf, int32_t* face) {
  MmMeshes m;
  emu_meshes(v, V, faces, F, offsets, S, m);
  for (int r = 0; r < P; ++r) {
    const int ms = mesh[r];
    double best = INFINITY;
    int arg = -1, odd = 0;
    if (ms >= 0 && ms < S)
      for (int f = m.off[ms]; f < m.off[ms + 1]; ++f) {
        MmTri t;
        mm_load_tri(m, f, t);
        mm_sdf_pair(t, f, pts + 3 * (size_t)r, best, arg, odd);
      }
    const bool ok = ms >= 0 && ms < S && arg >= 0;
    sdf[r] = ok ? mm_signed(best, odd) : NAN;
    face[r] = ok ? arg : -1;
  }
  return 0;
}

// How many faces of mesh s the vertical line through (px, py) crosses, at any z.
extern "C" int emu_column_crossings(const double* v, int V, const int32_t* faces, int F,
                                    const int64_t* offsets, int S, int s, double px, double py) {
  MmMeshes m;
  emu_meshes(v, V, faces, F, offsets, S, m);
  int n = 0;
  for (int f = m.off[s]; f < m.off[s + 1]; ++f) {
    MmTri t;
    mm_load_tri(m, f, t);
    double z;
    n += mm_crossing(t, px, py, z) ? 1 : 0;
  }
  return n;
}
