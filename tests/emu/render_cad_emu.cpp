// TEST INFRASTRUCTURE: serial host execution of morefusion_b200/csrc/render_cad.cu (built by
// tests/test_render_cad_emu.py with g++ -DMF_HOST_EMU).  Same argument list as mf_render_cad
// (include/morefusion_b200.h) minus the workspace and the stream.  k_rc_init and k_rc_setup run
// as they are, one thread at a time; the raster pass applies the .cu's own rc_cover to every
// pixel of each face's box, in face order (the kernel's tiles only change which thread tests a
// pixel, and union and minimum do not depend on order).
#define MF_HOST_EMU 1
#include <string.h>

#include <vector>

#include "../../morefusion_b200/csrc/render_cad.cu"

using namespace mf;

template <class F> static void run(unsigned grid, F f) {
  gridDim = {grid, 1, 1};
  blockDim = {1, 1, 1};
  for (unsigned b = 0; b < grid; ++b) {
    blockIdx = {b, 0, 0};
    threadIdx = {0, 0, 0};
    f();
  }
}

extern "C" int emu_render_cad(const double* vertices, int V, const int32_t* faces, int F,
                              const int64_t* offsets, int S, const int32_t* mesh,
                              const double* Ts_cad2cam, int N, double f, int height, int width,
                              float* depth, uint8_t* mask, int32_t* count) {
  RcParams p;
  p.v = vertices; p.faces = faces; p.mesh = mesh; p.T = Ts_cad2cam;
  p.V = V; p.F = F; p.N = N; p.S = S; p.H = height; p.W = width; p.f = f;
  p.f_max = 0;
  for (int s = 0; s <= S; ++s) p.off[s] = (int)offsets[s];
  for (int s = 0; s < S; ++s) p.f_max = std::max(p.f_max, p.off[s + 1] - p.off[s]);
  std::vector<RcBox> boxes((size_t)N * F);
  std::vector<RcGeom> geom((size_t)N * F);
  std::vector<int4> pose_box(N);
  run((unsigned)N, [&] { k_rc_init(N, pose_box.data(), count); });
  run((unsigned)((long long)N * p.f_max), [&] {
    k_rc_setup(p, boxes.data(), geom.data(), pose_box.data());
  });
  const size_t hw = (size_t)height * width;
  std::vector<uint8_t> hit(hw);
  std::vector<float> zmin(hw);
  for (int n = 0; n < N; ++n) {
    memset(hit.data(), 0, hw);
    int lo, hi;
    if (rc_pose_mesh(p, n, lo, hi))
      for (int k = lo; k < hi; ++k) {
        const RcBox& b = boxes[(size_t)n * F + k];
        if (b.x0 > b.x1) continue;
        for (int r = b.y0; r <= b.y1; ++r)
          for (int c = b.x0; c <= b.x1; ++c) {
            bool h = hit[(size_t)r * width + c];
            rc_cover(geom[(size_t)n * F + k], c, r, h, zmin[(size_t)r * width + c]);
            hit[(size_t)r * width + c] = h;
          }
      }
    int total = 0;
    for (size_t i = 0; i < hw; ++i) {
      depth[n * hw + i] = hit[i] ? zmin[i] : NAN;
      mask[n * hw + i] = hit[i];
      total += hit[i];
    }
    count[n] += total;
  }
  return 0;
}
