// TEST INFRASTRUCTURE: serial host execution of the occupancy server's scan with its boxes
// (k_map_server_trees, k_map_server_hits, k_map_server_boxes, k_map_scan_free<ServerScanParams>,
// k_map_server_centres) and of its render (k_map_render_rays, k_map_render_write) from
// morefusion_b200/csrc/mapping.cu (built by tests/test_mapping_render_emu.py with g++
// -DMF_HOST_EMU).  Same argument lists and launch sequences as the C ABI entry points
// (include/morefusion_b200.h), minus the stream.
#include "mapping_node_emu.cpp"

#include <string.h>

extern "C" int emu_map_integrate_server(const float* points, const int32_t* labels, int height,
                                        int width, const float* sensor_to_world, double max_range,
                                        const int32_t* lut, int lut_lo, int lut_n,
                                        const double* inst_resolution, int n_instances,
                                        int background, double background_resolution,
                                        int uncertain, uint32_t scan, float hit, float miss,
                                        float lo_min, float lo_max, void* centre_sums,
                                        uint32_t* centre_first, float* centres,
                                        int32_t* centre_set, void* cells, void* cnt,
                                        int64_t capacity, int32_t* counters,
                                        int32_t* tree_state, uint32_t* boxes) {
  MapTable t = tab(cells, cnt, capacity, counters);
  const long long n = (long long)height * width;
  ServerScanParams p;
  p.points = points; p.labels = labels; p.lut = lut; p.inst_res = inst_resolution;
  p.csum = (u64*)centre_sums; p.cfirst = centre_first;
  p.lut_lo = lut_lo; p.lut_n = lut_n; p.n = (int)n; p.width = width;
  p.bg = background; p.uncertain = uncertain;
  for (int a = 0; a < 12; ++a) p.m[a] = sensor_to_world[a];
  p.ox = sensor_to_world[3]; p.oy = sensor_to_world[7]; p.oz = sensor_to_world[11];
  p.max_range = max_range; p.res = background_resolution; p.scan = scan;
  p.hit = hit; p.miss = miss; p.lo_min = lo_min; p.lo_max = lo_max;
  run((unsigned)n, 1, [&] { k_map_server_trees(p, tree_state, boxes); });
  run((unsigned)n, 1, [&] { k_map_server_hits(p, t); });              // blockDim 1: lane 0 only
  run((unsigned)(n > n_instances ? n : n_instances), 1,
      [&] { k_map_server_boxes(p, n_instances, tree_state, boxes); });
  run((unsigned)n, 1, [&] { k_map_scan_free(p, t); });
  run((unsigned)n_instances, 1, [&] { k_map_server_centres(p, n_instances, centres, centre_set); });
  return 0;
}

extern "C" int emu_map_render(const float* points, int height, int width,
                              const float* sensor_to_world, float fx, float fy, float cx, float cy,
                              const int32_t* walk, const int32_t* walk_ids, int n_walk,
                              const double* inst_resolution, const uint32_t* boxes, int uncertain,
                              void* zbuf, int32_t* label, float* depth, void* cells, void* cnt,
                              int64_t capacity, int32_t* counters) {
  const long long n_even = (long long)((height + 1) / 2) * ((width + 1) / 2);
  memset(zbuf, 0xFF, (size_t)n_even * sizeof(u64));
  if (n_walk > 0) {
    RenderParams p;
    p.points = points; p.walk = walk; p.inst_res = inst_resolution; p.box = boxes;
    p.height = height; p.width = width; p.n_walk = n_walk;
    for (int a = 0; a < 12; ++a) p.m[a] = sensor_to_world[a];
    p.ox = sensor_to_world[3]; p.oy = sensor_to_world[7]; p.oz = sensor_to_world[11];
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy;
    MapTable t = tab(cells, cnt, capacity, counters);
    run((unsigned)(n_even * n_walk), 1, [&] { k_map_render_rays(p, t, (u64*)zbuf); });
  }
  run((unsigned)((long long)height * width), 1, [&] {
    k_map_render_write((const u64*)zbuf, walk_ids, height, width, uncertain, label, depth);
  });
  return 0;
}
