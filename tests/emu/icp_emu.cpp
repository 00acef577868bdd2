// TEST INFRASTRUCTURE: host execution of the per-thread helpers of morefusion_b200/csrc/icp.cu
// (built by tests/test_icp_emu.py with g++ -DMF_HOST_EMU -ffp-contract=off; the .cu is built with
// -fmad=false, so the results are the device's bit for bit).  horn_rotation and nearest are the
// code k_icp_run's thread runs per solve and per source point; cell_window is the search window
// nearest loops over.
#define MF_HOST_EMU 1

#include "../../morefusion_b200/csrc/icp.cu"

// R [n,3,3] of horn_rotation on C [n,3,3] (C[3 i + j] = sum (t_i - tm_i)(s_j - sm_j)).
extern "C" void emu_horn_rotation(const double* C, int n, double* R) {
  for (int i = 0; i < n; ++i) horn_rotation(C + 9 * (size_t)i, R + 9 * (size_t)i);
}

// (lo, hi) of cell_window per query coordinate: lohi [n,2].
extern "C" void emu_cell_window(const double* x, int n, double r, double origin, double h,
                                int32_t* lohi) {
  for (int i = 0; i < n; ++i) cell_window(x[i], r, origin, h, lohi + 2 * i, lohi + 2 * i + 1);
}

// nearest() of every query q [nq,3] over a cell list (points [nt,3] sorted by cell, cells [nt,3],
// index [nt], origin [3], cell_size): the sorted position (-1 without a match) and its d^2.
// r2 is passed apart from r, so that the strict d^2 < r2 test can be put on a chosen double.
extern "C" void emu_nearest(const double* q, int nq, const double* points, const int32_t* cells,
                            const int32_t* index, int nt, const double* origin, double cell_size,
                            double r, double r2, int32_t* pos, double* d2) {
  int32_t count = nt;
  mf_icp_target tg;
  tg.points = points;
  tg.cells = cells;
  tg.index = index;
  tg.count = &count;
  tg.origin = origin;
  tg.cell_size = cell_size;
  for (int i = 0; i < nq; ++i)
    pos[i] = nearest(q[3 * i], q[3 * i + 1], q[3 * i + 2], tg, nt, r, r2, d2 + i);
}
