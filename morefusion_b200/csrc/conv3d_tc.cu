// wgmma / TMA GEMM for sm_90a: the implicit-GEMM k4-s2 Conv3Ds (conv3, conv4) and the Conv1D
// heads of the singleview_3d pose model.
//
// Replaces the cuDNN ConvolutionND calls behind
//   morefusion/contrib/singleview_3d/models/model.py:73-74 (conv3, conv4), :77-91 (heads).
//
// out[m, n] = act( sum_k A(m,k) * W[n,k] + bias[n] )     bf16 operands, fp32 accumulation in registers.
//
// CTA tile 128 x BLOCK_N x 64, one CTA per SM, 384 threads:
//   warpgroup 0   (1 thread) TMA producer: per K block one box of A and one of W into a
//                 SWIZZLE_128B smem stage, mbarrier expect_tx / complete_tx
//   warpgroups 1-2           consumers: 4 x wgmma (m64 x BLOCK_N x k16) per stage on 64 rows each,
//                 one K block kept in flight, the stage released to the producer once its wgmma
//                 retired; then bias, ReLU and bf16 pack into a shared-memory staging buffer and
//                 TMA stores (row-major, or into the space-to-depth layout the next
//                 convolution's TMA boxes read); fp32 outputs are stored from the registers
// For the convolutions the A operand needs no im2col: with the space-to-depth input layout
// (cnn.cu) the 128 output voxels x 64 channels of one K block are ONE 5-D TMA box.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include "cnn.cuh"
#include "common.cuh"
#include "tc_ptx.cuh"

namespace mf {

constexpr int TC_BLOCK_M = 128;
constexpr int TC_BLOCK_K = 64;
constexpr int TC_A_BYTES = TC_BLOCK_M * TC_BLOCK_K * 2;   // 16 KiB

struct TcExtra {
  int kb_per_a;      // conv: K blocks per kernel-offset a (= Ci8 / 64)
  int kb_total;      // K blocks overall
  int kb_per_split;  // K blocks per split-K slice
  int splitk;
  float* ws;         // fp32 [splitk][M][N] partial sums when splitk > 1 (plain stores, no atomics)
  int* err;          // device error word (pipeline time-out), may be null
  int staged;        // bf16 outputs leave through the staging buffer and tmO (staged_epilogue)
};

// staging buffer of a consumer warpgroup: 64 rows x 128 columns bf16 (16 KB)
constexpr int TC_STG_COLS = 128, TC_STG_BYTES = 64 * TC_STG_COLS * 2;

constexpr int TC_MAX_GROUPS = 3;
// up to 3 same-shape GEMMs in one launch (the three pose heads): grid.z = group * splitk + split
struct TcArgs {
  CUtensorMap tmA[TC_MAX_GROUPS];
  CUtensorMap tmW[TC_MAX_GROUPS];
  CUtensorMap tmO[TC_MAX_GROUPS];   // staged: row-major 2-D {N, M} or s2d 5-D output map
  GemmParams p[TC_MAX_GROUPS];
  TcExtra e;
};

__device__ __forceinline__ long long out_row_offset(const GemmParams& p, int m) {
  if (p.out_mode != OUT_S2D_BF16) return (long long)m * p.ldo + p.col_off;
  int Do = p.Do, J = Do / 2 + 1;
  int ow = m % Do, oh = (m / Do) % Do, od = (m / (Do * Do)) % Do, b = m / (Do * Do * Do);
  int pd = od + 1, ph = oh + 1, pw = ow + 1;
  int r = ((pd & 1) << 2) | ((ph & 1) << 1) | (pw & 1);
  return ((((long long)b * J + (pd >> 1)) * J + (ph >> 1)) * J + (pw >> 1)) * (8LL * p.N) +
         (long long)r * p.N;
}

// ------------------------------------------------------------------ persistent kernel
// One CTA per SM loops over work units (group, m-tile, n-tile, k-split).  The shared-memory
// stage ring runs continuously across units, so the producer already streams the next unit's
// operands while the consumer warpgroups run the epilogue of the current one, and the per-CTA
// set-up (barrier init, descriptor prefetch, pipeline fill) is paid once per SM instead of once
// per tile -- which is what the short-K head GEMMs (2-16 K blocks per tile) are dominated by.
// With CTA pairs (CLUSTER = 2) a unit covers m-tiles 2 mt and 2 mt + 1, one per CTA of the pair,
// and m_tiles counts the pairs.
struct TcSched {
  int m_tiles, n_tiles, groups, splitk, n_units;
  long long* stamps;      // profiling hook (mf_gemm_bf16_tc_ex): clock64 per role per unit, CTA 0
  // stream-K (one group, splitk == 1): the units x K-blocks iteration space is cut into one
  // equal contiguous range per cluster, so every SM does the same number of K blocks whatever
  // the tile count (256 tiles on 132 SMs would otherwise leave 3 % of the machine idle in the
  // second wave, 64 tiles more than half of it).  A CTA whose range starts inside a tile stores
  // that segment's raw fp32 accumulator in its workspace slot and raises its flags; the CTA that
  // holds the tile's first K block owns the tile and adds the slots of the CTAs of its own rank
  // in the following clusters, in order, in its epilogue.
  int streamk;
  int* sk_flags;          // [gridDim.x][8] (one word per consumer warpgroup), zero between launches
  float* sk_ws;           // [gridDim.x][128 x BLOCK_N] fp32
};
#define TC_STAMP(slot)                                                        \
  do {                                                                        \
    if (sc.stamps && blockIdx.x == 0 && it < 16) sc.stamps[it * 8 + (slot)] = clock64(); \
  } while (0)

__device__ __forceinline__ void unit_decode(const TcSched& sc, int u, int& g, int& mt, int& nt,
                                            int& split) {
  split = u % sc.splitk;
  int r = u / sc.splitk;
  nt = r % sc.n_tiles;
  r /= sc.n_tiles;
  mt = r % sc.m_tiles;
  g = r / sc.m_tiles;
}

// One piece of work of a persistent CTA: K blocks [kb0, kb1) of unit u.
struct TcSeg {
  int u, kb0, kb1;
  int partial;            // stream-K: store the raw accumulator to this CTA's slot (not the output)
  int peer0, n_peers;     // stream-K owner: add the slots of the CTAs of its rank in clusters
                          // peer0 .. peer0 + n_peers - 1
};

// The schedule is dealt per cluster (cid of nc): both CTAs of a pair walk the same units and K
// ranges, each on its own m-tile.
struct TcSegIter {
  long long pos, hi, W;   // stream-K: position in the tiles x K-blocks space
  int u;                  // otherwise: next unit
  int cid, nc;
  __device__ __forceinline__ long long lo_of(int c) const { return W * c / nc; }
  __device__ __forceinline__ TcSegIter(const TcSched& sc, int kb_total, int cid_, int nc_)
      : cid(cid_), nc(nc_) {
    W = (long long)sc.n_units * kb_total;
    pos = sc.streamk ? lo_of(cid) : 0;
    hi = sc.streamk ? lo_of(cid + 1) : 0;
    u = cid;
  }
  __device__ __forceinline__ bool next(const TcSched& sc, const TcExtra& e, TcSeg& s) {
    s.partial = 0; s.peer0 = 0; s.n_peers = 0;
    if (sc.streamk) {
      if (pos >= hi) return false;
      const int t = (int)(pos / e.kb_total);
      const int k0 = (int)(pos - (long long)t * e.kb_total);
      const long long room = hi - pos;
      const int k1 = room < (long long)(e.kb_total - k0) ? k0 + (int)room : e.kb_total;
      s.u = t; s.kb0 = k0; s.kb1 = k1;
      s.partial = k0 != 0;
      if (k0 == 0 && k1 < e.kb_total) {
        const long long tile_end = (long long)(t + 1) * e.kb_total;
        s.peer0 = cid + 1;
        int c = s.peer0;
        while (c < nc && lo_of(c) < tile_end) ++c;
        s.n_peers = c - s.peer0;
      }
      pos += k1 - k0;
      return true;
    }
    if (u >= sc.n_units) return false;
    const int split = u % sc.splitk;
    s.u = u;
    s.kb0 = split * e.kb_per_split;
    s.kb1 = min(s.kb0 + e.kb_per_split, e.kb_total);
    u += nc;
    return true;
  }
};


// Warpgroup 0 produces (one thread issues the TMA loads), warpgroups 1 and 2 consume: each runs
// wgmma on 64 of the tile's 128 rows (m64 x BLOCK_N x k16, fp32 accumulators in registers) and
// then its own epilogue from those registers (staged_epilogue for bf16 outputs).
constexpr int TC_P_THREADS = 384;
// register split between the roles (setmaxnreg): 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;

// wgmma accumulator fragment of thread t of a consumer warpgroup: rows r0 = 16 (t / 32) + (t % 32) / 4
// and r0 + 8 of the warpgroup's 64, columns 8 j + 2 (t % 4) + {0, 1} in d[4 j + 2 i + {0, 1}]
// (i = 0 for row r0, 1 for r0 + 8).

// ------------------------------------------------------------------ staged bf16 epilogue
// A consumer warpgroup's 64 x BN bf16 tile goes from the accumulator fragment through its 16 KB
// staging buffer (HC = 128 columns per pass: two 64-column slices of 8 KB) to global memory by
// TMA stores that one thread issues; the warpgroup goes back to wgmma while they drain.  Inside a
// slice the layout is SW128: column c of a 128-byte box row `row` sits at row x 128 +
// ((c / 8) ^ key) x 16 + (c % 8) x 2, key = row % 8.  Where a fragment row lands in the slice and
// which TMA stores take the slice out is the box policy's:
//   row(k, off, key)   byte offset in the slice and SW128 key of the row the thread writes with
//                      store k (0, 1) of a column group: fragment row r0 + 8 (k ^ swap), swap = 1
//                      only when kSwap and the thread's r0 is odd
//   store(slice, c0)   the stores of the slice holding output columns [c0, c0 + 64)

// A row-major output (2-D map {N, M} at out + col_off, row pitch ldo, 64 x 64 boxes): fragment
// row r is row r of the slice's one box.  The 8 row groups of a store are 8 consecutive rows, 8
// distinct keys: no bank conflict.
struct StgRowMajor {
  static constexpr bool kSwap = false;
  const CUtensorMap* tm;
  int m0;                       // the warpgroup's first output row
  __device__ __forceinline__ void row(int k, uint32_t& off, uint32_t& key) const {
    const int r = (threadIdx.x >> 5 & 3) * 16 + (threadIdx.x & 31) / 4 + 8 * k;
    off = (uint32_t)r * 128;
    key = (uint32_t)r & 7;
  }
  __device__ __forceinline__ void store(uint32_t slice, int c0) const { tma_store_2d(tm, slice, c0, m0); }
};

// conv3's output scattered into the s2d layout of conv4's input x4 [B][J][J][J][8 N], J = 9:
// padded coordinate p = o + 1 of an output voxel lands in cell p / 2 at parity slot
// s = 4 (pd % 2) + 2 (ph % 2) + pw % 2, channels [s N, s N + N).  A warpgroup's 64 rows are 4 oh
// (oh0 = 4 i) x 16 ow at one od, so per (ph % 2, pw % 2) they fill 2 consecutive jh x 8
// consecutive jw cells: one box {64 channels, 8 jw, 2 jh, 1, 1} (2 KB) of a 5-D map over x4.  A
// slice holds the 4 boxes, box (ph % 2, pw % 2) at (2 (ph % 2) + pw % 2) x 2 KB; fragment row
// r = 16 oh_l + ow is row 8 (oh_l / 2) + ow / 2 of box (1 - oh_l % 2, 1 - ow % 2).  The zero ring
// of x4 (p = 0 and p = 17) lies outside every box and is never written.
// The row groups of one store are ow = 0..7 (or 8..15): even and odd ow land in two boxes at the
// same keys ow / 2, a 2-way bank conflict.  So the threads of odd ow swap their two rows (kSwap):
// store 0 writes ow = 0, 2, 4, 6 (keys 0-3) and 9, 11, 13, 15 (keys 4-7), store 1 the others.
struct StgS2D {
  static constexpr bool kSwap = true;
  const CUtensorMap* tm;
  int N;                        // channels per parity slot
  int s_d, jh0, jd, b;          // pd % 2 (as slot bit 4), first jh of parity ph % 2 = 1, jd, batch
  // Do = 16: m0 is the warpgroup's first output row (a multiple of 64)
  __device__ __forceinline__ StgS2D(const CUtensorMap* tm_, int N_, int m0) : tm(tm_), N(N_) {
    const int oh0 = (m0 >> 4) & 15, pd = ((m0 >> 8) & 15) + 1;
    s_d = (pd & 1) << 2;
    jh0 = oh0 >> 1;
    jd = pd >> 1;
    b = m0 >> 12;
  }
  __device__ __forceinline__ void row(int k, uint32_t& off, uint32_t& key) const {
    const int oh_l = threadIdx.x >> 5 & 3, ow0 = (threadIdx.x & 31) / 4;
    const int ow = ow0 + 8 * (k ^ (ow0 & 1));
    const int box = 2 * (1 - (oh_l & 1)) + 1 - (ow & 1);
    const int r = 8 * (oh_l >> 1) + (ow >> 1);
    off = (uint32_t)(box * 2048 + r * 128);
    key = (uint32_t)r & 7;
  }
  __device__ __forceinline__ void store(uint32_t slice, int c0) const {
    if (c0 >= N) return;        // a tile wider than the slot
#pragma unroll
    for (int box = 0; box < 4; ++box) {
      const int sh = box >> 1, sw = box & 1;   // ph % 2, pw % 2
      tma_store_5d(tm, slice + box * 2048, (s_d | sh << 1 | sw) * N + c0, 1 - sw, jh0 + 1 - sh, jd, b);
    }
  }
};

// Bias, ReLU (folded into cvt.rn.relu) and bf16 of the warpgroup's accumulators d (fragment as
// above, columns n0 ..), staged H = min(BN, HC) columns per pass.  Thread 0 of the warpgroup
// waits before a pass until the stores of the previous pass have read the buffer: `first_wait()`
// before the first pass (it may do more, as the heads' publish does), bulk_wait_read0 before the
// others; it calls `written()` once the last pass is in shared memory, then issues that pass's
// stores.  The stores of the last pass are left in flight (one bulk group per pass).
template <int BN, int HC, class Boxes, class FirstWait, class Written>
__device__ __forceinline__ void staged_epilogue(const float (&d)[BN / 2], uint32_t stg, int n0, int pN,
                                                const float* pbias, int prelu, const Boxes& boxes,
                                                FirstWait first_wait, Written written) {
  constexpr int H = BN < HC ? BN : HC;        // columns per staging pass
  const int lane = threadIdx.x & 31, t = threadIdx.x & 127, wg = (threadIdx.x >> 7) - 1;
  const int cq = 2 * (lane & 3);
  const bool swap = Boxes::kSwap && ((lane >> 2) & 1);
  uint32_t off0, key0, off1, key1;
  boxes.row(0, off0, key0);
  boxes.row(1, off1, key1);
  const uint32_t at0 = stg + off0 + cq * 2, at1 = stg + off1 + cq * 2;
  // one loop over the fragment's column groups j (fully unrolled, so d[] stays in registers); a
  // staging pass starts every H / 8 of them
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int jj = j % (H / 8);
    if (jj == 0) {
      if (t == 0) {
        if (j == 0) first_wait();
        else bulk_wait_read0();        // the staging buffer's previous stores have read it
      }
      wg_bar(1 + wg);
    }
    const int n = n0 + 8 * j + cq;
    const bool in = n < pN;
    const float b0 = (pbias && in) ? __ldg(pbias + n) : 0.f, b1 = (pbias && in) ? __ldg(pbias + n + 1) : 0.f;
    uint32_t v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float x0 = d[4 * j + 2 * i] + b0, x1 = d[4 * j + 2 * i + 1] + b1;
      v[i] = prelu ? pack_bf16x2_relu(x0, x1) : pack_bf16x2(x0, x1);
    }
    if (Boxes::kSwap) {
      const uint32_t v0 = swap ? v[1] : v[0], v1 = swap ? v[0] : v[1];
      v[0] = v0;
      v[1] = v1;
    }
    const uint32_t sl = (uint32_t)(jj >> 3) * 8192, c = (uint32_t)jj & 7;
    sts_b32(at0 + sl + ((c ^ key0) << 4), v[0]);
    sts_b32(at1 + sl + ((c ^ key1) << 4), v[1]);
    if (jj == H / 8 - 1) {
      fence_proxy_async_smem();
      wg_bar(1 + wg);
      if (t == 0) {
        if (j == BN / 8 - 1) written();
        const int c0 = n0 + (j / (H / 8)) * H;
#pragma unroll
        for (int s = 0; s < H / 64; ++s) boxes.store(stg + s * 8192, c0 + 64 * s);
        bulk_commit();
      }
    }
  }
}

// Wait until the stream-K peers of this warpgroup have parked their partial sums (their flag
// words are `stride` ints apart)
__device__ __forceinline__ void sk_wait_peers(const int* flags, int n_peers, int stride, int* err) {
  for (int pi = 0; pi < n_peers; ++pi) {
    int v = 0;
    for (long long spin = 0; spin < (1LL << 24); ++spin) {
      asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(flags + pi * stride) : "memory");
      if (v) break;
      __nanosleep(64);
    }
    if (!v && err) atomicExch(err, 7);
  }
}

// CLUSTER = 2 (the convolutions): the two CTAs of a cluster take m-tiles 2 mt and 2 mt + 1 of the
// same n-tile and K range, so they need the same W tile: each producer loads its own A box and
// half of W (rows rank x BLOCK_N / 2 ..), multicast into the same stage of both CTAs.  A stage is
// then written by both producers, so its empty barrier counts the consumer warpgroups of both
// CTAs, and each consumer warpgroup releases the stage in its own CTA and in its peer.
template <int BLOCK_N, int STAGES, int CLUSTER>
__global__ void __launch_bounds__(TC_P_THREADS, 1)
k_gemm_tc_persistent(const __grid_constant__ TcArgs args, const TcSched sc) {
  static_assert(CLUSTER == 1 || CLUSTER == 2, "CTA pairs at most");
  constexpr int B_BYTES = BLOCK_N * TC_BLOCK_K * 2;
  constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
  constexpr int NR = BLOCK_N / 2;                 // accumulators per consumer thread
  extern __shared__ unsigned char smem_dyn[];
  // SWIZZLE_128B operands need 1024-byte alignment
  unsigned char* smem = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[STAGES];
  __shared__ uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TcExtra& e = args.e;
  const int crank = CLUSTER == 1 ? 0 : (int)cluster_ctarank();
  const int cid = blockIdx.x / CLUSTER, nc = gridDim.x / CLUSTER;

  if (threadIdx.x == 0) {
    for (int g = 0; g < sc.groups; ++g) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmA[g])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmW[g])) : "memory");
      if (e.staged)
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmO[g])) : "memory");
    }
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CLUSTER);  // one arrival per consumer warpgroup of the cluster
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the peer multicasts into this CTA's stages and arrives on its barriers: both inits first
  if constexpr (CLUSTER == 1) __syncthreads();
  else cluster_sync();

  if (warp < 4) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (threadIdx.x != 0) {
      if constexpr (CLUSTER > 1) cluster_sync();
      return;
    }
    // ===== TMA producer
    int kc = 0;                                        // K blocks issued so far (ring position)
    int it = 0;
    TcSegIter iter(sc, e.kb_total, cid, nc);
    TcSeg seg;
    for (; iter.next(sc, e, seg); ++it) {
      int g, mt, nt, split;
      unit_decode(sc, seg.u, g, mt, nt, split);
      mt = mt * CLUSTER + crank;
      const GemmParams& p = args.p[g];
      TC_STAMP(0);
      const int m0 = mt * TC_BLOCK_M, n0 = nt * BLOCK_N;
      int cb = 0, cw = 0, ch = 0, cd = 0;
      if (p.mode == GEMM_CONV_S2D) {
        int Do = p.Do;
        cw = m0 % Do;                       // 0 for Do in {8,16}: tiles start at ow = 0
        ch = (m0 / Do) % Do;
        cd = (m0 / (Do * Do)) % Do;
        cb = m0 / (Do * Do * Do);
      }
      for (int kb = seg.kb0; kb < seg.kb1; ++kb, ++kc) {
        const int s = kc % STAGES;
        const uint32_t ph = (kc / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1, e.err, 1, 64);
        mbar_expect_tx(&full_bar[s], STAGE_BYTES);
        unsigned char* sa = smem + (size_t)s * STAGE_BYTES;
        unsigned char* sb = sa + TC_A_BYTES;
        int wk = kb * TC_BLOCK_K;                      // W column of the K block
        if (p.mode == GEMM_CONV_S2D) {
          // the 128 output voxels x 64 channels of one K block are ONE 5-D box.  K is walked
          // channel block by channel block with the 8 cell offsets a innermost, so the 8
          // overlapping boxes of a channel block are read back to back while they are in L2.
          const int a = kb & 7, c = (kb >> 3) * TC_BLOCK_K;
          wk = a * e.kb_per_a * TC_BLOCK_K + c;
          tma_load_5d(sa, &args.tmA[g], &full_bar[s], c, cw + (a & 1), ch + ((a >> 1) & 1),
                      cd + ((a >> 2) & 1), cb);
        } else {
          tma_load_2d(sa, &args.tmA[g], &full_bar[s], wk, m0);
        }
        if constexpr (CLUSTER == 1) {
          tma_load_2d(sb, &args.tmW[g], &full_bar[s], wk, n0);
        } else {
          // rows [crank x BLOCK_N / 2, + BLOCK_N / 2) of the W tile, at their offset in the
          // K-major SW128 layout (1024 B per 8 rows), into this stage of both CTAs
          tma_load_2d_multicast(sb + crank * (B_BYTES / 2), &args.tmW[g], &full_bar[s], wk,
                                n0 + crank * (BLOCK_N / 2), (uint16_t)0x3);
        }
      }
      TC_STAMP(1);
    }
    if constexpr (CLUSTER > 1) cluster_sync();
    return;
  }

  // ===== consumers: wgmma main loop, then the epilogue of the warpgroup's 64 rows
  setmaxnreg_inc<TC_CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1, t = threadIdx.x & 127;
  const int r0 = (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
  const bool stamper = wg == 0 && t == 0;
  const uint32_t stg = smem_u32(smem) + STAGES * STAGE_BYTES + wg * TC_STG_BYTES;
  constexpr long long SLOT_FLOATS = (long long)TC_BLOCK_M * BLOCK_N;
  // a stage is free again for the producers that write it: this CTA's, and the peer's (its half
  // of W)
  auto release = [&](int s) {
    mbar_arrive(&empty_bar[s]);
    if constexpr (CLUSTER > 1) mbar_arrive_cluster(&empty_bar[s], crank ^ 1);
  };
  int kc = 0, it = 0;
  TcSegIter iter(sc, e.kb_total, cid, nc);
  TcSeg seg;
  for (; iter.next(sc, e, seg); ++it) {
    int g, mt, nt, split;
    unit_decode(sc, seg.u, g, mt, nt, split);
    mt = mt * CLUSTER + crank;
    if (stamper) TC_STAMP(2);
    float d[NR];
    int prev = -1;
    for (int kb = seg.kb0; kb < seg.kb1; ++kb, ++kc) {
      const int s = kc % STAGES;
      mbar_wait(&full_bar[s], (kc / STAGES) & 1, e.err, 2, 20);
      if (stamper && kb == seg.kb0) TC_STAMP(3);
      const uint32_t sa = smem_u32(smem + (size_t)s * STAGE_BYTES);
      fence_regs(d);
      wgmma_fence();
      wgmma_kblock<BLOCK_N, 0, 0>(d, make_sw128_desc(sa + wg * 8192), make_sw128_desc(sa + TC_A_BYTES),
                                  kb == seg.kb0);
      wgmma_commit();
      fence_regs(d);
      // keep one K block in flight: the stage of the previous one is free once it retired
      wgmma_wait<1>();
      if (prev >= 0 && t == 0) release(prev);
      prev = s;
    }
    wgmma_wait<0>();
    fence_regs(d);
    if (t == 0) release(prev);
    if (stamper) TC_STAMP(4);

    const GemmParams& p = args.p[g];
    const int m0 = mt * TC_BLOCK_M + wg * 64, n0 = nt * BLOCK_N;
    if (seg.partial) {
      // stream-K: this CTA holds a later K range of a tile another CTA owns.  Slot layout is
      // register-major / thread-minor, so every warp access is 256 contiguous bytes.
      float2* slot = reinterpret_cast<float2*>(sc.sk_ws + (long long)blockIdx.x * SLOT_FLOATS +
                                               (long long)wg * 64 * BLOCK_N);
#pragma unroll
      for (int i = 0; i < NR / 2; ++i) slot[i * 128 + t] = make_float2(d[2 * i], d[2 * i + 1]);
      __threadfence();
      wg_bar(1 + wg);
      if (t == 0)
        asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(sc.sk_flags + blockIdx.x * 8 + wg),
                     "r"(1) : "memory");
      if (stamper) { TC_STAMP(5); TC_STAMP(6); TC_STAMP(7); }
      continue;
    }
    if (seg.n_peers > 0) {
      // the peers ran these K blocks at the START of their range, this CTA reaches the tile at
      // the END of its own: normally no wait.  Peer pi is the CTA of this rank in cluster
      // peer0 + pi.
      const int peer_cta0 = seg.peer0 * CLUSTER + crank;
      if (t == 0) sk_wait_peers(sc.sk_flags + peer_cta0 * 8 + wg, seg.n_peers, 8 * CLUSTER, e.err);
      wg_bar(1 + wg);
      for (int pi = 0; pi < seg.n_peers; ++pi) {
        const float2* ps = reinterpret_cast<const float2*>(
            sc.sk_ws + (long long)(peer_cta0 + pi * CLUSTER) * SLOT_FLOATS + (long long)wg * 64 * BLOCK_N);
#pragma unroll
        for (int i = 0; i < NR / 2; ++i) {
          const float2 a = __ldcg(ps + i * 128 + t);
          d[2 * i] += a.x;
          d[2 * i + 1] += a.y;
        }
      }
      wg_bar(1 + wg);
      if (t == 0)                 // slots consumed: re-arm the flags for the next launch
        for (int pi = 0; pi < seg.n_peers; ++pi) sc.sk_flags[(peer_cta0 + pi * CLUSTER) * 8 + wg] = 0;
    }
    if (stamper) TC_STAMP(5);
    if (e.staged) {
      // through shared memory and TMA stores, left draining under the next segment's main loop
      auto first_wait = [] { bulk_wait_read0(); };
      auto written = [&] { if (stamper) TC_STAMP(6); };
      if (p.out_mode == OUT_S2D_BF16)
        staged_epilogue<BLOCK_N, TC_STG_COLS>(d, stg, n0, p.N, p.bias, p.relu, StgS2D(&args.tmO[g], p.N, m0),
                                              first_wait, written);
      else
        staged_epilogue<BLOCK_N, TC_STG_COLS>(d, stg, n0, p.N, p.bias, p.relu, StgRowMajor{&args.tmO[g], m0},
                                              first_wait, written);
      if (stamper) TC_STAMP(7);
      continue;
    }
    const int pN = p.N, pM = p.M, prelu = p.relu, pmode = p.out_mode;
    const float* pbias = p.bias;
    void* pout = p.out;
    const int ma = m0 + r0, mb = ma + 8;
    const long long roa = ma < pM ? out_row_offset(p, ma) : 0, rob = mb < pM ? out_row_offset(p, mb) : 0;
#pragma unroll
    for (int j = 0; j < NR / 4; ++j) {
      const int n = n0 + 8 * j + cq;
      if (n >= pN) continue;
      const bool has1 = n + 1 < pN;
      const float b0 = pbias ? __ldg(pbias + n) : 0.f, b1 = (pbias && has1) ? __ldg(pbias + n + 1) : 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int m = i ? mb : ma;
        if (m >= pM) continue;
        const long long ro = i ? rob : roa;
        float x0 = d[4 * j + 2 * i], x1 = d[4 * j + 2 * i + 1];
        if (pN & 31) {
          // ragged N (small-N heads, fp32 row-major output only; enforced on the host): rows
          // are not 8-byte aligned, scalar stores
          float* dst = reinterpret_cast<float*>(pout) + ro + n;
          x0 += b0;
          dst[0] = prelu ? fmaxf(x0, 0.f) : x0;
          if (has1) {
            x1 += b1;
            dst[1] = prelu ? fmaxf(x1, 0.f) : x1;
          }
          continue;
        }
        if (e.splitk > 1) {
          *reinterpret_cast<float2*>(e.ws + ((long long)split * pM + m) * pN + n) = make_float2(x0, x1);
          continue;
        }
        x0 += b0;
        x1 += b1;
        if (pmode == OUT_F32) {
          if (prelu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(pout) + ro + n) = make_float2(x0, x1);
        } else {        // ReLU folded into the conversion (cvt.rn.relu)
          *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(pout) + ro + n) =
              prelu ? pack_bf16x2_relu(x0, x1) : pack_bf16x2(x0, x1);
        }
      }
    }
    if (stamper) { TC_STAMP(6); TC_STAMP(7); }
  }
  if (e.staged && t == 0) bulk_wait_read0();   // the staging buffer is read before the CTA leaves
  // no CTA leaves while its peer may still multicast into it or arrive on its barriers
  if constexpr (CLUSTER > 1) cluster_sync();
}

// ------------------------------------------------------------------ the pose heads as ONE launch
// Layers 1-3 of the three heads (model.py:239-254: head1 = the three first layers side by side,
// 3 x conv2_*, 3 x conv3_*) are 7 GEMMs whose only coupling is per 128-row tile: a layer-2 tile
// needs the layer-1 tiles of its rows, a layer-3 tile the layer-2 tile of its head and rows.  As
// separate launches each layer ends in a partially filled wave plus a launch gap.  Here all their
// tiles are ONE unit list of a persistent kernel.  Layer 1 (N = 1920 = 7 x 256 + 128) is listed
// as two GEMMs, 256-wide tiles and one 128-wide tile, so no MMA work is spent on empty columns;
// that makes 8 entries.
//
// CTA pairs: a unit is (GEMM, m-tile pair, n-tile); the two CTAs of a cluster take m-tiles 2 i
// and 2 i + 1 and need the same W tile, so each producer loads its own A box and half of the W
// rows, multicast into the same stage of both CTAs (as k_gemm_tc_persistent<..., 2>).  An odd
// m-tile count is padded to an even one: the extra tile lies wholly past M, its A boxes are zero
// filled by TMA, its stores are clipped by TMA, and it neither waits on nor bumps a counter.
//
// Dependencies: a unit's producer waits for a global arrival counter of its own input m-tile
// before its first A load; each consumer warpgroup bumps the counter of its output m-tile once its
// TMA stores are complete.  Counters are never reset: every launch reads an epoch word at start
// (thresholds = (epoch + 1) x arrivals per launch) and the last CTA to finish bumps it, so
// CUDA-graph replays need no memset.
//
// Why there is no deadlock: every cluster is resident at once (the grid is at most the number of
// co-resident pairs), both CTAs of a pair walk the same units in list order, and a unit only
// waits for units earlier in the list.  A warpgroup may hold back the signal of its last tile
// while it runs the main loop of the next unit (so the wait for the stores to complete overlaps
// MMA work), but only when that next unit is a layer-1 unit, which waits on nothing; before any
// unit that has a dependency it publishes first.  So the earliest unfinished unit of the list
// always has its inputs published, its stage ring drained by earlier units of its own cluster,
// and can finish.
constexpr int HD_GEMMS = 8;
struct HeadsArgs {
  CUtensorMap tmA[HD_GEMMS];
  CUtensorMap tmW[HD_GEMMS];    // box rows: half the N tile (one half per CTA of the pair)
  CUtensorMap tmO[HD_GEMMS];    // bf16 output, 64 x 64 boxes, SWIZZLE_128B
  const float* bias[HD_GEMMS];
  int N[HD_GEMMS];
  int relu[HD_GEMMS];
  int bn[HD_GEMMS];             // N tile: 256 or 128
  int kb[HD_GEMMS];             // K blocks
  int n_tiles[HD_GEMMS];
  int unit_begin[HD_GEMMS + 1];
  int dep_base[HD_GEMMS];       // counter (per m tile) to wait on, -1 = none
  int dep_target[HD_GEMMS];     // its arrivals per launch
  int sig_base[HD_GEMMS];       // counter (per m tile) to bump, -1 = none
  int m_tiles, n_units;
  int* sync;                    // [0] epoch, [1] finished CTAs, [16 ..] counters
  int* err;
};

// unit u -> GEMM q, m-tile pair mp, n-tile nt
__device__ __forceinline__ void hd_decode(const HeadsArgs& a, int u, int& q, int& mp, int& nt) {
  q = 0;
#pragma unroll
  for (int i = 1; i < HD_GEMMS; ++i) q += (u >= a.unit_begin[i]) ? 1 : 0;
  const int r = u - a.unit_begin[q];
  nt = r % a.n_tiles[q];
  mp = r / a.n_tiles[q];
}

// this warpgroup's stores of its last tile are complete: publish the tile to its consumers
// (their producers acquire the counter, then fence.proxy.async before reading it through TMA)
__device__ __forceinline__ void hd_publish(const HeadsArgs& a, int counter) {
  bulk_wait0();
  asm volatile("fence.proxy.async;" ::: "memory");
  __threadfence();
  atomicAdd(a.sync + 16 + counter, 1);
}

// One unit on a consumer warpgroup: main loop over the GEMM's K blocks, then the bf16 epilogue of
// the warpgroup's 64 rows through its staging buffer (64 x HC, two or four 64 x 64 SW128 boxes)
// and TMA stores, HC columns at a time.  One instantiation per N tile width, so each has its own
// accumulator registers.  `pending` (thread 0 only): counter of an earlier tile whose signal was
// held back (-1: none); published here once this unit's main loop is done.  Only u stays live
// across the main loop (the unit is decoded again after it): the 128 accumulators leave few
// registers under the 168 a 384-thread CTA may use.
template <int BN, int STAGES, int HC>
__device__ __forceinline__ void heads_unit(const HeadsArgs& args, uint32_t smem, uint32_t stg,
                                           uint64_t* full_bar, uint64_t* empty_bar, uint32_t peer_empty,
                                           int u, int crank, int& kc, int& pending) {
  constexpr int STAGE_BYTES = TC_A_BYTES + 256 * TC_BLOCK_K * 2;
  const int wg = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  int q, mp, nt;
  hd_decode(args, u, q, mp, nt);
  const int kbn = args.kb[q];
  // a stage is free again for both producers that write it: this CTA's and the peer's
  // (`peer_empty`: the peer's empty_bar[0] in the cluster window)
  auto release = [&](int s) {
    mbar_arrive(&empty_bar[s]);
    mbar_arrive_remote(peer_empty + 8 * s);
  };
  // defined before the first (non-accumulating) wgmma: left undefined, ptxas kept the two tile
  // widths' accumulators live across each other's units and spilled them
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  int prev = -1;
  for (int kb = 0; kb < kbn; ++kb, ++kc) {
    const int s = kc % STAGES;
    mbar_wait(&full_bar[s], (kc / STAGES) & 1, args.err, 2, 20);
    const uint32_t sa = smem + s * STAGE_BYTES;
    fence_regs(d);
    wgmma_fence();
    wgmma_kblock<BN, 0, 0>(d, make_sw128_desc(sa + wg * 8192), make_sw128_desc(sa + TC_A_BYTES), kb == 0);
    wgmma_commit();
    fence_regs(d);
    wgmma_wait<1>();
    if (prev >= 0 && t == 0) release(prev);
    prev = s;
  }
  wgmma_wait<0>();
  fence_regs(d);
  if (t == 0) release(prev);

  hd_decode(args, u, q, mp, nt);
  const float* pbias = args.bias[q];
  const int pN = args.N[q], prelu = args.relu[q];
  const int m0 = (2 * mp + crank) * TC_BLOCK_M + wg * 64, n0 = nt * BN;
  // before the first pass: publish the tile whose signal was held back, or wait for the staging
  // buffer's previous stores to have read it
  auto first_wait = [&] {
    if (pending >= 0) { hd_publish(args, pending); pending = -1; }
    else bulk_wait_read0();
  };
  staged_epilogue<BN, HC>(d, stg, n0, pN, pbias, prelu, StgRowMajor{&args.tmO[q], m0}, first_wait, [] {});
}

template <int STAGES, int HC>
__global__ void __launch_bounds__(TC_P_THREADS, 1)
k_heads_tc(const __grid_constant__ HeadsArgs args) {
  constexpr int STAGE_BYTES = TC_A_BYTES + 256 * TC_BLOCK_K * 2;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[STAGES];
  __shared__ uint64_t empty_bar[STAGES];
  __shared__ int epoch_slot;

  const int warp = threadIdx.x >> 5;
  const int crank = (int)cluster_ctarank();
  const int cid = blockIdx.x >> 1, nc = gridDim.x >> 1;
  if (threadIdx.x == 0) {
    int ep;
    asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(ep) : "l"(args.sync) : "memory");
    epoch_slot = ep;
#pragma unroll
    for (int q = 0; q < HD_GEMMS; ++q) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmA[q])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmW[q])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&args.tmO[q])) : "memory");
    }
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);   // one arrival per consumer warpgroup of the pair
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the peer multicasts into this CTA's stages and arrives on its barriers: both inits first
  cluster_sync();
  const unsigned epoch1 = (unsigned)epoch_slot + 1u;

  if (warp < 4) {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ===== TMA producer
      int kc = 0;
      for (int u = cid; u < args.n_units; u += nc) {
        int q, mp, nt;
        hd_decode(args, u, q, mp, nt);
        const int mt = 2 * mp + crank;
        if (args.dep_base[q] >= 0 && mt < args.m_tiles) {
          // input rows of this tile are written by earlier units (other SMs, TMA stores)
          const int* c = args.sync + 16 + args.dep_base[q] + mt;
          const unsigned target = epoch1 * (unsigned)args.dep_target[q];
          long long t0 = clock64();
          for (;;) {
            int v;
            asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(c) : "memory");
            if ((int)((unsigned)v - target) >= 0) break;
            __nanosleep(100);
            if (clock64() - t0 > 4000000000LL) {
              if (args.err) atomicExch(args.err, 9);
              __threadfence_system();
              __trap();
            }
          }
          // order the acquired (generic-proxy) view before this thread's async-proxy (TMA) reads
          asm volatile("fence.proxy.async;" ::: "memory");
        }
        const int bn = args.bn[q], wrows = bn / 2;
        const int m0 = mt * TC_BLOCK_M, n0 = nt * bn;
        const uint32_t bytes = (uint32_t)(TC_A_BYTES + bn * TC_BLOCK_K * 2);
        const int kbn = args.kb[q];
        for (int kb = 0; kb < kbn; ++kb, ++kc) {
          const int s = kc % STAGES;
          const uint32_t ph = (kc / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1, args.err, 1, 64);
          mbar_expect_tx(&full_bar[s], bytes);
          unsigned char* sa = smem + (size_t)s * STAGE_BYTES;
          tma_load_2d(sa, &args.tmA[q], &full_bar[s], kb * TC_BLOCK_K, m0);
          // W rows [crank x bn / 2, + bn / 2) of the tile, at their offset in the K-major SW128
          // layout (1024 B per 8 rows), into this stage of both CTAs
          tma_load_2d_multicast(sa + TC_A_BYTES + crank * wrows * 128, &args.tmW[q], &full_bar[s],
                                kb * TC_BLOCK_K, n0 + crank * wrows, (uint16_t)0x3);
        }
      }
    }
  } else {
    // ===== consumers: wgmma on 64 rows each, epilogue through shared memory and TMA stores
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = (warp >> 2) - 1;
    const bool lead = (threadIdx.x & 127) == 0;
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t stg = smem_base + STAGES * STAGE_BYTES + wg * (64 * HC * 2);
    const uint32_t peer_empty = mapa_shared(smem_u32(empty_bar), crank ^ 1);
    int kc = 0;
    int pending = -1;
    for (int u = cid; u < args.n_units; u += nc) {
      int q, mp, nt;
      hd_decode(args, u, q, mp, nt);
      // a unit that waits on other tiles must not run behind an unpublished tile (see above)
      if (lead && pending >= 0 && args.dep_base[q] >= 0) { hd_publish(args, pending); pending = -1; }
      if (args.bn[q] == 256)
        heads_unit<256, STAGES, HC>(args, smem_base, stg, full_bar, empty_bar, peer_empty, u, crank, kc, pending);
      else
        heads_unit<128, STAGES, HC>(args, smem_base, stg, full_bar, empty_bar, peer_empty, u, crank, kc, pending);
      hd_decode(args, u, q, mp, nt);
      const int mt = 2 * mp + crank;
      if (lead && args.sig_base[q] >= 0 && mt < args.m_tiles) pending = args.sig_base[q] + mt;
    }
    if (lead) {
      if (pending >= 0) hd_publish(args, pending);
      else bulk_wait_read0();          // the staging buffer is read before the CTA leaves
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int d = atomicAdd(args.sync + 1, 1);
    if (d == (int)gridDim.x - 1) {          // last CTA: next launch gets the next epoch
      args.sync[1] = 0;
      __threadfence();
      atomicAdd(args.sync, 1);
    }
  }
  // no CTA leaves while its peer may still multicast into it or arrive on its barriers
  cluster_sync();
}

// split-K epilogue: sum the slices, bias + activation + layout; 4 columns per thread
__global__ void k_splitk_finish(const float* __restrict__ ws, GemmParams p, int splitk) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long MN = (long long)p.M * p.N;
  if (i * 4 >= MN) return;
  int m = (int)((i * 4) / p.N), n = (int)((i * 4) % p.N);   // N % 32 == 0
  float4 v = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + n)) : make_float4(0, 0, 0, 0);
  for (int s = 0; s < splitk; ++s) {
    float4 a = __ldcs(reinterpret_cast<const float4*>(ws + s * MN) + i);
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
  }
  if (p.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
  long long off = out_row_offset(p, m) + n;
  if (p.out_mode == OUT_F32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off) = v;
  } else {
    __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(p.out) + off) = u;
  }
}

// ------------------------------------------------------------------ host: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

static int encode(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims,
                  const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  PFN_encodeTiled fn = get_encode();
  if (!fn) return MF_E_UNSUPPORTED;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                  dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MF_OK : MF_E_BADARG;
}

// the stage ring, the two consumer warpgroups' staging buffers and 1 KB for the alignment:
// 4 x 48 KB or 6 x 32 KB, + 32 KB + 1 KB = 225 KB of the 227 KB a block may use
template <int BLOCK_N, int STAGES>
static constexpr int persistent_smem() {
  return STAGES * (TC_A_BYTES + BLOCK_N * TC_BLOCK_K * 2) + 2 * TC_STG_BYTES + 1024;
}

template <int BLOCK_N, int STAGES>
static int launch_persistent(const TcArgs& args, const TcSched& sc, int n_sm, cudaStream_t stream) {
  constexpr int smem = persistent_smem<BLOCK_N, STAGES>();
  MF_ENSURE_DYN_SMEM((k_gemm_tc_persistent<BLOCK_N, STAGES, 1>), smem);
  int grid = (sc.n_units < n_sm && !sc.streamk) ? sc.n_units : n_sm;
  k_gemm_tc_persistent<BLOCK_N, STAGES, 1><<<grid, TC_P_THREADS, smem, stream>>>(args, sc);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

// launch configuration of `grid` CTAs in clusters of 2 (`attr` must outlive it)
template <int BLOCK_N, int STAGES>
static cudaLaunchConfig_t pair_config(cudaLaunchAttribute* attr, int grid, cudaStream_t stream) {
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = 2;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(TC_P_THREADS);
  cfg.dynamicSmemBytes = persistent_smem<BLOCK_N, STAGES>();
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

// How many CTA pairs can be resident at once (one CTA per SM).  Remembered per device, as
// MF_ENSURE_DYN_SMEM does, so that calls made while a CUDA graph is captured only read it.
template <int BLOCK_N, int STAGES>
static int pair_clusters(int dev, int n_sm, int* n_clusters) {
  static int known[64];
  MF_ENSURE_DYN_SMEM((k_gemm_tc_persistent<BLOCK_N, STAGES, 2>), (persistent_smem<BLOCK_N, STAGES>()));
  if (dev >= 0 && dev < 64 && known[dev] > 0) {
    *n_clusters = known[dev];
    return MF_OK;
  }
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t cfg = pair_config<BLOCK_N, STAGES>(&attr, n_sm & ~1, 0);
  MF_CUDA_TRY(cudaOccupancyMaxActiveClusters(n_clusters, k_gemm_tc_persistent<BLOCK_N, STAGES, 2>, &cfg));
  if (dev >= 0 && dev < 64) known[dev] = *n_clusters;
  return MF_OK;
}

// at most `n_clusters` pairs, all resident: stream-K needs every CTA on an SM at once
template <int BLOCK_N, int STAGES>
static int launch_persistent_pairs(const TcArgs& args, const TcSched& sc, int n_clusters,
                                   cudaStream_t stream) {
  const int clusters = (sc.n_units < n_clusters && !sc.streamk) ? sc.n_units : n_clusters;
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t cfg = pair_config<BLOCK_N, STAGES>(&attr, 2 * clusters, stream);
  MF_CUDA_TRY(cudaLaunchKernelEx(&cfg, k_gemm_tc_persistent<BLOCK_N, STAGES, 2>, args, sc));
  MF_LAUNCH_CHECK();
  return MF_OK;
}

static int check_shape(const GemmParams& p) {
  // shapes this kernel family covers; everything else goes to the SIMT kernel
  if (p.K < 64 || p.K % 8 != 0 || p.ldw % 8 != 0) return MF_E_UNSUPPORTED;
  if (p.N % 32 != 0 || p.N < 128) {
    // ragged / small N: only fp32 row-major outputs, a single N tile, no split-K
    if (p.out_mode != OUT_F32 || p.N > 128 || p.N < 8) return MF_E_UNSUPPORTED;
  }
  if (((uintptr_t)p.A & 15) || ((uintptr_t)p.W & 15) || ((uintptr_t)p.out & 15))
    return MF_E_UNSUPPORTED;
  if (p.N % 32 == 0 && p.out_mode != OUT_S2D_BF16 && ((p.ldo % 8) || (p.col_off % 8)))
    return MF_E_UNSUPPORTED;
  return MF_OK;
}

// w_rows: rows of the W box (the N tile, or half of it when a CTA pair shares the tile)
static int make_maps(const GemmParams& p, int w_rows, CUtensorMap* tmA, CUtensorMap* tmW, int* kb_per_a) {
  int rc;
  *kb_per_a = 0;
  if (p.mode == GEMM_CONV_S2D) {
    const int Do = p.Do, Js = Do + 1;
    if (!(Do == 8 || Do == 16) || p.Ci8 % 64 != 0 || p.K != 8 * p.Ci8) return MF_E_UNSUPPORTED;
    if (p.M % (Do * Do * Do) != 0) return MF_E_UNSUPPORTED;
    const int Bn = p.M / (Do * Do * Do);
    *kb_per_a = p.Ci8 / 64;
    cuuint64_t dims[5] = {(cuuint64_t)p.Ci8, (cuuint64_t)Js, (cuuint64_t)Js, (cuuint64_t)Js,
                          (cuuint64_t)Bn};
    cuuint64_t str[4] = {(cuuint64_t)p.Ci8 * 2, (cuuint64_t)Js * p.Ci8 * 2,
                         (cuuint64_t)Js * Js * p.Ci8 * 2, (cuuint64_t)Js * Js * Js * p.Ci8 * 2};
    // 128 consecutive output voxels (w fastest): 16x8x1 for Do=16, 8x8x2 for Do=8
    cuuint32_t box[5] = {64, (cuuint32_t)Do, 8, (cuuint32_t)(Do == 16 ? 1 : 2), 1};
    rc = encode(tmA, p.A, 5, dims, str, box);
  } else {
    if (p.lda % 8 != 0) return MF_E_UNSUPPORTED;
    cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.M};
    cuuint64_t str[1] = {(cuuint64_t)p.lda * 2};
    cuuint32_t box[2] = {64, 128};
    rc = encode(tmA, p.A, 2, dims, str, box);
  }
  if (rc) return rc;
  cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.N};
  cuuint64_t str[1] = {(cuuint64_t)p.ldw * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)w_rows};
  return encode(tmW, p.W, 2, dims, str, box);
}

// Whether a bf16 output can leave through the staged epilogue (staged_epilogue): row-major with
// a 16-byte aligned first column and pitch, or s2d at Do = 16 whose slots are whole 64-channel
// boxes.  fp32 outputs, ragged N and anything a TMA store cannot address take the register path.
static bool staged_ok(const GemmParams& p) {
  if (p.N % 32 != 0) return false;
  if (p.out_mode == OUT_BF16)
    return ((uintptr_t)p.out + 2 * (uintptr_t)p.col_off) % 16 == 0 && p.ldo % 8 == 0 && p.ldo >= p.N;
  if (p.out_mode == OUT_S2D_BF16)
    return p.Do == 16 && p.N % 64 == 0 && p.M % 4096 == 0 && (uintptr_t)p.out % 16 == 0;
  return false;
}

// Output map of the staged epilogue: row-major {N, M} at out + col_off in 64 x 64 boxes, or the
// s2d layout [B][9][9][9][8 N] of the next convolution's input in {64, 8, 2, 1, 1} boxes (StgS2D)
static int make_out_map(const GemmParams& p, CUtensorMap* tm) {
  if (p.out_mode == OUT_S2D_BF16) {
    const cuuint64_t J = 9, C = 8 * (cuuint64_t)p.N;
    const cuuint64_t dims[5] = {C, J, J, J, (cuuint64_t)(p.M / 4096)};
    const cuuint64_t str[4] = {C * 2, J * C * 2, J * J * C * 2, J * J * J * C * 2};
    const cuuint32_t box[5] = {64, 8, 2, 1, 1};
    return encode(tm, p.out, 5, dims, str, box);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)p.N, (cuuint64_t)p.M};
  const cuuint64_t str[1] = {(cuuint64_t)p.ldo * 2};
  const cuuint32_t box[2] = {64, 64};
  return encode(tm, reinterpret_cast<const bf16*>(p.out) + p.col_off, 2, dims, str, box);
}

}  // namespace mf

using namespace mf;


extern "C" size_t mf_gemm_bf16_tc_workspace_bytes(int M, int N) {
  size_t splitk = (size_t)M * N * 4 * 4 + 256;              // up to 4 split-K slices
  size_t streamk = (size_t)256 * TC_BLOCK_M * 256 * 4;      // one 128 x 256 fp32 slot per SM (<= 256)
  return splitk > streamk ? splitk : streamk;
}

extern "C" int mf_gemm_bf16_tc_ex(const GemmParams* hp, int n_groups, void* workspace,
                                  size_t workspace_bytes, int32_t* sync, long long* stamps,
                                  int one_shot, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!hp || n_groups < 1 || n_groups > TC_MAX_GROUPS) return MF_E_BADARG;
  TcArgs args;
  memset(&args, 0, sizeof(args));
  const GemmParams& p0 = hp[0];
  for (int g = 0; g < n_groups; ++g) {
    int rc = check_shape(hp[g]);
    if (rc) return rc;
    const bool small_n = p0.N <= 128 && hp[g].N <= 128 && hp[g].out_mode == OUT_F32 &&
                         p0.out_mode == OUT_F32;
    if (hp[g].M != p0.M || (hp[g].N != p0.N && !small_n) || hp[g].K != p0.K ||
        hp[g].mode != p0.mode || hp[g].Do != p0.Do || hp[g].Ci8 != p0.Ci8)
      return MF_E_UNSUPPORTED;
    args.p[g] = hp[g];
  }
  const int BN = (p0.N >= 256) ? 256 : 128;
  int n_sm = 132, dev = 0;
  MF_CUDA_TRY(cudaGetDevice(&dev));
  MF_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
  // The convolutions run as CTA pairs sharing the W tile (their m-tile count is even: M is a
  // multiple of Do^3 >= 512), when pairs can cover every SM; linear GEMMs (odd m-tile counts
  // such as M = 8000) as single CTAs.
  int cluster = 1, n_pairs = 0;
  if (p0.mode == GEMM_CONV_S2D) {
    int rc = BN == 256 ? pair_clusters<256, 4>(dev, n_sm, &n_pairs)
                       : pair_clusters<128, 6>(dev, n_sm, &n_pairs);
    if (rc) return rc;
    if (2 * n_pairs >= (n_sm & ~1)) cluster = 2;
  }
  args.e.kb_total = (p0.K + TC_BLOCK_K - 1) / TC_BLOCK_K;
  for (int g = 0; g < n_groups; ++g) {
    int rc = make_maps(hp[g], BN / cluster, &args.tmA[g], &args.tmW[g], &args.e.kb_per_a);
    if (rc) return rc;
  }
  int maxN = p0.N;
  for (int g = 1; g < n_groups; ++g) maxN = hp[g].N > maxN ? hp[g].N : maxN;
  const int m_tiles = (p0.M + TC_BLOCK_M - 1) / TC_BLOCK_M, n_tiles = (maxN + BN - 1) / BN;
  int splitk = 1;
  const int tiles = m_tiles * n_tiles * n_groups;
  // stream-K when the caller provides the flag words and whole-tile scheduling would idle > 5 %
  // of the SMs (or there are fewer tiles than SMs) on a long-K problem with bf16 output
  bool streamk = false;
  // (short-K problems are epilogue-bound: the extra accumulator round trip costs more than the
  // idle tail it removes)
  bool sk_ok = sync && one_shot != 1 && args.e.kb_total >= 32 && n_sm <= MF_GEMM_TC_SYNC_INTS / 8;
  for (int g = 0; g < n_groups; ++g)
    sk_ok = sk_ok && hp[g].N % 32 == 0 && hp[g].out_mode != OUT_F32;
  if (sk_ok) {
    const int waves = (tiles + n_sm - 1) / n_sm;
    const double busy = (double)tiles / ((double)waves * n_sm);
    const size_t need = (size_t)n_sm * TC_BLOCK_M * BN * 4;
    if (busy < 0.95 && workspace && workspace_bytes >= need) streamk = true;
  }
  if (!streamk && n_groups == 1 && 2 * tiles <= n_sm && args.e.kb_total >= 64 && p0.N % 32 == 0) {
    splitk = n_sm / tiles;
    if (splitk > 4) splitk = 4;
    if (splitk < 1) splitk = 1;
  }
  args.e.kb_per_split = (args.e.kb_total + splitk - 1) / splitk;
  splitk = (args.e.kb_total + args.e.kb_per_split - 1) / args.e.kb_per_split;
  args.e.splitk = splitk;
  args.e.err = nullptr;
  if (splitk > 1) {
    if (!workspace || workspace_bytes < (size_t)splitk * p0.M * p0.N * 4) return MF_E_WORKSPACE;
    args.e.ws = (float*)workspace;
  }
  // bf16 outputs leave through shared memory and TMA stores when every group's output allows it
  bool staged = splitk == 1;
  for (int g = 0; g < n_groups; ++g) staged = staged && staged_ok(hp[g]);
  for (int g = 0; staged && g < n_groups; ++g) {
    int rc = make_out_map(hp[g], &args.tmO[g]);
    if (rc) return rc;
  }
  args.e.staged = staged ? 1 : 0;
  const int m_units = m_tiles / cluster;
  TcSched sc{m_units, n_tiles, n_groups, splitk, m_units * n_tiles * n_groups * splitk,
             stamps, streamk ? 1 : 0, sync, (float*)workspace};
  int rc;
  if (cluster == 2)
    rc = BN == 256 ? launch_persistent_pairs<256, 4>(args, sc, n_pairs, stream)
                   : launch_persistent_pairs<128, 6>(args, sc, n_pairs, stream);
  else
    rc = BN == 256 ? launch_persistent<256, 4>(args, sc, n_sm, stream)
                   : launch_persistent<128, 6>(args, sc, n_sm, stream);
  if (rc) return rc;
  if (splitk > 1) {
    MF_PREFER_MAX_SMEM(k_splitk_finish);
    k_splitk_finish<<<div_up((long long)p0.M * p0.N / 4, 256), 256, 0, stream>>>(args.e.ws, p0, splitk);
    MF_LAUNCH_CHECK();
  }
  return MF_OK;
}

extern "C" int mf_gemm_bf16_tc_grouped(const GemmParams* hp, int n_groups, void* workspace,
                                       size_t workspace_bytes, void* stream_) {
  return mf_gemm_bf16_tc_ex(hp, n_groups, workspace, workspace_bytes, nullptr, nullptr, 0, stream_);
}

// Shared memory of k_heads_tc: a 4-stage ring of 48 KB stages and a 32 KB staging buffer (16 KB,
// 64 rows x 128 columns, per consumer warpgroup: a 256-wide tile drains in two passes).
constexpr int HD_STAGES = 4, HD_STG_COLS = 128;
constexpr int HD_SMEM = HD_STAGES * (TC_A_BYTES + 256 * TC_BLOCK_K * 2) + 2 * 64 * HD_STG_COLS * 2 + 1024;

// launch configuration of `grid` CTAs of k_heads_tc in clusters of 2 (`attr` must outlive it)
static cudaLaunchConfig_t heads_config(cudaLaunchAttribute* attr, int grid, cudaStream_t stream) {
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = 2;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(TC_P_THREADS);
  cfg.dynamicSmemBytes = HD_SMEM;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

extern "C" int mf_cnn_heads_tc(const GemmParams* layers, int n_layers, int32_t* sync, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!layers || n_layers != 7 || !sync) return MF_E_BADARG;
  const int M = layers[0].M;
  const int m_tiles = (M + TC_BLOCK_M - 1) / TC_BLOCK_M, m_pairs = (m_tiles + 1) / 2;
  if (16 + 4 * m_tiles > MF_HEADS_SYNC_INTS) return MF_E_TOOLARGE;
  for (int l = 0; l < 7; ++l) {
    const GemmParams& p = layers[l];
    int rc = check_shape(p);
    if (rc) return rc;
    if (p.M != M || p.mode != GEMM_LINEAR || p.out_mode != OUT_BF16 || p.N % 32 != 0 || p.N < 128)
      return MF_E_UNSUPPORTED;
    if (l >= 2 && l <= 3 && (p.N != layers[1].N || p.K != layers[1].K)) return MF_E_UNSUPPORTED;
    if (l >= 5 && (p.N != layers[4].N || p.K != layers[4].K)) return MF_E_UNSUPPORTED;
  }
  // GEMM list: layer 1 in 256-wide tiles and, when the last 1-128 columns would leave a 256-wide
  // tile half empty or more, those columns as a GEMM of their own in one 128-wide tile; then the
  // three layer-2 and the three layer-3 GEMMs
  GemmParams g[HD_GEMMS];
  int bn[HD_GEMMS];
  const int tail = layers[0].N % 256 <= 128 ? layers[0].N % 256 : 0;
  g[0] = layers[0];
  g[0].N -= tail;
  bn[0] = 256;
  g[1] = layers[0];
  g[1].N = tail;
  g[1].W = reinterpret_cast<const bf16*>(layers[0].W) + (size_t)g[0].N * layers[0].ldw;
  g[1].bias = layers[0].bias ? layers[0].bias + g[0].N : nullptr;
  g[1].col_off += g[0].N;
  bn[1] = 128;
  for (int l = 1; l < 7; ++l) {
    g[l + 1] = layers[l];
    bn[l + 1] = layers[l].N >= 256 ? 256 : 128;
  }
  HeadsArgs a;
  memset(&a, 0, sizeof(a));
  int units = 0;
  for (int q = 0; q < HD_GEMMS; ++q) {
    const GemmParams& p = g[q];
    a.bias[q] = p.bias;
    a.N[q] = p.N;
    a.relu[q] = p.relu;
    a.bn[q] = bn[q];
    a.kb[q] = (p.K + TC_BLOCK_K - 1) / TC_BLOCK_K;
    a.n_tiles[q] = (p.N + bn[q] - 1) / bn[q];
    a.unit_begin[q] = units;
    units += m_pairs * a.n_tiles[q];
    if (p.N == 0) continue;
    int dummy = 0;
    int rc = make_maps(p, bn[q] / 2, &a.tmA[q], &a.tmW[q], &dummy);
    if (rc) return rc;
    rc = make_out_map(p, &a.tmO[q]);
    if (rc) return rc;
  }
  a.unit_begin[HD_GEMMS] = units;
  // counters: [0, m_tiles) layer-1 rows; [m_tiles * (1 + h), ...) layer-2 rows of head h; one
  // arrival per consumer warpgroup and tile
  for (int q = 0; q < 2; ++q) {
    a.dep_base[q] = -1;
    a.sig_base[q] = 0;
  }
  for (int h = 0; h < 3; ++h) {
    a.dep_base[2 + h] = 0;
    a.dep_target[2 + h] = (a.n_tiles[0] + a.n_tiles[1]) * 2;
    a.sig_base[2 + h] = m_tiles * (1 + h);
    a.dep_base[5 + h] = m_tiles * (1 + h);
    a.dep_target[5 + h] = a.n_tiles[2 + h] * 2;
    a.sig_base[5 + h] = -1;
  }
  a.m_tiles = m_tiles;
  a.n_units = units;
  a.sync = sync;
  a.err = nullptr;
  MF_ENSURE_DYN_SMEM((k_heads_tc<HD_STAGES, HD_STG_COLS>), HD_SMEM);
  int n_sm = 132, dev = 0;
  MF_CUDA_TRY(cudaGetDevice(&dev));
  MF_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
  // Units wait on units of other CTAs, so every pair must be resident: at most as many pairs as
  // fit at once.  Remembered per device, so that calls made while a CUDA graph is captured only
  // read it.  When pairs cannot cover every SM the caller runs the three grouped launches.
  static int known[64];
  int n_pairs = dev >= 0 && dev < 64 ? known[dev] : 0;
  cudaLaunchAttribute attr;
  if (n_pairs <= 0) {
    const cudaLaunchConfig_t q = heads_config(&attr, n_sm & ~1, 0);
    MF_CUDA_TRY(cudaOccupancyMaxActiveClusters(&n_pairs, k_heads_tc<HD_STAGES, HD_STG_COLS>, &q));
    if (dev >= 0 && dev < 64) known[dev] = n_pairs;
  }
  if (2 * n_pairs < (n_sm & ~1)) return MF_E_UNSUPPORTED;
  const int clusters = units < n_pairs ? units : n_pairs;
  const cudaLaunchConfig_t cfg = heads_config(&attr, 2 * clusters, stream);
  MF_CUDA_TRY(cudaLaunchKernelEx(&cfg, k_heads_tc<HD_STAGES, HD_STG_COLS>, a));
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_gemm_bf16_tc(const GemmParams* hp, void* workspace, size_t workspace_bytes,
                               void* stream_) {
  return mf_gemm_bf16_tc_grouped(hp, 1, workspace, workspace_bytes, stream_);
}

