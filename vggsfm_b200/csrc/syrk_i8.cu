// Schur SYRK on the INT8 tensor cores: Sraw -= Zt^T Zt in FP64-equivalent precision computed with INT8 wgmma (Ozaki
// splitting), exposed as vgg_syrk_ozaki.  The LM loop runs the FP64 tensor-core kernel of csrc/ba_schur.cu instead:
// INT8 wgmma has 32x the FP64 tensor-core rate of sm_90a (4096 int8 MAC against 128 DMMA FMA per clock and SM), and
// s = 7 slices need 28 int8 products per FP64-equivalent product, so even at peak this path is only 32/28 = 1.14x
// the DMMA rate before the slicing pass; at 400 x 4096 it measured 2x slower (DESIGN section 4.2).
//   1. every column d of Z (a reduced camera parameter) gets a power-of-two scale 2^e_d >= max_k |Z[k][d]|;
//      x = Z 2^-e_d is rounded to B = 8s-2 fractional bits and written as s balanced base-256 digits
//      (int8 "slices", most significant first): x = 2^-B sum_p d_p 256^(s-p)          (oz_slice_kernel)
//   2. (Z^T Z)_ij = 2^(e_i+e_j-2B) sum_t 256^(2s-t) C_t,  C_t = sum_{p+q=t} sum_k d_p[k][i] d_q[k][j]:
//      every C_t is an exact int32 (|d| <= 128, at most 7 pairs and 16384 k per work item: |C_t| < 2^31); orders t > s+1 are below
//      the rounding of step 1 and are dropped, leaving s(s+1)/2 int8 GEMMs (28 for s = 7)  (oz_syrk_kernel)
//   3. the epilogue recombines the C_t of a tile in FP64 registers and adds -value into Sraw with f64 RED
//      (or multimem.red in fabric mode) through syrk_red_upper, the epilogue of the FP64 kernel too.
//
// oz_syrk_kernel is a persistent, warp-specialised wgmma kernel (one CTA per SM):
//   warpgroup 0    producer: the int8 slices are stored in HBM as 8 KB tile images that are already in the 64-byte
//                  swizzled K-major shared-memory layout wgmma wants, so a tile is ONE 1-D bulk copy (cp.async.bulk)
//                  completing on an mbarrier -- no tensor map, no driver API;
//   warpgroups 1-2 consumers, 64 tile rows each: wgmma.m64n128k32.s32.s8.s8 for every (p,q) pair of the work item's
//                  order group into up to two register accumulators (one per order t), then combine the orders in
//                  FP64, scale by 2^(e_i+e_j) and RED into the lower triangle.
// Work items (tile, order group, k range) are built on the host, longest first, and strided over the CTAs.
#include "common.cuh"
#include "syrk_work.h"

#include <algorithm>
#include <vector>

namespace vgg {

namespace {

constexpr int OZ_BM = 128;                       // tile rows (reduced camera parameters)
constexpr int OZ_BK = 64;                        // k bytes per block = one 64-byte swizzle atom
constexpr int OZ_TILE_BYTES = OZ_BM * OZ_BK;     // 8 KB
constexpr int OZ_STAGES = 2;
constexpr int OZ_STAGE_TILES = 14;
constexpr int OZ_STAGE_BYTES = OZ_STAGE_TILES * OZ_TILE_BYTES;   // 112 KB
constexpr int OZ_THREADS = 384;                  // producer warpgroup + 2 consumer warpgroups (64 tile rows each)
constexpr int OZ_MAX_ACC = 2;                    // orders per group: 2 x 64 int32 accumulator registers per thread
constexpr int OZ_MAX_PAIRS = 20;
constexpr int OZ_MAX_ITEM_KB = 256;               // k blocks per work item: 7 pairs x 128^2 x 256 x 64 < 2^31 (exact int32 accumulators)
constexpr int OZ_PREFETCH = 4;                   // k blocks of L2 prefetch distance ahead of the bulk copies
constexpr int OZ_MAX_GROUPS = 4;
constexpr int OZ_EXPO_BAD = INT32_MIN;           // column holds a non-finite value
constexpr size_t OZ_SMEM_BYTES = (size_t)OZ_STAGES * OZ_STAGE_BYTES + 1024 + 128;

struct OzGroup {
  int n_a, n_b, n_pairs, n_acc;
  int exp_base;                                  // 8 (2s - tmax) - 2B
  uint8_t a_slice[8], b_slice[8];                // slice held by tile slot i / n_a + i
  uint8_t pair_a[OZ_MAX_PAIRS], pair_b[OZ_MAX_PAIRS], pair_acc[OZ_MAX_PAIRS];
  uint8_t pair_b_diag[OZ_MAX_PAIRS];             // on diagonal tiles B_q is the A slot that holds slice q
  uint8_t acc_shift[4];                          // 8 (tmax - t) of accumulator a
};
struct OzPlan {
  int slices, n_groups;
  OzGroup g[OZ_MAX_GROUPS];
};
struct OzWork {
  int bi, bj, group, kb0, kb1;
};

// ---------------------------------------------------------------------------------------------------------
// 1. column scales
__global__ void oz_rowmax_kernel(int Kpad, int Dpad, int k_per, const double* __restrict__ Zt,
                                 unsigned long long* __restrict__ amax) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= Dpad) return;
  const int k0 = blockIdx.y * k_per, k1 = min(Kpad, k0 + k_per);
  double m = 0.0;
  bool bad = false;
  for (int k = k0; k < k1; ++k) {
    const double a = fabs(Zt[(size_t)k * Dpad + d]);
    bad |= !(a <= 1.7976931348623157e308);
    m = fmax(m, a);
  }
  if (bad) m = __longlong_as_double(0x7ff0000000000000LL);
  if (m > 0.0) atomicMax(&amax[d], (unsigned long long)__double_as_longlong(m));
}

// 2. slices, written as pre-swizzled 8 KB tile images: tile (slice p, row block rb, k block kb) holds rows
//    d = rb*128 + r, bytes k = kb*64 + kk at offset r*64 + (((kk >> 4) ^ ((r >> 1) & 3)) << 4) + (kk & 15)
//    (the 64-byte swizzle, Swizzle<2,4,3>, of a K-major 128 x 64 B tile whose base is 1024-byte aligned).
//    Balanced base-256 digits come from ONE 64-bit add: with X = rint(x 2^B), |X| <= 2^B, the bytes of
//    X + 0x80..80 (s bytes of 0x80) are d_p + 128, so d_p = byte ^ 0x80.  A warp owns 8 rows x 4 chunks: its loads are
//    4 x 64-byte segments per k and its stores 512 contiguous bytes per slice.
__global__ void __launch_bounds__(512) oz_slice_kernel(int Kpad, int Dpad, int KB, int s,
                                                       const double* __restrict__ Zt,
                                                       const unsigned long long* __restrict__ amax,
                                                       int* __restrict__ expo, double* __restrict__ pow2,
                                                       int8_t* __restrict__ slices, size_t slice_stride) {
  const int rb = blockIdx.x, kb = blockIdx.y;
  const int r = (threadIdx.x >> 5) * 8 + ((threadIdx.x & 31) >> 2), cphys = threadIdx.x & 3;
  const int c = cphys ^ ((r >> 1) & 3);
  const int d = rb * OZ_BM + r;
  const double m = __longlong_as_double((long long)amax[d]);
  int e = 0;
  bool bad = false, zero = true;
  if (m > 0.0) {
    if (m <= 1.7976931348623157e308) {
      e = ilogb(m) + 1;
      zero = e < -900;                 // columns below 2^-900 are treated as exact zeros (keeps 2^(B-e) finite)
      if (zero) e = 0;
    } else {
      bad = true;
    }
  }
  if (kb == 0 && cphys == 0) {
    expo[d] = bad ? OZ_EXPO_BAD : e;
    pow2[d] = bad ? 0.0 : ldexp(1.0, e);
  }
  const int B = 8 * s - 2;
  const double scale = (bad || zero) ? 0.0 : __longlong_as_double((long long)(1023 + B - e) << 52);   // 2^(B-e), exact
  const unsigned long long bias = 0x0080808080808080ull >> (8 * (7 - s));
  uint32_t dig[7][4];
#pragma unroll
  for (int p = 0; p < 7; ++p) dig[p][0] = dig[p][1] = dig[p][2] = dig[p][3] = 0u;
  const int kbase = kb * OZ_BK + c * 16;
  double z[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) z[i] = (kbase + i < Kpad) ? Zt[(size_t)(kbase + i) * Dpad + d] : 0.0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const unsigned long long Y = ((unsigned long long)__double2ll_rn(z[i] * scale) + bias) ^ bias;   // byte j = digit of 256^j
    const uint32_t lo = (uint32_t)Y, hi = (uint32_t)(Y >> 32);
#pragma unroll
    for (int p = 0; p < 7; ++p) {
      if (p < s) {
        const int j = s - 1 - p;                           // slice p (most significant first) is byte j
        const uint32_t byte = ((j < 4 ? lo >> (8 * j) : hi >> (8 * (j - 4))) & 255u);
        dig[p][i >> 2] |= byte << (8 * (i & 3));
      }
    }
  }
  const size_t off = ((size_t)rb * KB + kb) * OZ_TILE_BYTES + (size_t)r * OZ_BK + (size_t)(cphys << 4);
#pragma unroll
  for (int p = 0; p < 7; ++p)
    if (p < s) *reinterpret_cast<uint4*>(slices + (size_t)p * slice_stride + off) = make_uint4(dig[p][0], dig[p][1], dig[p][2], dig[p][3]);
}

// ---------------------------------------------------------------------------------------------------------
// wgmma (PTX ISA 8.0+, sm_90a)
// pull a global range into L2 ahead of the bulk copy that will read it (hides the HBM latency of first-touch tiles)
__device__ __forceinline__ void l2_prefetch(const void* gptr, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gptr), "r"(bytes) : "memory");
}

// d[64 x 128] (+)= A[64 x 32] * B[128 x 32]^T, int8 x int8 -> int32, both operands K-major in shared memory.
// Fragment of thread (warp w of the warpgroup, lane l): d[j] is row 16 w + l / 4 + 8 ((j >> 1) & 1),
// column 8 (j >> 2) + 2 (l & 3) + (j & 1).
__device__ __forceinline__ void wgmma_i8(int32_t (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, 1;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}

// ---------------------------------------------------------------------------------------------------------
// 3. persistent wgmma SYRK.  Warpgroup 0 is the producer, warpgroups 1 and 2 own rows 0-63 / 64-127 of the 128 x 128
// tile: they issue the wgmmas of every (p,q) pair of the work item's order group into up to OZ_MAX_ACC register
// accumulators (one per order t), then combine the orders in FP64 and RED the tile into Sraw themselves.
template <int NACC>
__device__ __forceinline__ void oz_mma_pair(int32_t (&acc)[OZ_MAX_ACC][64], int a, uint64_t da, uint64_t db) {
  if (NACC > 1 && a == 1) wgmma_i8(acc[1], da, db);
  else wgmma_i8(acc[0], da, db);
}

__global__ void __launch_bounds__(OZ_THREADS, 1)
    oz_syrk_kernel(const __grid_constant__ OzPlan plan, const OzWork* __restrict__ work, int nwork, int KB,
                   const int8_t* __restrict__ slices, size_t slice_stride, const int* __restrict__ expo,
                   const double* __restrict__ pow2, int Dpad, double* __restrict__ Cmat, ptrdiff_t mc_off,
                   const __grid_constant__ FabricDev fd) {
  extern __shared__ __align__(1024) uint8_t oz_smem[];
  uint8_t* tiles = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<size_t>(oz_smem), 1024));
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + (size_t)OZ_STAGES * OZ_STAGE_BYTES);
  uint64_t* empty = full + OZ_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    for (int s = 0; s < OZ_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);                   // one arrive per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== producer =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");     // registers go to the consumers' accumulators
    if (threadIdx.x == 0) {
      int stage = 0, phase = 0;
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        const OzWork wk = work[w];
        const OzGroup& g = plan.g[wk.group];
        const bool diag = wk.bi == wk.bj;
        for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
          const int kpf = kb + OZ_PREFETCH;
          if (kpf < wk.kb1) {
            for (int i = 0; i < g.n_a; ++i)
              l2_prefetch(slices + (size_t)g.a_slice[i] * slice_stride + ((size_t)wk.bi * KB + kpf) * OZ_TILE_BYTES, OZ_TILE_BYTES);
            for (int i = 0; i < (diag ? 0 : g.n_b); ++i)
              l2_prefetch(slices + (size_t)g.b_slice[i] * slice_stride + ((size_t)wk.bj * KB + kpf) * OZ_TILE_BYTES, OZ_TILE_BYTES);
          }
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* dst = tiles + (size_t)stage * OZ_STAGE_BYTES;
          mbar_expect_tx(&full[stage], (uint32_t)(g.n_a + (diag ? 0 : g.n_b)) * OZ_TILE_BYTES);
          for (int i = 0; i < g.n_a; ++i)
            tma_load_1d(dst + (size_t)i * OZ_TILE_BYTES,
                        slices + (size_t)g.a_slice[i] * slice_stride + ((size_t)wk.bi * KB + kb) * OZ_TILE_BYTES,
                        OZ_TILE_BYTES, &full[stage]);
          for (int i = 0; i < (diag ? 0 : g.n_b); ++i)
            tma_load_1d(dst + (size_t)(g.n_a + i) * OZ_TILE_BYTES,
                        slices + (size_t)g.b_slice[i] * slice_stride + ((size_t)wk.bj * KB + kb) * OZ_TILE_BYTES,
                        OZ_TILE_BYTES, &full[stage]);
          if (++stage == OZ_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup 1 -> tile rows 0..63, warpgroup 2 -> rows 64..127 =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int half = wg - 1, wq = warp & 3;
  const uint32_t a_row_off = (uint32_t)half * 64u * OZ_BK;      // 64 rows = 8 swizzle atoms: the pattern is unchanged
  int stage = 0, phase = 0;
  int32_t acc[OZ_MAX_ACC][64];
  for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
    const OzWork wk = work[w];
    const OzGroup& g = plan.g[wk.group];
    const bool diag = wk.bi == wk.bj;
#pragma unroll
    for (int a = 0; a < OZ_MAX_ACC; ++a)
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[a][j] = 0;
    for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t base = smem_u32(tiles + (size_t)stage * OZ_STAGE_BYTES);
      wgmma_fence();
      for (int pr = 0; pr < g.n_pairs; ++pr) {
        const uint32_t a_addr = base + (uint32_t)g.pair_a[pr] * OZ_TILE_BYTES + a_row_off;
        const uint32_t b_addr = base + (uint32_t)(diag ? g.pair_b_diag[pr] : g.n_a + g.pair_b[pr]) * OZ_TILE_BYTES;
        const int a = g.pair_acc[pr];
#pragma unroll
        for (int ks = 0; ks < OZ_BK / 32; ++ks)
          oz_mma_pair<OZ_MAX_ACC>(acc, a, wgmma_desc_sw64(a_addr + ks * 32), wgmma_desc_sw64(b_addr + ks * 32));
      }
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == OZ_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    // combine the orders, scale and accumulate into Sraw (syrk_red_upper, common.cuh)
    const int row_base = wk.bi * OZ_BM + half * 64 + wq * 16 + (lane >> 2);
    const int col_base = wk.bj * OZ_BM + 2 * (lane & 3);
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int r = row_base + 8 * rh;
      const int er = expo[r];
      // 2^(e_r + e_c + exp_base) as two exact multiplications while the exponents are tame, ldexp otherwise
      const bool tame = er != OZ_EXPO_BAD && er > -400 && er < 400;
      const double sr = tame ? __longlong_as_double((long long)(1023 + er + g.exp_base) << 52) : 0.0;
#pragma unroll
      for (int n8 = 0; n8 < 16; ++n8)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int j = 4 * n8 + 2 * rh + c;
          const int col = col_base + 8 * n8 + c;
          double v = 0.0;
#pragma unroll
          for (int a = 0; a < OZ_MAX_ACC; ++a)
            if (a < g.n_acc) v = fma((double)acc[a][j], (double)(1ull << g.acc_shift[a]), v);
          const int ec = expo[col];
          if (er == OZ_EXPO_BAD || ec == OZ_EXPO_BAD) v = __longlong_as_double(0x7ff8000000000000LL);
          else if (tame && ec > -400 && ec < 400) v = v * sr * pow2[col];
          else v = ldexp(v, er + ec + g.exp_base);
          syrk_red_upper(Cmat, Dpad, r, col, wk.bj, diag, v, mc_off, fd);
        }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side: order groups and work list
bool build_plan(int s, OzPlan* plan, int max_acc) {
  if (s < 3 || s > 7) return false;
  plan->slices = s;
  const int B = 8 * s - 2;
  const int tlast = s + 1;                       // orders 2 .. s+1 are kept
  int ng = 0;
  for (int t0 = 2; t0 <= tlast; t0 += max_acc) {
    if (ng >= OZ_MAX_GROUPS) return false;
    OzGroup& g = plan->g[ng++];
    const int t1 = std::min(t0 + max_acc - 1, tlast);
    g.n_acc = t1 - t0 + 1;
    g.exp_base = 8 * (2 * s - t1) - 2 * B;
    int slot_a[8], slot_b[8];
    for (int i = 0; i < 8; ++i) slot_a[i] = slot_b[i] = -1;
    g.n_a = g.n_b = g.n_pairs = 0;
    for (int t = t0; t <= t1; ++t) {
      g.acc_shift[t - t0] = (uint8_t)(8 * (t1 - t));
      for (int p = 1; p <= s; ++p) {
        const int q = t - p;
        if (q < 1 || q > s) continue;
        if (slot_a[p] < 0) {
          slot_a[p] = g.n_a;
          g.a_slice[g.n_a++] = (uint8_t)(p - 1);
        }
        if (slot_b[q] < 0) {
          slot_b[q] = g.n_b;
          g.b_slice[g.n_b++] = (uint8_t)(q - 1);
        }
        if (g.n_pairs >= OZ_MAX_PAIRS) return false;
        g.pair_a[g.n_pairs] = (uint8_t)slot_a[p];
        g.pair_b[g.n_pairs] = (uint8_t)slot_b[q];
        g.pair_acc[g.n_pairs] = (uint8_t)(t - t0);
        ++g.n_pairs;
      }
    }
    for (int pr = 0; pr < g.n_pairs; ++pr) {              // the order groups are symmetric in (p, q): slice q has an A slot
      const int q = g.b_slice[g.pair_b[pr]] + 1;
      if (slot_a[q] < 0) return false;
      g.pair_b_diag[pr] = (uint8_t)slot_a[q];
    }
    if (g.n_a + g.n_b > OZ_STAGE_TILES) return false;
  }
  plan->n_groups = ng;
  return true;
}


struct OzHostState {
  int Kpad = -1, Dpad = -1, slices = -1, sms = 0;
  OzPlan plan;
  std::vector<OzWork> work;
  OzWork* pinned = nullptr;       // page-locked copy of `work`, so the per-call upload is a true async copy
  size_t pinned_cap = 0;
};

thread_local OzHostState g_oz;

int oz_max_parts(int KB) { return std::max(16, (KB + OZ_MAX_ITEM_KB - 1) / OZ_MAX_ITEM_KB); }

size_t oz_workspace_bytes(int Kpad, int Dpad, int s) {
  const int KB = (Kpad + OZ_BK - 1) / OZ_BK;
  const int nb = Dpad / OZ_BM;
  size_t bytes = 0;
  bytes += align_up((size_t)Dpad * 8, 256);                                   // amax
  bytes += align_up((size_t)Dpad * 4, 256);                                   // expo
  bytes += align_up((size_t)Dpad * 8, 256);                                   // pow2
  bytes += align_up((size_t)nb * (nb + 1) / 2 * OZ_MAX_GROUPS * oz_max_parts(KB) * sizeof(OzWork), 256);    // work list (upper bound)
  bytes += align_up((size_t)s * nb * KB * OZ_TILE_BYTES, 1024) + 1024;        // slices
  return bytes;
}

}  // namespace

size_t syrk_i8_workspace_bytes(int Kpad, int Dpad, int slices) { return oz_workspace_bytes(Kpad, Dpad, slices); }

// Sraw -= Zt^T Zt with s int8 slices.  Zt [Kpad][Dpad] (Dpad % 128 == 0), Cmat [Dpad][Dpad] row-major, LOWER triangle
// written, same contract as launch_syrk.
int launch_syrk_i8(int Kpad, int Dpad, const double* Zt, double* Cmat, int s, void* ws, size_t ws_bytes, cudaStream_t st) {
  VGG_REQUIRE(Dpad % OZ_BM == 0, "syrk_i8: Dpad must be a multiple of 128");
  VGG_REQUIRE(ws_bytes >= oz_workspace_bytes(Kpad, Dpad, s), "syrk_i8: workspace too small");
  const int KB = (Kpad + OZ_BK - 1) / OZ_BK;
  const int nb = Dpad / OZ_BM;
  OzHostState& hs = g_oz;
  if (hs.Kpad != Kpad || hs.Dpad != Dpad || hs.slices != s) {
    VGG_REQUIRE(build_plan(s, &hs.plan, OZ_MAX_ACC), "syrk_i8: slices must be in [3,7]");
    int dev = 0;
    VGG_CUDA_CHECK(cudaGetDevice(&dev));
    VGG_CUDA_CHECK(cudaDeviceGetAttribute(&hs.sms, cudaDevAttrMultiProcessorCount, dev));
    VGG_CUDA_CHECK(cudaFuncSetAttribute(oz_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM_BYTES));
    // work items: (tile, group, k range), longest first (build_work_list picks the k-split granularity)
    {
      std::vector<int> pairs;
      for (int g = 0; g < hs.plan.n_groups; ++g) pairs.push_back(hs.plan.g[g].n_pairs);
      // epilogue_cost: pair-kblock equivalents of one item's epilogue (order combination + REDs); OZ_MAX_ITEM_KB keeps
      // the int32 accumulators exact
      build_work_list<OzWork>(pairs, syrk_tile_jobs(nb, {}), KB, hs.sms, OZ_MAX_ITEM_KB, 24,
                              [](const SyrkTileJob& j, int g, int k0, int k1) { return OzWork{j.bi, j.bj, g, k0, k1}; }, &hs.work);
    }
    if (hs.work.size() > hs.pinned_cap) {
      if (hs.pinned) cudaFreeHost(hs.pinned);
      hs.pinned_cap = hs.work.size();
      VGG_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&hs.pinned), sizeof(OzWork) * hs.pinned_cap, cudaHostAllocDefault));
    }
    std::copy(hs.work.begin(), hs.work.end(), hs.pinned);
    hs.Kpad = Kpad;
    hs.Dpad = Dpad;
    hs.slices = s;
  }
  Carver c(ws, ws_bytes);
  unsigned long long* amax = c.take<unsigned long long>(Dpad);
  int* expo = c.take<int>(Dpad);
  double* pow2 = c.take<double>(Dpad);
  OzWork* work_d = c.take<OzWork>((size_t)nb * (nb + 1) / 2 * OZ_MAX_GROUPS * oz_max_parts(KB));
  c.off = align_up(c.off, 1024);
  int8_t* slices = reinterpret_cast<int8_t*>(c.base + c.off);
  const size_t slice_stride = (size_t)nb * KB * OZ_TILE_BYTES;
  const int nwork = (int)hs.work.size();

  VGG_CUDA_CHECK(cudaMemcpyAsync(work_d, hs.pinned, sizeof(OzWork) * nwork, cudaMemcpyHostToDevice, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(amax, 0, sizeof(unsigned long long) * Dpad, st));
  {
    const int ksplit = 64;
    const int k_per = (Kpad + ksplit - 1) / ksplit;
    oz_rowmax_kernel<<<dim3(Dpad / 128, ksplit), 128, 0, st>>>(Kpad, Dpad, k_per, Zt, amax);
    VGG_LAUNCH_CHECK();
  }
  oz_slice_kernel<<<dim3(nb, KB), 512, 0, st>>>(Kpad, Dpad, KB, s, Zt, amax, expo, pow2, slices, slice_stride);
  VGG_LAUNCH_CHECK();
  const int grid = std::min(hs.sms, nwork);
  oz_syrk_kernel<<<grid, OZ_THREADS, OZ_SMEM_BYTES, st>>>(hs.plan, work_d, nwork, KB, slices, slice_stride, expo, pow2, Dpad,
                                                          Cmat, 0, FabricDev{});
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace vgg

extern "C" {

int vgg_syrk_ozaki_workspace_bytes(int Kpad, int Dpad, int slices, size_t* bytes) {
  using namespace vgg;
  VGG_REQUIRE(bytes && Kpad > 0 && Dpad > 0 && Dpad % 128 == 0 && slices >= 3 && slices <= 7, "bad argument");
  *bytes = syrk_i8_workspace_bytes(Kpad, Dpad, slices);
  return VGG_OK;
}

int vgg_syrk_ozaki(int Kpad, int Dpad, const double* Zt, double* Cmat, int slices, void* workspace, size_t ws_bytes,
                   void* stream) {
  using namespace vgg;
  g_launch_count = 0;
  VGG_REQUIRE(Zt && Cmat && workspace, "null pointer");
  return launch_syrk_i8(Kpad, Dpad, Zt, Cmat, slices, workspace, ws_bytes, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
