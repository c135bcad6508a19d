// Shared device/host helpers for the vggsfm_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/vggsfm_b200.h"

namespace vgg {

void set_error(const char* fmt, ...);
extern thread_local long long g_launch_count;   // kernels launched by the current C-ABI call

#define VGG_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      vgg::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return VGG_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

#define VGG_LAUNCH_CHECK()                 \
  do {                                     \
    vgg::g_launch_count++;                 \
    VGG_CUDA_CHECK(cudaGetLastError());    \
  } while (0)

#define VGG_REQUIRE(cond, msg)                                   \
  do {                                                           \
    if (!(cond)) {                                               \
      vgg::set_error("%s:%d: %s", __FILE__, __LINE__, msg);      \
      return VGG_EINVAL;                                         \
    }                                                            \
  } while (0)

__host__ __device__ constexpr inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// bump allocator over the caller-provided workspace
struct Carver {
  char* base;
  size_t off = 0, cap;
  Carver(void* p, size_t c) : base(static_cast<char*>(p)), cap(c) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* r = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return r;
  }
  bool ok() const { return base == nullptr || off <= cap; }
};

// Band structure of a sequential (video) problem on the device (csrc/ba_solve.cu, compute_band_hint); null = dense.
// Points are stored in creation order, so every range is contiguous.
//   fg_tracks[2 g]  .. [2 g + 1]    track range [lo, hi) visible to the 32-frame group g
struct BandDev {
  const int* fg_tracks;
};

// Destination table of the fused multi-GPU reduction (csrc/fabric.cu): world <= 1 means "not in use".
struct FabricDev {
  int world, rank;
  double* peer[8];     // rank r's copy of the buffer being addressed (same layout on every rank, peer-mapped)
};

#ifdef __CUDACC__
// Correlation sampling (csrc/corr.cu, csrc/corr_tc.cu): a query's coordinate on a level of `size` positions, clamped
// into [-(R+2), size+R+1] before its footprint origin (int)floorf(c) is formed.  Inside that window the clamp is the
// identity.  Beyond it every tap c + d (|d| <= R) lies outside the map either way, so zeros padding still reads only
// zeros and border padding still reads the clamped edge.  NaN goes to the low end (fmaxf): 0 with zeros padding and
// column / row 0 with border padding, which is what grid_sample on CUDA returns for a NaN tap.  The int conversion and
// the footprint arithmetic on it are then defined for every input, ±inf and |c| >= 2^31 included.
__device__ __forceinline__ float corr_window(float c, int R, int size) {
  return fminf(fmaxf(c, -(float)(R + 2)), (float)(size + R + 1));
}

// ---------------------------------------------------------------------------------------------
// TMA 1-D bulk copies + mbarrier (PTX ISA 8.x, sm_90+; SASS: UBLKCP / SYNCS)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared, completion on mbarrier.  size multiple of 16, both addresses 16B aligned.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global bulk store (bulk async-group completion)
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// make generic-proxy shared-memory writes visible to the async proxy (TMA)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma (sm_90a): shared-memory matrix descriptor of a K-major operand in the 64-byte swizzle (Swizzle<2,4,3>; 8-row
// core-matrix groups 512 B apart, tile base 512-byte aligned), and the warpgroup fence / commit / wait
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// cp.async 16B (LDGSTS)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// FP64 tensor-core MMA at the full sm_90 rate (the m8n8k4 shape runs at half of it).
// d[16 x 8] += a[16 x 16] b[16 x 8]; lane (g = lane / 4, t = lane % 4) holds a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)],
// b[j] = B[t + 4 j][g], d = (g, 2t), (g, 2t + 1), (g + 8, 2t), (g + 8, 2t + 1)
__device__ __forceinline__ void dmma_m16n8k16(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// Warp reduce-scatter: every lane contributes v[0..KP), KP a power of two <= 32.  Returns in lane l
// the warp-wide sum of v[l & (KP-1)].  Costs KP-1 (+log2(32/KP)) 64-bit shuffles instead of 5*KP.
template <int KP>
__device__ __forceinline__ double warp_reduce_scatter(double (&v)[KP], int lane) {
#pragma unroll
  for (int off = KP / 2; off >= 1; off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const double mine = up ? v[i + off] : v[i];
      const double send = up ? v[i] : v[i + off];
      v[i] = mine + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  double r = v[0];
#pragma unroll
  for (int off = KP; off < 32; off <<= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
  return r;
}

__device__ __forceinline__ double warp_sum(double r) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
  return r;
}
__device__ __forceinline__ double warp_max(double r) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, off));
  return r;
}

// Epilogue of the Schur SYRK kernels (csrc/ba_schur.cu, csrc/syrk_i8.cu): subtract v = (Zt^T Zt)[r][col] of an UPPER
// tile (row block of r <= column block bj of col; diag: the two blocks are the same).  The element goes to its mirror
// (col, r) of the row-major LOWER triangle, which is what csrc/chol.cu factors; nothing is written above the diagonal.
// Destinations of the lower triangle:
//   fd.world > 1   reduce-scatter: row block bj lives on rank (bj mod world) until the gather (csrc/fabric.cu); one
//                  system-scope RED over NVLink per element, only into the owner's copy
//   mc_off != 0    one multimem RED on the NVSwitch multicast address, landing in every rank's copy
//   otherwise      a local f64 RED
__device__ __forceinline__ void syrk_red_upper(double* Cmat, int Dpad, int r, int col, int bj, bool diag, double v,
                                               ptrdiff_t mc_off, const FabricDev& fd) {
  if (v == 0.0 || (diag && col < r)) return;
  const size_t off = (size_t)col * Dpad + r;
  if (fd.world > 1) {
    asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(fd.peer[bj % fd.world] + off), "d"(-v) : "memory");
  } else if (mc_off) {
    asm volatile("multimem.red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(Cmat + off + mc_off), "d"(-v) : "memory");
  } else {
    atomicAdd(Cmat + off, -v);
  }
}
#endif  // __CUDACC__

}  // namespace vgg
