// Coarse-tracker correlation on the tensor cores (wgmma f16, fp32 register accumulators).
//
// CorrBlock.corr + CorrBlock.sample of the coarse tracker (vggsfm/models/track_modules/blocks.py:363-416: per level one
// torch.matmul of the [N,C] targets with all H*W positions, fp16 under autocast, then (2r+1)^2 bilinear taps) for
// C = 128 channels.  The CUDA-core footprint kernel (csrc/corr.cu) gathers the footprints through L2, which at the C4
// shape (128 frames x 1024 queries, 128x128 maps, 5 levels, r = 4) is slower than the dense product itself.  Here the
// dense product runs on the tensor cores, and the 5.7 GB volume is never written: one CTA per SM walks work items
// (frame, 128 queries); per level and per tile of 256 positions each of two consumer warpgroups (64 queries) issues
// wgmma M=64 x N=256 x K=128 (8 instructions of K=16) from shared memory into registers and keeps only the (2r+2)^2
// footprint values each query needs, in a shared-memory footprint table; after a level's last tile the same warps
// interpolate the (2r+1)^2 taps and write them.  While one warpgroup extracts, the other one's MMAs run.
//   operands: K-major, 64-byte swizzle (k-blocks of 32 fp16 channels), stored in global memory as ready-made tile
//   images -- B (feature positions) once per CorrBlock, A (targets) once per call -- so the producer warp moves a whole
//   256 x 128 operand tile with ONE 64 KB bulk copy (cp.async.bulk), no tensor map.
// grid_sample semantics kept: align_corners=True, padding "zeros" (taps outside the map read 0, and so do non-finite
// coordinates, as on CUDA: corr_window in common.cuh), tap order out[a*(2r+1)+b] at x = cx + (a-r), y = cy + (b-r).
// Maps whose width is a power of two (128 -> 8 at C4).
#include <cuda_fp16.h>
#include <algorithm>
#include "common.cuh"

namespace vgg {

namespace {

constexpr int CT_M = 128;                 // queries per work item (two consumer warpgroups of 64)
constexpr int CT_N = 256;                 // positions per tile
constexpr int CT_C = 128;                 // channels
constexpr int CT_KB = 4;                  // k-blocks of 32 channels (64 bytes)
constexpr int CT_A_BYTES = CT_M * CT_C * 2;          // 32 KB
constexpr int CT_B_BYTES = CT_N * CT_C * 2;          // 64 KB
constexpr int CT_STAGES = 2;
constexpr int CT_THREADS = 384;           // warpgroup 0 producer, warpgroups 1..2 MMA + footprint extraction (64 queries each)
constexpr int CT_FB_LD = 101;             // footprint table row stride (floats): 10*10 (+1: conflict-free per-query rows)
constexpr size_t CT_SMEM = 1024 + CT_A_BYTES + (size_t)CT_STAGES * CT_B_BYTES + (size_t)CT_M * CT_FB_LD * 4 + 256;

struct CtLevels {
  int H[8], W[8], logW[8], ntiles[8];
  size_t tile_off[8];                     // byte offset of level l's tile images inside one image's block
  size_t img_stride;                      // bytes of tile images per image (all levels)
};

__device__ __forceinline__ void mbar_arrive1(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// d[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, f16 x f16 -> f32, both operands K-major in shared memory; accumulate = 0
// overwrites d.  Fragment of thread (warp w of the warpgroup, lane l): d[j] is row 16 w + l / 4 + 8 ((j >> 1) & 1), column
// 8 (j >> 2) + 2 (l & 3) + (j & 1).
__device__ __forceinline__ void wgmma_f16(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21,"
      "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41,"
      "%42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61,"
      "%62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81,"
      "%82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100,"
      "%101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116,"
      "%117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
        "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
        "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),
        "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]),
        "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]),
        "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]),
        "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]),
        "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]),
        "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

// byte offset of (row r, channel c) inside a k-block tile image of `rows` x 64 B (64-byte swizzle, Swizzle<2,4,3>)
__device__ __forceinline__ int sw64_off(int r, int c_in_kb /*0..31*/) {
  const int byte = c_in_kb * 2;
  return r * 64 + ((((byte >> 4) ^ ((r >> 1) & 3))) << 4) + (byte & 15);
}

// ---- B operand: channels-last half pyramid level -> tile images [img][ntile][kb][256 x 64 B] -----------------------
__global__ void ct_build_b_kernel(int BS, int HW, int ntiles, const __half* __restrict__ lvl /*[BS,HW,128]*/,
                                  uint8_t* __restrict__ tiles, size_t tile_off, size_t img_stride) {
  // one thread per (img, position, 16-byte chunk of 8 channels): 16 chunks per position
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)BS * ntiles * CT_N * 16;
  if (i >= total) return;
  const int chunk = (int)(i & 15);
  const size_t pp = i >> 4;
  const int r = (int)(pp % CT_N);
  const size_t tt = pp / CT_N;
  const int t = (int)(tt % ntiles);
  const size_t img = tt / ntiles;
  const int p = t * CT_N + r;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (p < HW) v = *reinterpret_cast<const uint4*>(lvl + ((size_t)img * HW + p) * CT_C + chunk * 8);
  const int kb = chunk >> 2, cin = (chunk & 3) * 8;
  uint8_t* dst = tiles + img * img_stride + tile_off + ((size_t)t * CT_KB + kb) * (CT_N * 64) + sw64_off(r, cin);
  *reinterpret_cast<uint4*>(dst) = v;
}

// ---- A operand: float targets [BS,N,128] -> fp16 tile images [img][mtile][kb][128 x 64 B] ---------------------------
__global__ void ct_build_a_kernel(int BS, int N, int mtiles, const float* __restrict__ targets, uint8_t* __restrict__ a_tiles) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)BS * mtiles * CT_M * 16;
  if (i >= total) return;
  const int chunk = (int)(i & 15);
  const size_t pp = i >> 4;
  const int r = (int)(pp % CT_M);
  const size_t tt = pp / CT_M;
  const int m = (int)(tt % mtiles);
  const size_t img = tt / mtiles;
  const int n = m * CT_M + r;
  __half h[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) h[k] = __float2half(0.f);
  if (n < N) {
    const float4 a = *reinterpret_cast<const float4*>(targets + ((size_t)img * N + n) * CT_C + chunk * 8);
    const float4 b = *reinterpret_cast<const float4*>(targets + ((size_t)img * N + n) * CT_C + chunk * 8 + 4);
    h[0] = __float2half(a.x); h[1] = __float2half(a.y); h[2] = __float2half(a.z); h[3] = __float2half(a.w);
    h[4] = __float2half(b.x); h[5] = __float2half(b.y); h[6] = __float2half(b.z); h[7] = __float2half(b.w);
  }
  const int kb = chunk >> 2, cin = (chunk & 3) * 8;
  uint8_t* dst = a_tiles + ((img * mtiles + m) * CT_KB + kb) * (size_t)(CT_M * 64) + sw64_off(r, cin);
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(h);
}

template <int R>
__global__ void __launch_bounds__(CT_THREADS, 1)
    corr_tc_kernel(int BS, int N, int L, int mtiles, const __grid_constant__ CtLevels lv, const uint8_t* __restrict__ b_tiles,
                   const uint8_t* __restrict__ a_tiles, const float* __restrict__ coords, float* __restrict__ out) {
  constexpr int FP = 2 * R + 2, K = 2 * R + 1;
  extern __shared__ __align__(1024) uint8_t ct_smem[];
  uint8_t* base = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<size_t>(ct_smem), 1024));
  uint8_t* a_sm = base;
  uint8_t* b_sm = base + CT_A_BYTES;
  float* fb = reinterpret_cast<float*>(b_sm + (size_t)CT_STAGES * CT_B_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(fb + CT_M * CT_FB_LD);
  uint64_t* a_full = bars;            // 1
  uint64_t* a_empty = bars + 1;       // 1
  uint64_t* b_full = bars + 2;        // [2]
  uint64_t* b_empty = bars + 4;       // [2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  if (threadIdx.x == 0) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, 8);
    for (int s = 0; s < CT_STAGES; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 8);      // one arrive per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int nitems = BS * mtiles;

  if (wg == 0) {
    // ===== producer: one bulk copy per operand tile =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");     // registers go to the consumers' accumulators
    if (threadIdx.x == 0) {
      int stage = 0, phase = 0, item_no = 0;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++item_no) {
        const int img = item / mtiles;
        mbar_wait(a_empty, (uint32_t)((item_no & 1) ^ 1));
        mbar_expect_tx(a_full, CT_A_BYTES);
        tma_load_1d(a_sm, a_tiles + (size_t)item * CT_A_BYTES, CT_A_BYTES, a_full);
        for (int l = 0; l < L; ++l) {
          const uint8_t* src = b_tiles + (size_t)img * lv.img_stride + lv.tile_off[l];
          for (int t = 0; t < lv.ntiles[l]; ++t) {
            mbar_wait(&b_empty[stage], (uint32_t)(phase ^ 1));
            mbar_expect_tx(&b_full[stage], CT_B_BYTES);
            tma_load_1d(b_sm + (size_t)stage * CT_B_BYTES, src + (size_t)t * CT_B_BYTES, CT_B_BYTES, &b_full[stage]);
            if (++stage == CT_STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup half (= wg - 1) owns queries 64 half .. 64 half + 63 of the item; a thread holds the
  //       accumulators of queries q0 and q0 + 8 =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int half = wg - 1, wq = warp & 3;
  const int q0 = half * 64 + wq * 16 + (lane >> 2);
  const int cbase = 2 * (lane & 3);
  const float inv_sqrt_c = rsqrtf((float)CT_C);
  float acc[128];
  int stage = 0, phase = 0, item_no = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++item_no) {
    const int img = item / mtiles, m = item % mtiles;
    float cx0[2] = {0.f, 0.f}, cy0[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = m * CT_M + q0 + 8 * h;
      if (n < N) {
        cx0[h] = coords[((size_t)img * N + n) * 2];
        cy0[h] = coords[((size_t)img * N + n) * 2 + 1];
      }
    }
    mbar_wait(a_full, (uint32_t)(item_no & 1));
    const uint32_t a_addr = smem_u32(a_sm) + (uint32_t)half * 64u * 64u;   // 64 rows = 8 swizzle atoms
    for (int l = 0; l < L; ++l) {
      const int H = lv.H[l], W = lv.W[l], logW = lv.logW[l];
      const float scale = 1.0f / (float)(1 << l);
      int x0[2], y0[2];                                                   // footprint origins of the two queries
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        x0[h] = (int)floorf(corr_window(cx0[h] * scale, R, W)) - R;
        y0[h] = (int)floorf(corr_window(cy0[h] * scale, R, H)) - R;
      }
      for (int i = (threadIdx.x & 127); i < 64 * FP * FP; i += 128)
        fb[(half * 64 + i / (FP * FP)) * CT_FB_LD + i % (FP * FP)] = 0.f;
      wg_bar(1 + half);                                                   // table zeroed by the whole warpgroup
      for (int t = 0; t < lv.ntiles[l]; ++t) {
        mbar_wait(&b_full[stage], (uint32_t)phase);
        const uint32_t b_addr = smem_u32(b_sm + (size_t)stage * CT_B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < CT_KB; ++kb)
#pragma unroll
          for (int ks = 0; ks < 2; ++ks)
            wgmma_f16(acc, wgmma_desc_sw64(a_addr + kb * (CT_M * 64) + ks * 32), wgmma_desc_sw64(b_addr + kb * (CT_N * 64) + ks * 32),
                      (kb | ks) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive1(&b_empty[stage]);                    // the stage may be refilled
        if (++stage == CT_STAGES) { stage = 0; phase ^= 1; }
        // keep the footprint values: position p = t * 256 + column
        const int p_lo = t * CT_N, p_hi = p_lo + CT_N - 1;
        bool need[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          need[h] = (p_hi >> logW) >= y0[h] && (p_lo >> logW) < y0[h] + FP;
        if (!__any_sync(0xffffffffu, need[0] || need[1])) continue;
#pragma unroll
        for (int j = 0; j < 128; ++j) {
          const int h = (j >> 1) & 1;
          const int p = p_lo + 8 * (j >> 2) + cbase + (j & 1);
          const int dy = (p >> logW) - y0[h], dx = (p & (W - 1)) - x0[h];
          if ((unsigned)dy < (unsigned)FP && (unsigned)dx < (unsigned)FP)
            fb[(q0 + 8 * h) * CT_FB_LD + dy * FP + dx] = acc[j] * inv_sqrt_c;
        }
      }
      // ---- interpolation of the K*K taps: warp wq takes its 16 queries one at a time, lanes across the taps, so that
      //      the stores of a query are contiguous
      wg_bar(1 + half);                                                   // every footprint of the warpgroup is in
      for (int qq = 0; qq < 16; ++qq) {
        const int ql = half * 64 + wq * 16 + qq;
        const int nq = m * CT_M + ql;
        if (nq >= N) break;
        const float qcx = corr_window(coords[((size_t)img * N + nq) * 2] * scale, R, W);
        const float qcy = corr_window(coords[((size_t)img * N + nq) * 2 + 1] * scale, R, H);
        const float wx = qcx - floorf(qcx), wy = qcy - floorf(qcy);
        const float* f = fb + ql * CT_FB_LD;
        float* orow = out + ((size_t)img * N + nq) * (size_t)(L * K * K) + (size_t)l * K * K;
        for (int o = lane; o < K * K; o += 32) {
          const int a = o / K, b = o % K;
          const float d00 = f[b * FP + a], d01 = f[b * FP + a + 1], d10 = f[(b + 1) * FP + a], d11 = f[(b + 1) * FP + a + 1];
          orow[o] = d00 * (1.f - wx) * (1.f - wy) + d01 * wx * (1.f - wy) + d10 * (1.f - wx) * wy + d11 * wx * wy;
        }
      }
      wg_bar(1 + half);                                                   // tables are re-zeroed next level
    }
    __syncwarp();
    if (lane == 0) mbar_arrive1(a_empty);                                // all MMAs of the item have consumed A
  }
}

int ct_levels(int H, int W, int L, CtLevels* lv) {
  size_t off = 0;
  int h = H, w = W;
  for (int l = 0; l < L; ++l) {
    if (h <= 0 || w <= 0 || (w & (w - 1)) != 0) return -1;
    lv->H[l] = h;
    lv->W[l] = w;
    int lg = 0;
    while ((1 << lg) < w) ++lg;
    lv->logW[l] = lg;
    lv->ntiles[l] = (h * w + CT_N - 1) / CT_N;
    lv->tile_off[l] = off;
    off += (size_t)lv->ntiles[l] * CT_B_BYTES;
    h /= 2;
    w /= 2;
  }
  lv->img_stride = off;
  return 0;
}

}  // namespace

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_corr_tc_supported(int C, int H, int W, int num_levels, int radius) {
  CtLevels lv;
  return C == CT_C && num_levels >= 1 && num_levels <= 8 && (radius == 3 || radius == 4) && ct_levels(H, W, num_levels, &lv) == 0;
}

int vgg_corr_tc_bytes(int BS, int C, int H, int W, int num_levels, int N, size_t* tile_bytes, size_t* target_bytes) {
  VGG_REQUIRE(BS > 0 && N >= 0, "bad sizes");
  CtLevels lv;
  VGG_REQUIRE(C == CT_C && num_levels >= 1 && num_levels <= 8 && ct_levels(H, W, num_levels, &lv) == 0,
              "tensor-core correlation: C must be 128 and the map width a power of two");
  if (tile_bytes) *tile_bytes = (size_t)BS * lv.img_stride;
  if (target_bytes) *target_bytes = (size_t)BS * ((N + CT_M - 1) / CT_M) * CT_A_BYTES;
  return VGG_OK;
}

int vgg_corr_tc_build(int BS, int C, int H, int W, int num_levels, const void* pyramid_half, void* tiles, void* stream) {
  VGG_REQUIRE(pyramid_half && tiles, "null pointer");
  CtLevels lv;
  VGG_REQUIRE(C == CT_C && ct_levels(H, W, num_levels, &lv) == 0, "tensor-core correlation: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  const char* p = reinterpret_cast<const char*>(pyramid_half);
  for (int l = 0; l < num_levels; ++l) {
    const int HW = lv.H[l] * lv.W[l];
    const size_t total = (size_t)BS * lv.ntiles[l] * CT_N * 16;
    ct_build_b_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(BS, HW, lv.ntiles[l], reinterpret_cast<const __half*>(p),
                                                                      reinterpret_cast<uint8_t*>(tiles), lv.tile_off[l],
                                                                      lv.img_stride);
    VGG_LAUNCH_CHECK();
    p += align_up((size_t)BS * HW * C * 2, 256);      // level stride of vgg_corr_build_pyramid (elem_size 2)
  }
  return VGG_OK;
}

int vgg_corr_tc_sample(int BS, int N, int C, int H, int W, int num_levels, int radius, const void* tiles, const float* targets,
                       const float* coords, void* target_tiles, float* out, void* stream) {
  VGG_REQUIRE(BS >= 0 && N >= 0, "bad sizes");
  VGG_REQUIRE(radius == 3 || radius == 4, "tensor-core correlation: radius 3 or 4");
  CtLevels lv;
  VGG_REQUIRE(C == CT_C && ct_levels(H, W, num_levels, &lv) == 0, "tensor-core correlation: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  if (BS == 0 || N == 0) return VGG_OK;                // nothing to sample: empty tensors may pass null pointers
  VGG_REQUIRE(tiles && targets && coords && target_tiles && out, "null pointer");
  const int mtiles = (N + CT_M - 1) / CT_M;
  {
    const size_t total = (size_t)BS * mtiles * CT_M * 16;
    ct_build_a_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(BS, N, mtiles, targets, reinterpret_cast<uint8_t*>(target_tiles));
    VGG_LAUNCH_CHECK();
  }
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    VGG_CUDA_CHECK(cudaGetDevice(&dev));
    VGG_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    VGG_CUDA_CHECK(cudaFuncSetAttribute(corr_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CT_SMEM));
    VGG_CUDA_CHECK(cudaFuncSetAttribute(corr_tc_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CT_SMEM));
  }
  const int grid = std::min(sms, BS * mtiles);
  if (radius == 4)
    corr_tc_kernel<4><<<grid, CT_THREADS, CT_SMEM, st>>>(BS, N, num_levels, mtiles, lv, reinterpret_cast<const uint8_t*>(tiles),
                                                        reinterpret_cast<const uint8_t*>(target_tiles), coords, out);
  else
    corr_tc_kernel<3><<<grid, CT_THREADS, CT_SMEM, st>>>(BS, N, num_levels, mtiles, lv, reinterpret_cast<const uint8_t*>(tiles),
                                                        reinterpret_cast<const uint8_t*>(target_tiles), coords, out);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // extern "C"
