// Block-scaled e4m3 quantisers of the fp8 fully-connected path (compute_type "fp8").
//
// Scale rule (oracle: utils/mxfp8.py::block_exponent): a block's scale is 2^e, e the smallest
// integer with amax <= 448 * 2^e, computed from the exponent and mantissa bits of amax and clamped
// to [-127, 127]; an all-zero block gets e = -127. A code is the e4m3 value of x * 2^-e (round to
// nearest even, saturating); the power-of-two scale makes the product exact, so the codes equal the
// oracle's bit for bit.
//
// Scales are fp32 2^e, stored k-block-major [KB][rows_pad] with rows_pad = rows rounded up to 128:
// the GEMM's producer fetches one stage's 128 scales with one bulk copy. Padding rows hold the
// all-zero scale 2^-127.
//
// One kernel, one 128 x 128 tile per CTA, the tile read once:
// * quant_act   (bf16 in): row-block codes [rows][ldq] (1 x 128 blocks along cols) and / or
//   transposed column-block codes [cols][ldqt] (1 x 128 blocks along rows);
// * quant_weight (fp32 in): one scale per 128 x 128 tile, codes in both layouts, so W and W^T
//   carry the same quantised weight.
#include "common.cuh"
#include <cuda_fp8.h>

namespace zn {
namespace f8 {

constexpr int T = 128;           // tile edge = scale block
constexpr int WARPS = 8;         // warp w: tile rows 16 w .. 16 w + 15; lane l: columns 4 l .. 4 l + 3
constexpr int RPW = T / WARPS;
constexpr int TP = T + 4;        // byte pitch of the transpose buffer

__device__ __forceinline__ int block_exp(float amax) {
  const uint32_t b = __float_as_uint(amax);
  const int ef = (b >> 23) & 0xff;
  if (ef == 0) return -127;                       // zero or subnormal block maximum
  // amax = m 2^E, m in [1, 2): m <= 1.75 (448 = 1.75 2^8) -> e = E - 8, else E - 7
  const int e = ef - 127 - 8 + ((b & 0x7fffffu) > 0x600000u ? 1 : 0);
  return max(-127, min(127, e));
}
__device__ __forceinline__ float pow2i(int e) {   // exact 2^e, e in [-127, 127]
  return e >= -126 ? __uint_as_float((uint32_t)(e + 127) << 23) : __uint_as_float(0x00400000u);
}
__device__ __forceinline__ uint32_t e4m3(float v) {
  return (uint32_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}

template <typename TI>
__device__ __forceinline__ void load4(const TI* p, bool vec, int left, float (&v)[4]);
template <>
__device__ __forceinline__ void load4<float>(const float* p, bool vec, int left, float (&v)[4]) {
  if (vec && left >= 4) {
    const float4 u = *reinterpret_cast<const float4*>(p);
    v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < left ? p[j] : 0.f;
  }
}
template <>
__device__ __forceinline__ void load4<__nv_bfloat16>(const __nv_bfloat16* p, bool vec, int left,
                                                     float (&v)[4]) {
  if (vec && left >= 4) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < left ? __bfloat162float(p[j]) : 0.f;
  }
}

// 4 codes -> bytes dst[0..n) (n = 4: one aligned 32-bit store)
__device__ __forceinline__ void store4(uint8_t* dst, uint32_t packed, int n) {
  if (n >= 4) {
    *reinterpret_cast<uint32_t*>(dst) = packed;
  } else {
    for (int j = 0; j < n; ++j) dst[j] = (uint8_t)(packed >> (8 * j));
  }
}

template <typename TI>
__global__ void __launch_bounds__(WARPS * 32)
quant_k(const TI* __restrict__ x, long long ldx, int rows, int cols, int tile,
        uint8_t* __restrict__ q, long long ldq, float* __restrict__ sq,
        uint8_t* __restrict__ qt, long long ldqt, float* __restrict__ sqt) {
  __shared__ float red[WARPS][T];
  __shared__ float tscale[T];
  __shared__ __align__(16) uint8_t tt[T * TP];
  pdl_entry();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.y * T, c0 = blockIdx.x * T;
  const int c = c0 + 4 * lane;
  const int rows_pad = (rows + T - 1) / T * T, cols_pad = (cols + T - 1) / T * T;
  const bool vec = (ldx % 4 == 0) && (((uintptr_t)x & 15) == 0);
  float v[RPW][4];
#pragma unroll
  for (int i = 0; i < RPW; ++i) {
    const int r = r0 + warp * RPW + i;
    if (r < rows && c < cols) {
      load4<TI>(x + (long long)r * ldx + c, vec, cols - c, v[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) v[i][j] = 0.f;
    }
  }
  float cmax[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < RPW; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) cmax[j] = fmaxf(cmax[j], fabsf(v[i][j]));

  int te = 0;
  if (tile) {
    float m = fmaxf(fmaxf(cmax[0], cmax[1]), fmaxf(cmax[2], cmax[3]));
    m = warp_max(m);
    if (lane == 0) red[warp][0] = m;
    __syncthreads();
    m = red[0][0];
#pragma unroll
    for (int w = 1; w < WARPS; ++w) m = fmaxf(m, red[w][0]);
    te = block_exp(m);
    __syncthreads();
  }

  if (q != nullptr) {
    // row blocks: scale of tile row r = max over the 128 columns of this tile
    const int kb = blockIdx.x;
#pragma unroll
    for (int i = 0; i < RPW; ++i) {
      const int r = r0 + warp * RPW + i;
      int e = te;
      if (!tile) {
        float m = fmaxf(fmaxf(fabsf(v[i][0]), fabsf(v[i][1])), fmaxf(fabsf(v[i][2]), fabsf(v[i][3])));
        e = block_exp(warp_max(m));
      }
      if (lane == 0) sq[(long long)kb * rows_pad + r] = pow2i(e);
      const float inv = pow2i(-e);
      if (r < rows && c < cols) {
        const uint32_t packed = e4m3(v[i][0] * inv) | (e4m3(v[i][1] * inv) << 8) |
                                (e4m3(v[i][2] * inv) << 16) | (e4m3(v[i][3] * inv) << 24);
        store4(q + (long long)r * ldq + c, packed, cols - c);
      }
    }
  }

  if (qt != nullptr) {
    // column blocks: scale of tile column c = max over the 128 rows of this tile
    if (!tile) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red[warp][4 * lane + j] = cmax[j];
      __syncthreads();
      if (threadIdx.x < T) {
        float m = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) m = fmaxf(m, red[w][threadIdx.x]);
        tscale[threadIdx.x] = (float)block_exp(m);
      }
      __syncthreads();
    }
    float inv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int e = tile ? te : (int)tscale[4 * lane + j];
      inv[j] = pow2i(-e);
      if (warp == 0) sqt[(long long)blockIdx.y * cols_pad + c + j] = pow2i(e);
    }
#pragma unroll
    for (int i = 0; i < RPW; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        tt[(4 * lane + j) * TP + warp * RPW + i] = (uint8_t)e4m3(v[i][j] * inv[j]);
    __syncthreads();
    // transposed rows: tile column cc -> qt[c0 + cc][r0 .. r0 + 127], 4 bytes per lane
    const int rr = r0 + 4 * lane;
#pragma unroll 4
    for (int k = 0; k < RPW; ++k) {
      const int cc = warp * RPW + k;
      if (c0 + cc < cols && rr < rows)
        store4(qt + (long long)(c0 + cc) * ldqt + rr,
               *reinterpret_cast<const uint32_t*>(tt + cc * TP + 4 * lane), rows - rr);
    }
  }
}

}  // namespace f8

// x [rows][ldx] (bf16 when !x_f32, else fp32). q / sq: row-block codes [rows][ldq] and scales
// [ceil(cols / 128)][rows_pad]; qt / sqt: transposed column-block codes [cols][ldqt] and scales
// [ceil(rows / 128)][cols_pad]; either pair may be null. tile != 0: one scale per 128 x 128 tile.
// Returns 0, or non-zero (nothing launched) on a shape / alignment the kernel does not serve.
int launch_fp8_quant(const void* x, int x_f32, long long ldx, int rows, int cols, int tile,
                     uint8_t* q, long long ldq, float* sq, uint8_t* qt, long long ldqt, float* sqt,
                     cudaStream_t st) {
  using namespace f8;
  if (rows < 1 || cols < 1 || ldx < cols) return -6;
  if (q == nullptr && qt == nullptr) return -6;
  if (q != nullptr && ((ldq % 16) || ldq < cols || ((uintptr_t)q & 15) || sq == nullptr)) return -3;
  if (qt != nullptr && ((ldqt % 16) || ldqt < rows || ((uintptr_t)qt & 15) || sqt == nullptr)) return -3;
  const dim3 grid((cols + T - 1) / T, (rows + T - 1) / T);
  cudaError_t e;
  if (x_f32)
    e = launch_k(quant_k<float>, grid, dim3(WARPS * 32), 0, st, (const float*)x, ldx, rows, cols,
                 tile, q, ldq, sq, qt, ldqt, sqt);
  else
    e = launch_k(quant_k<__nv_bfloat16>, grid, dim3(WARPS * 32), 0, st, (const __nv_bfloat16*)x, ldx,
                 rows, cols, tile, q, ldq, sq, qt, ldqt, sqt);
  return (int)e;
}

}  // namespace zn
