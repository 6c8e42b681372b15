// wgmma / TMA GEMM family for sm_90a (bf16 operands, fp32 accumulate in registers).
//
//   D[M, N] = sum_k A[m, k] * B[n, k]      (one 128 x BLOCK_N tile per CTA, optional split-K)
//
// Operand sources (template):
//   A_TMA_K   A stored [M][K] (K contiguous)  -> TMA box {64, 128}, K-major SW128 descriptor
//   A_TMA_MN  A stored [K][M] (M contiguous)  -> TMA boxes {64, 64}, MN-major SW128 descriptor
//   A_GATHER_K / A_GATHER_MN: implicit-GEMM convolution; producer warps gather NHWC patches
//   (im2col of x, or the dgrad gather of err_out) as 16-byte chunks straight into the swizzled
//   shared-memory tile — no im2col buffer in HBM (the reference unpacks 16 images at a time into
//   a temp buffer and calls cuBLAS, /root/reference/conv.py:268-297, gd_conv.py:313-423).
//   B_TMA_K   B stored [N][K];  B_TMA_MN  B stored [K][N].
//
// Warp roles: warpgroup 0 (warps 0-3) issues the wgmma for both 64-row halves of the tile, then
// runs the epilogue (registers -> shared memory -> bias/activation/alpha-beta -> global); its
// thread 0 issues the TMA loads. Gather kernels add warpgroup 1 (warps 4-7) as producers.
// 4-stage smem ring (3 stages for short gather reductions, see launch_cfg).
//
// This covers: FC forward (TMA_K x TMA_K, fused bias+activation), FC dgrad (TMA_K x TMA_MN,
// alpha/beta), FC wgrad (TMA_MN x TMA_MN), conv fprop (GATHER_K x TMA_K, fused bias+act),
// conv dgrad (GATHER_K x TMA_MN, no atomics), conv wgrad (GATHER_MN or HALO_MN x TMA_MN, split-K
// partials that the fused update kernel sums in fixed order).
#include "common.cuh"
#include "umma.cuh"
#include <stdlib.h>

namespace zn {

using namespace umma;

// A_IM2COL_K: the same implicit-GEMM operand as A_GATHER_K, but fetched by TMA in im2col mode
// (one instruction per [128 pixels x 64 channels] block instead of a 128-thread LDGSTS gather) -
// channel counts that are multiples of 64 only.
// A_HALO: stride-1 conv fprop / dgrad whose inner channel count is 8, 16 or 32 (tap mode with
// tpk >= 2). Each 64-row half of the tile is one 8x8 block of output (dgrad: input) pixels; the
// block's (8 + KY - 1) x (8 + KX - 1) input window is loaded ONCE by TMA into shared memory as
// planes [C / 8][halo_y][halo_x][8 channels], and every k16 step points a no-swizzle A
// descriptor into it: a core matrix (8 pixels of one block row x 8 channels) is 128 contiguous
// bytes of a plane, SBO = one halo row. The tap-mode gather instead fetches each input byte once
// per filter tap (25x for 5x5). The k16 steps issue the same products in the same order as the
// gather, so the results are bit-identical.
// A_HALO_MN: the conv weight gradient's im2col operand (M = kidx, K = pixels) for the same stride-1,
// 8 / 16 / 32-channel geometries. A k-block (64 consecutive pixels = 64 / OW whole output rows, or
// a 64-pixel row segment) needs one band of the input, (rows + KY - 1) x (cols + KX - 1) pixels,
// loaded by TMA per 8-channel plane into each ring stage next to the err tile. The A operand is
// MN-major without swizzle: a core matrix (8 pixels x 8 channels) is 128 contiguous bytes of a
// plane, and the 8 core matrices along M of one m64 wgmma are the 8 kx slots of one (plane, ky)
// "group", 16 bytes apart (slots >= KX read neighbouring pixels and are dropped). Every pixel
// k16 step of the gather is issued unchanged, so the results are bit-identical to it.
enum { A_TMA_K = 0, A_TMA_MN = 1, A_GATHER_K = 2, A_GATHER_MN = 3, A_IM2COL_K = 4, A_HALO = 5,
       A_HALO_MN = 6 };
enum { B_TMA_K = 0, B_TMA_MN = 1 };
enum { G_NONE = 0, G_IM2COL = 1, G_DGRAD = 2 };

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // bf16 elements = 128 bytes = one SW128 row
constexpr int STAGES_DEFAULT = 4;   // 3 for short gather reductions: see launch_cfg
constexpr int A_BYTES = BLOCK_M * 128;
constexpr int HALO_MAX_BYTES = 32 * 1024;   // one block's halo (A_HALO), at most
constexpr int BAND_MAX_BYTES = 16 * 1024;   // the planes of one ring stage's band (A_HALO_MN), at most
constexpr int BAND_GROUPS = 3;              // A_HALO_MN: m64 groups (accumulator sets) per CTA

struct ConvGeomU {
  int N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL;
  int vec;   // 1 when 16-byte chunks never straddle a tap (C % 8 == 0 resp. F % 8 == 0)
  // tap mode (GVEC == 2): a 64-wide block of the reduction index covers ``tpk`` whole taps
  // (inner = 64 / tpk channels each) or a 64-channel slice of one tap (tpk == 1, inner % 64 == 0)
  int tpk, ntaps, inner;
  // wgrad only: 16 bytes holding bf16 {1, 0, 0, 0, 0, 0, 0, 0}. The gathered im2col operand gets a
  // "ones" row at reduction-weight index Kw (first padding row of the last M tile), so that
  // row Kw of the product is sum_pixels err[pixel][f] = the bias gradient - for free.
  const __nv_bfloat16* ones;
};

struct GemmParams {
  int M, N, K;                 // logical GEMM sizes (K = reduction)
  int k_blocks_per_split;      // in BLOCK_K units
  // epilogue
  void* out; int out_bf16; long long ldo; int out_trans;
  const float* bias; int act; float alpha, beta;
  float* bias_out;             // wgrad: row M of the product -> bias_out[blockIdx.z][N] (see ones)
  const __nv_bfloat16* dmul;   // dgrad: out *= f'(dmul[row][col]) - the producer layer's activation
  int dact;                    //        derivative (dmul = this layer's input, same layout as out)
  long long split_stride;      // > 0: fp32 partial [blockIdx.z][...]
  // gather source
  const __nv_bfloat16* gsrc; ConvGeomU g; int gather_kind;
  int gK;                      // valid extent of the gathered K (fprop/dgrad) or M (wgrad) index
  int ktab_n;                  // entries of the gather lookup table (dynamic shared memory)
  // A_HALO: 8x8 pixel blocks per image row / column, and the bytes one block's halo occupies
  // (A_HALO_MN: the bytes of one ring stage's band)
  int hnbx, hnby, hbytes;
  // A_HALO_MN: band width / height in pixels, bytes per plane, (plane, ky) groups, and groups
  // including the bias group (one more when bias_out is set)
  int bw, bh, bplane, bgroups, bvgroups;
};

// ---- gather: 8 consecutive "inner" indices of one "pixel" -> 16 bytes ------------------------
// All div/mod of the reduction index is hoisted into a per-CTA shared-memory table built once:
// vec mode   : ktab[k / 8] = (ky << 24) | (kx << 16) | c0     (16-byte chunks never straddle a tap)
// scalar mode: ktab[k]     = (ky << 24) | (kx << 16) | c
constexpr int KTAB = 4096;

struct PixCtx { const __nv_bfloat16* base; int y, x, valid; };

__device__ __forceinline__ PixCtx decode_out_pixel(const __nv_bfloat16* src, const ConvGeomU& g,
                                                   int pix, int limit) {
  // im2col source = x [N,H,W,C]; (y, x) = top-left input coordinate of the patch
  PixCtx c; c.valid = pix < limit;
  const int p = c.valid ? pix : 0;
  const int ox = p % g.OW; const int t = p / g.OW; const int oy = t % g.OH; const int n = t / g.OH;
  c.y = oy * g.SY - g.PT; c.x = ox * g.SX - g.PL;
  c.base = src + (long long)n * g.H * g.W * g.C;
  return c;
}
__device__ __forceinline__ PixCtx decode_in_pixel(const __nv_bfloat16* src, const ConvGeomU& g,
                                                  int pix, int limit) {
  // dgrad source = err_out [N,OH,OW,F]; (y, x) = input pixel + padding
  PixCtx c; c.valid = pix < limit;
  const int p = c.valid ? pix : 0;
  const int ix = p % g.W; const int t = p / g.W; const int iy = t % g.H; const int n = t / g.H;
  c.y = iy + g.PT; c.x = ix + g.PL;
  c.base = src + (long long)n * g.OH * g.OW * g.F;
  return c;
}
__device__ __forceinline__ void build_ktab(int* ktab, const ConvGeomU& g, int kind, int klimit) {
  if (g.tpk > 0) {                                // tap mode: ktab[tap] = (ky << 8) | kx
    for (int e = threadIdx.x; e < g.ntaps; e += blockDim.x)
      ktab[e] = ((e / g.KX) << 8) | (e % g.KX);
    return;
  }
  const int inner = (kind == 1) ? g.C : g.F;      // G_IM2COL : G_DGRAD
  const int step = g.vec ? 8 : 1;
  const int n = min(KTAB, (klimit + step - 1) / step);
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int k = e * step;
    const int c = k % inner; const int tap = k / inner;
    const int kx = tap % g.KX; const int ky = tap / g.KX;
    ktab[e] = (ky << 24) | (kx << 16) | c;
  }
}
__device__ __forceinline__ const __nv_bfloat16* im2col_addr(const ConvGeomU& g, const PixCtx& c, int e) {
  const int iy = c.y + (e >> 24), ix = c.x + ((e >> 16) & 0xff);
  if ((unsigned)iy >= (unsigned)g.H || (unsigned)ix >= (unsigned)g.W) return nullptr;
  return c.base + (iy * g.W + ix) * g.C + (e & 0xffff);
}
__device__ __forceinline__ const __nv_bfloat16* dgrad_addr(const ConvGeomU& g, const PixCtx& c, int e) {
  int ty = c.y - (e >> 24), tx = c.x - ((e >> 16) & 0xff);
  if (g.SY != 1 || g.SX != 1) {
    if (ty < 0 || tx < 0 || (ty % g.SY) || (tx % g.SX)) return nullptr;
    ty /= g.SY; tx /= g.SX;
  }
  if ((unsigned)ty >= (unsigned)g.OH || (unsigned)tx >= (unsigned)g.OW) return nullptr;
  return c.base + (ty * g.OW + tx) * g.F + (e & 0xffff);
}
template <int KIND, int VEC>
__device__ __forceinline__ uint4 gather_chunk(const int* ktab, const ConvGeomU& g, const PixCtx& c,
                                              int k0, int klimit) {
  uint4 z = make_uint4(0, 0, 0, 0);
  if (!c.valid || k0 >= klimit) return z;
  if (VEC) {
    const __nv_bfloat16* p = (KIND == 1) ? im2col_addr(g, c, ktab[k0 >> 3]) : dgrad_addr(g, c, ktab[k0 >> 3]);
    return p ? *reinterpret_cast<const uint4*>(p) : z;
  }
  __nv_bfloat16 v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = k0 + j;
    const __nv_bfloat16* p = nullptr;
    if (k < klimit) p = (KIND == 1) ? im2col_addr(g, c, ktab[k]) : dgrad_addr(g, c, ktab[k]);
    v[j] = p ? *p : __float2bfloat16_rn(0.f);
  }
  return *reinterpret_cast<uint4*>(v);
}

// Tap-mode gather: the 8 chunks (64 reduction indices starting at k0, k0 % 64 == 0) of one pixel.
// One table lookup + one bounds check + one address per *tap*; the chunks of a tap are
// consecutive 16-byte loads. ~6 instructions per chunk instead of ~100 for the generic path.
template <int KIND, int TPK>
__device__ __forceinline__ void gather_taps(uint4 (&nv)[8], const int* ttab, const ConvGeomU& g,
                                            const PixCtx& c, int k0) {
  constexpr int CPT = 8 / TPK;
  int tap0, c0;
  if (TPK == 1) { tap0 = k0 / g.inner; c0 = k0 - tap0 * g.inner; }
  else { tap0 = (k0 >> 6) * TPK; c0 = 0; }
  const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int j = 0; j < TPK; ++j) {
    const int tap = tap0 + j;
    bool ok = c.valid && tap < g.ntaps;
    const int e = ttab[ok ? tap : 0];
    const int ky = e >> 8, kx = e & 0xff;
    int off;
    if (KIND == G_IM2COL) {
      const int iy = c.y + ky, ix = c.x + kx;
      ok = ok && (unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W;
      off = (iy * g.W + ix) * g.C;
    } else {                                      // dgrad, unit stride only
      const int ty = c.y - ky, tx = c.x - kx;
      ok = ok && (unsigned)ty < (unsigned)g.OH && (unsigned)tx < (unsigned)g.OW;
      off = (ty * g.OW + tx) * g.F;
    }
    const uint4* ptr = reinterpret_cast<const uint4*>(c.base + (ok ? off + c0 : 0));
#pragma unroll
    for (int q = 0; q < CPT; ++q) nv[j * CPT + q] = ok ? ptr[q] : z;
  }
}
// Asynchronous variant: the same taps, but every 16-byte chunk is an LDGSTS (cp.async) straight
// into its swizzled shared-memory slot (row_base + ((c8 ^ sw) << 4)); out-of-image chunks are
// zero-filled by the copy itself. No registers are staged and the thread never waits for global
// memory: the stage's full-barrier gets this thread's arrival when its copies have landed, so
// up to STAGES k-blocks of gathers are in flight per thread.
template <int KIND, int TPK, bool ONES = false>
__device__ __forceinline__ void gather_taps_async(uint32_t row_base, int sw, const int* ttab,
                                                  const ConvGeomU& g, const PixCtx& c, int k0) {
  constexpr int CPT = 8 / TPK;
  int tap0, c0;
  if (TPK == 1) { tap0 = k0 / g.inner; c0 = k0 - tap0 * g.inner; }
  else { tap0 = (k0 >> 6) * TPK; c0 = 0; }
#pragma unroll
  for (int j = 0; j < TPK; ++j) {
    const int tap = tap0 + j;
    bool ok = c.valid && tap < g.ntaps;
    const int e = ttab[ok ? tap : 0];
    const int ky = e >> 8, kx = e & 0xff;
    int off;
    if (KIND == G_IM2COL) {
      const int iy = c.y + ky, ix = c.x + kx;
      ok = ok && (unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W;
      off = (iy * g.W + ix) * g.C;
    } else {
      const int ty = c.y - ky, tx = c.x - kx;
      ok = ok && (unsigned)ty < (unsigned)g.OH && (unsigned)tx < (unsigned)g.OW;
      off = (ty * g.OW + tx) * g.F;
    }
    // ONES: this 64-wide block holds reduction-weight index Kw (see ConvGeomU::ones) - only the
    // wgrad kernel instantiates it, and only for the one block of the last M tile that needs it
    const bool one = ONES && c.valid && tap == g.ntaps && c0 == 0;
    const __nv_bfloat16* ptr = one ? g.ones : c.base + (ok ? off + c0 : 0);
    const uint32_t nbytes = ok ? 16u : 0u;
#pragma unroll
    for (int q = 0; q < CPT; ++q) {
      const int c8 = j * CPT + q;
      cp_async_16(row_base + (uint32_t)((c8 ^ sw) << 4), one ? ptr : ptr + q * 8,
                  (one && q == 0) ? 16u : nbytes);
    }
  }
}
template <int KIND, bool ONES = false>
__device__ __forceinline__ void gather_row_async(uint32_t row_base, int sw, const int* ktab,
                                                 const ConvGeomU& g, const PixCtx& c, int k0) {
  switch (g.tpk) {
    case 1: gather_taps_async<KIND, 1, ONES>(row_base, sw, ktab, g, c, k0); break;
    case 2: gather_taps_async<KIND, 2, ONES>(row_base, sw, ktab, g, c, k0); break;
    case 4: gather_taps_async<KIND, 4, ONES>(row_base, sw, ktab, g, c, k0); break;
    default: gather_taps_async<KIND, 8, ONES>(row_base, sw, ktab, g, c, k0); break;
  }
}

template <int KIND, int GVEC>
__device__ __forceinline__ void gather_row(uint4 (&nv)[8], const int* ktab, const ConvGeomU& g,
                                           const PixCtx& c, int k0, int klimit) {
  if (GVEC == 2) {
    switch (g.tpk) {
      case 1: gather_taps<KIND, 1>(nv, ktab, g, c, k0); break;
      case 2: gather_taps<KIND, 2>(nv, ktab, g, c, k0); break;
      case 4: gather_taps<KIND, 4>(nv, ktab, g, c, k0); break;
      default: gather_taps<KIND, 8>(nv, ktab, g, c, k0); break;
    }
  } else {
#pragma unroll
    for (int c8 = 0; c8 < 8; ++c8) nv[c8] = gather_chunk<KIND, GVEC>(ktab, g, c, k0 + c8 * 8, klimit);
  }
}

// ---- A_HALO geometry ---------------------------------------------------------------------------
// One plane (8 channels) of a block's halo, padded to the 128-byte alignment of a TMA destination.
__host__ __device__ __forceinline__ int halo_plane_bytes(const ConvGeomU& g) {
  return ((8 + g.KY - 1) * (8 + g.KX - 1) * 16 + 127) & ~127;
}
// Per k16 step s of the reduction: (LBO << 16) | byte offset of the step's first core matrix in a
// block's halo. The step covers reduction indices 16 s .. 16 s + 15, laid out as the tap-mode
// gather lays them out: tpk = 8: taps 2 s and 2 s + 1, 8 channels each (LBO = distance between the
// two taps' windows); tpk = 4: tap s, planes 0 and 1; tpk = 2: tap s / 2, planes 2 (s % 2) and
// 2 (s % 2) + 1 (LBO = one plane). Padding taps (>= KY * KX, zero rows of B) read the last real
// tap: finite data, so 0 x A stays 0.
template <int KIND>
__device__ __forceinline__ void build_halo_tab(int* tab, const GemmParams& p) {
  const ConvGeomU& g = p.g;
  const int hx = 8 + g.KX - 1, plane = halo_plane_bytes(g);
  auto off = [&](int t) {
    t = min(t, g.ntaps - 1);
    int ky = t / g.KX, kx = t - ky * g.KX;
    if (KIND == G_DGRAD) { ky = g.KY - 1 - ky; kx = g.KX - 1 - kx; }   // correlation, flipped taps
    return (ky * hx + kx) * 16;
  };
  for (int s = threadIdx.x; s < p.ktab_n; s += blockDim.x) {
    int a, lbo;
    if (g.tpk == 8) { a = off(2 * s); lbo = off(2 * s + 1) - a; }
    else if (g.tpk == 4) { a = off(s); lbo = plane; }
    else { a = (s & 1) * 2 * plane + off(s >> 1); lbo = plane; }
    tab[s] = (lbo << 16) | a;
  }
}
// GEMM row (output pixel; dgrad: input pixel) of row r of 8x8 block b, or -1 outside the image
template <int KIND>
__device__ __forceinline__ int halo_row(const GemmParams& p, int b, int r) {
  const ConvGeomU& g = p.g;
  const int bx = b % p.hnbx, b2 = b / p.hnbx, by = b2 % p.hnby, n = b2 / p.hnby;
  const int PH = KIND == G_IM2COL ? g.OH : g.H, PW = KIND == G_IM2COL ? g.OW : g.W;
  const int y = by * 8 + (r >> 3), x = bx * 8 + (r & 7);
  return (n < g.N && y < PH && x < PW) ? (n * PH + y) * PW + x : -1;
}
// TMA loads of block b's (8 + KY - 1) x (8 + KX - 1) input window into dst, one 8-channel plane
// per box, completing on bar (the caller arms it with halo_tx_bytes); out-of-image positions
// (padding, ragged edges, a block past the last image) arrive as zeros
template <int KIND>
__device__ __forceinline__ void load_halo(uint8_t* dst, const CUtensorMap* tmap, uint64_t* bar,
                                          const GemmParams& p, int b) {
  const ConvGeomU& g = p.g;
  const int nplanes = (KIND == G_IM2COL ? g.C : g.F) / 8, plane = halo_plane_bytes(g);
  const int bx = b % p.hnbx, b2 = b / p.hnbx, by = b2 % p.hnby, n = b2 / p.hnby;
  // fprop: output pixel (y, x) with tap (ky, kx) reads x[y + ky - PT][x + kx - PL];
  // dgrad: input pixel (y, x) reads err_out[y + PT - ky][x + PL - kx]
  const int x0 = KIND == G_IM2COL ? bx * 8 - g.PL : bx * 8 + g.PL - (g.KX - 1);
  const int y0 = KIND == G_IM2COL ? by * 8 - g.PT : by * 8 + g.PT - (g.KY - 1);
#pragma unroll 1
  for (int c = 0; c < nplanes; ++c) tma_load_4d(dst + c * plane, tmap, bar, c * 8, x0, y0, n);
}
template <int KIND>
__device__ __forceinline__ uint32_t halo_tx_bytes(const GemmParams& p) {
  const ConvGeomU& g = p.g;
  return (uint32_t)((KIND == G_IM2COL ? g.C : g.F) / 8) * (8 + g.KY - 1) * (8 + g.KX - 1) * 16;
}

template <int BLOCK_N, int B_MODE>
__host__ __device__ constexpr int b_bytes() {
  return B_MODE == B_TMA_K ? BLOCK_N * 128 : ((BLOCK_N + 63) / 64) * 8192;
}

// generic (rare) epilogue element: split-K partials, transposed / fp32 / alpha-beta outputs.
// Deliberately not inlined: keeps the unrolled epilogue small.
__device__ __noinline__ void epi_store_slow(const GemmParams& p, int row, int n, float v, int z) {
  const long long o = p.out_trans ? (long long)n * p.ldo + row : (long long)row * p.ldo + n;
  if (p.split_stride > 0) {
    reinterpret_cast<float*>(p.out)[(long long)z * p.split_stride + o] = v;
    return;
  }
  v *= p.alpha;
  if (p.bias) v += p.bias[n];
  v = act_fwd5(p.act, v);
  if (p.out_bf16) {
    __nv_bfloat16* q = reinterpret_cast<__nv_bfloat16*>(p.out) + o;
    if (p.beta != 0.f) v += p.beta * __bfloat162float(*q);
    *q = __float2bfloat16_rn(v);
  } else {
    float* q = reinterpret_cast<float*>(p.out) + o;
    if (p.beta != 0.f) v += p.beta * *q;
    *q = v;
  }
}

// A_HALO_MN epilogue: the three groups' accumulators go through shared memory (stg, the idle ring)
// as rows [group][slot][channel]; row (slot, channel) of group (plane, ky) is kidx
// (ky * KX + slot) * C + plane * 8 + channel of partials[z][f][kidx], slots >= KX are dropped, and
// row 0 of the bias group is bias_out[z][f]. Consecutive threads take consecutive rows, so that
// a column's stores are runs of consecutive kidx. Empty splits store their zeros like the others.
template <int BLOCK_N>
__device__ __forceinline__ void band_epilogue(const GemmParams& p, float* stg, const float (&a0)[BLOCK_N / 2],
                                              const float (&a1)[BLOCK_N / 2], const float (&a2)[BLOCK_N / 2]) {
  constexpr int SROW = BLOCK_N + 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = r0 + 8 * hh, c = 8 * i + cq, e = 4 * i + 2 * hh;
      *reinterpret_cast<float2*>(stg + r * SROW + c) = make_float2(a0[e], a0[e + 1]);
      *reinterpret_cast<float2*>(stg + (64 + r) * SROW + c) = make_float2(a1[e], a1[e + 1]);
      *reinterpret_cast<float2*>(stg + (128 + r) * SROW + c) = make_float2(a2[e], a2[e + 1]);
    }
  }
  named_bar_sync(1, 128);
  const ConvGeomU& g = p.g;
  const int n0 = blockIdx.x * BLOCK_N, ncols = min(BLOCK_N, p.N - n0);
  float* const rbase = reinterpret_cast<float*>(p.out) + (long long)blockIdx.z * p.split_stride;
#pragma unroll 1
  for (int row = threadIdx.x; row < BAND_GROUPS * 64; row += 128) {
    const int gv = blockIdx.y * BAND_GROUPS + (row >> 6), slot = (row >> 3) & 7, ch = row & 7;
    const float* const srow = stg + row * SROW;
    if (gv < p.bgroups) {
      if (slot >= g.KX) continue;
      const int pl = gv / g.KY, ky = gv - pl * g.KY;
      float* const q = rbase + (long long)n0 * p.ldo + (ky * g.KX + slot) * g.C + pl * 8 + ch;
#pragma unroll 4
      for (int c = 0; c < ncols; ++c) q[(long long)c * p.ldo] = srow[c];
    } else if (gv == p.bgroups && (row & 63) == 0 && p.bias_out) {
      for (int c = 0; c < ncols; ++c) p.bias_out[(long long)blockIdx.z * p.N + n0 + c] = srow[c];
    }
  }
}

// The accumulator fragment of one m64 wgmma (warpgroup thread t = threadIdx.x % 128) -> rows
// row0 .. row0 + 63 of the fp32 staging [rows][BLOCK_N + 4] (the pad makes the row reads of 8
// consecutive threads hit distinct banks)
template <int BLOCK_N>
__device__ __forceinline__ void stage_acc(float* stg, int row0, const float (&acc)[BLOCK_N / 2]) {
  constexpr int SROW = BLOCK_N + 4;
  const int t = threadIdx.x & 127, r0 = row0 + 16 * (t >> 5) + ((t & 31) >> 2), cq = 2 * (t & 3);
#pragma unroll
  for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      *reinterpret_cast<float2*>(stg + (r0 + 8 * hh) * SROW + 8 * i + cq) =
          make_float2(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
  }
}

// The epilogue of one GEMM row (row < 0: outside the image, nothing is stored): columns
// n0 + c_lo .. n0 + c_hi - 1 (c_lo, c_hi multiples of 8) of the fp32 staging row srow, with the
// tile's bias slice s_bias (indexed from n0); z is the split (fp32 partials, wgrad bias row).
// A rolled loop over 8-column chunks (it runs once per tile, so every instruction of it is an
// instruction-cache miss: a short loop body fetched once beats an unrolled one), output mode
// decided once. SLOW = false compiles out the out-of-line epi_store_slow call, for callers that
// never need it (bf16 row-major output without beta): a call inside a loop that issues wgmma makes
// ptxas serialise the wgmma.
template <bool SLOW = true>
__device__ __forceinline__ void epilogue_row(const GemmParams& p, int row, const float* srow,
                                             const float* s_bias, int n0, int c_lo, int c_hi, int z) {
  enum { EPI_BF16, EPI_RAW_T, EPI_RAW, EPI_SLOW, EPI_NONE, EPI_BIASROW, EPI_F32 };
  const bool raw32 = !p.out_bf16 && p.beta == 0.f && p.alpha == 1.f && !p.bias && p.act == 0;
  float* const rbase = reinterpret_cast<float*>(p.out) +
                       (p.split_stride > 0 ? (long long)z * p.split_stride : 0LL);
  int mode;
  if (row < 0) mode = EPI_NONE;
  else if (row >= p.M) mode = (p.bias_out && row == p.M) ? EPI_BIASROW : EPI_NONE;
  else if (p.split_stride == 0 && !p.out_trans && p.out_bf16 && p.beta == 0.f) mode = EPI_BF16;
  else if (p.split_stride == 0 && !p.out_trans && !p.out_bf16 && p.beta == 0.f && !raw32)
    mode = EPI_F32;        // fp32 row-major with bias / activation (LSTM gate pre-activations,
                           // softmax logits): same inline path as bf16, fp32 stores
  else if (raw32 && p.out_trans) mode = EPI_RAW_T;
  else if (raw32 && (p.ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(rbase) & 15) == 0)
    mode = EPI_RAW;
  else mode = EPI_SLOW;

  auto emit = [&](const uint32_t (&r)[8], int c0) {
    const int nb = n0 + c0;
    if (mode == EPI_NONE) return;
    if (mode == EPI_BIASROW) {       // product row M = column sums of err (see ConvGeomU::ones)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (nb + j < p.N) p.bias_out[(long long)z * p.N + nb + j] = __uint_as_float(r[j]);
      return;
    }
    if (mode == EPI_BF16 || mode == EPI_F32) {
      float v[8];
      {
        const float4 b0 = *reinterpret_cast<const float4*>(s_bias + c0);
        const float4 b1 = *reinterpret_cast<const float4*>(s_bias + c0 + 4);
        v[0] = b0.x; v[1] = b0.y; v[2] = b0.z; v[3] = b0.w;
        v[4] = b1.x; v[5] = b1.y; v[6] = b1.z; v[7] = b1.w;
      }
      // activation selected once per chunk (not per element): the executed path stays short
      switch (p.act) {
        // out = act(alpha * acc + bias): alpha is the err_input_alpha of dgrad (no bias,
        // linear); every other caller passes alpha = 1
        case ACT_LINEAR:
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaf(__uint_as_float(r[j]), p.alpha, v[j]);
          break;
        case ACT_STRICT_RELU:
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(__uint_as_float(r[j]), p.alpha, v[j]), 0.f);
          break;
        case ACT_TANH:
#pragma unroll
          for (int j = 0; j < 8; ++j)
            v[j] = 1.7159f * tanh_approx(0.6666f * fmaf(__uint_as_float(r[j]), p.alpha, v[j]));
          break;
        default:
#pragma unroll
          for (int j = 0; j < 8; ++j)
            v[j] = act_fwd5_fast(p.act, fmaf(__uint_as_float(r[j]), p.alpha, v[j]));
      }
      if (p.dmul != nullptr && mode == EPI_BF16) {
        // err_input *= f'(x): x has the layout of the output (row pitch ldo)
        const __nv_bfloat16* dx = p.dmul + (long long)row * p.ldo + nb;
        if (nb + 8 <= p.N && (p.ldo & 7) == 0) {
          float xv[8];
          ld8(dx, xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] *= act_deriv(p.dact, 0.f, xv[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (nb + j < p.N) v[j] *= act_deriv(p.dact, 0.f, __bfloat162float(dx[j]));
        }
      }
      if (mode == EPI_F32) {
        float* qf = reinterpret_cast<float*>(p.out) + (long long)row * p.ldo + nb;
        if (nb + 8 <= p.N && (p.ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0) {
          reinterpret_cast<float4*>(qf)[0] = make_float4(v[0], v[1], v[2], v[3]);
          reinterpret_cast<float4*>(qf)[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (nb + j < p.N) qf[j] = v[j];
        }
        return;
      }
      __nv_bfloat16* q = reinterpret_cast<__nv_bfloat16*>(p.out) + (long long)row * p.ldo + nb;
      if (nb + 8 <= p.N && (p.ldo & 7) == 0) {
        st8(q, v);                   // bf16 pack: one 16-byte store per 8 outputs
      } else {                       // ragged last chunk / row pitch not a multiple of 16 bytes
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (nb + j < p.N) q[j] = __float2bfloat16_rn(v[j]);
      }
    } else if (mode == EPI_RAW_T) {
      // raw fp32 (split-K partials / FC weight gradients), transposed: for a fixed column the
      // 32 lanes hold consecutive rows = one coalesced 128-byte store per column
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (nb + j < p.N) rbase[(long long)(nb + j) * p.ldo + row] = __uint_as_float(r[j]);
    } else if (mode == EPI_RAW && nb + 8 <= p.N) {
      float4* q = reinterpret_cast<float4*>(rbase + (long long)row * p.ldo + nb);
      q[0] = make_float4(__uint_as_float(r[0]), __uint_as_float(r[1]), __uint_as_float(r[2]),
                         __uint_as_float(r[3]));
      q[1] = make_float4(__uint_as_float(r[4]), __uint_as_float(r[5]), __uint_as_float(r[6]),
                         __uint_as_float(r[7]));
    } else if (raw32) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (nb + j < p.N) rbase[(long long)row * p.ldo + nb + j] = __uint_as_float(r[j]);
    } else if (SLOW) {
#pragma unroll
      for (int j = 0; j < 8; ++j)     // (static indices: r stays in registers)
        if (nb + j < p.N) epi_store_slow(p, row, nb + j, __uint_as_float(r[j]), z);
    }
  };

#pragma unroll 1
  for (int c0 = c_lo; c0 < c_hi; c0 += 8) {
    if (n0 + c0 >= p.N) break;     // chunk beyond the last column
    uint32_t ra[8];
    const float4 x0 = *reinterpret_cast<const float4*>(srow + c0);
    const float4 x1 = *reinterpret_cast<const float4*>(srow + c0 + 4);
    ra[0] = __float_as_uint(x0.x); ra[1] = __float_as_uint(x0.y);
    ra[2] = __float_as_uint(x0.z); ra[3] = __float_as_uint(x0.w);
    ra[4] = __float_as_uint(x1.x); ra[5] = __float_as_uint(x1.y);
    ra[6] = __float_as_uint(x1.z); ra[7] = __float_as_uint(x1.w);
    emit(ra, c0);
  }
}

// Threads: warpgroup 0 (warps 0-3) issues the wgmma and runs the epilogue, its thread 0 also issues
// the TMA loads; gather kernels add warpgroup 1 (warps 4-7) as the implicit-GEMM producers.
template <int A_MODE>
__host__ __device__ constexpr int kthreads() {
  return (A_MODE == A_GATHER_K || A_MODE == A_GATHER_MN) ? 256 : 128;
}
// fp32 staging of the accumulator tile for the row-per-thread epilogue: [128][BLOCK_N + 4]
// (the pad makes the row reads of 8 consecutive threads hit distinct banks)
template <int BLOCK_N>
__host__ __device__ constexpr int stage_f32_bytes() {
  return ((BLOCK_M * (BLOCK_N + 4) * 4) + 1023) & ~1023;
}

// A_HALO_MN: the same staging for BAND_GROUPS x 64 rows
template <int BLOCK_N>
__host__ __device__ constexpr int band_f32_bytes() {
  return ((BAND_GROUPS * 64 * (BLOCK_N + 4) * 4) + 1023) & ~1023;
}

// bytes of one ring stage that hold A (the halo kernels keep A outside the constexpr ring: A_HALO
// in two halos, A_HALO_MN in a second ring of bands whose stage size is known at launch)
template <int A_MODE>
__host__ __device__ constexpr int a_stage_bytes() {
  return (A_MODE == A_HALO || A_MODE == A_HALO_MN) ? 0 : A_BYTES;
}

template <int BLOCK_N, int A_MODE, int B_MODE, int STAGES>
__host__ __device__ constexpr int min_ctas() {
  // the accumulators (BLOCK_N fp32 registers per MMA thread) of a 256-thread gather CTA at
  // BLOCK_N = 128 do not fit the 128 registers a second CTA would leave
  // halo kernels (128 threads): registers for four CTAs per SM, 128 per thread; their shared
  // memory (B ring + two halos, 27-82 KB on the CIFAR shapes) decides how many actually fit
  // band kernels: BAND_GROUPS x BLOCK_N / 2 accumulators per thread, two CTAs per SM
  return A_MODE == A_HALO_MN ? 2
         : A_MODE == A_HALO ? (BLOCK_N >= 128 ? 2 : 4)
         : (kthreads<A_MODE>() == 256 && BLOCK_N >= 128) ? 1
         : ((2 * (STAGES * (A_BYTES + b_bytes<BLOCK_N, B_MODE>()) + 2048) <= 227 * 1024) ? 2 : 1);
}

template <int BLOCK_N, int A_MODE, int B_MODE, int GKIND, int GVEC, int STAGES>
__global__ void __launch_bounds__(kthreads<A_MODE>(), (min_ctas<BLOCK_N, A_MODE, B_MODE, STAGES>()))
gemm_umma_k(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const GemmParams p) {
  pdl_trigger();
  constexpr int B_BYTES = b_bytes<BLOCK_N, B_MODE>();
  constexpr int A_STAGE = a_stage_bytes<A_MODE>();
  constexpr int STAGE_BYTES = A_STAGE + B_BYTES;
  constexpr bool A_GATHER = (A_MODE == A_GATHER_K || A_MODE == A_GATHER_MN);
  constexpr bool HALO = (A_MODE == A_HALO);
  constexpr bool BAND = (A_MODE == A_HALO_MN);
  constexpr bool A_MN = (A_MODE == A_TMA_MN || A_MODE == A_GATHER_MN || BAND);
  constexpr bool B_MN = (B_MODE == B_TMA_MN);
  static_assert(!B_MN || BLOCK_N >= 64, "MN-major B tiles are built from 64-wide swizzle atoms");
  static_assert(HALO || BAND || stage_f32_bytes<BLOCK_N>() <= STAGES * STAGE_BYTES,
                "epilogue staging exceeds the ring");
  static_assert(!BAND || (B_MN && GKIND == G_IM2COL), "A_HALO_MN is the conv wgrad operand");
  constexpr uint32_t TX_BYTES = (A_GATHER || HALO || BAND ? 0 : A_BYTES) + B_BYTES;
  constexpr int ACC = BLOCK_N / 2;                        // fp32 registers per 64-row half
  constexpr int SROW = BLOCK_N + 4;

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];
  __shared__ __align__(8) uint64_t halo_bar;

  // 1024-byte aligned tile area (SWIZZLE_128B atoms are 1024 B)
  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  // halo kernels: the two blocks' halos follow the B ring; the epilogue's fp32 staging overlays
  // ring and halos from the start of the tile area, and may be the larger of the two
  // band kernels: the ring of bands (STAGES x hbytes) follows the B ring, then the 128-byte block
  // of bias "ones" rows; their staging is band_f32_bytes
  uint8_t* const halo = tiles + (size_t)STAGES * STAGE_BYTES;
  const int tile_area = HALO ? max(STAGES * STAGE_BYTES + 2 * p.hbytes, stage_f32_bytes<BLOCK_N>())
                        : BAND ? max(STAGES * (STAGE_BYTES + p.hbytes) + 128, band_f32_bytes<BLOCK_N>())
                               : STAGES * STAGE_BYTES;
  // behind the tile area: the gather lookup table (only as many entries as this geometry needs - a
  // fixed-size table would cost the BLOCK_N = 64 conv kernels their second CTA per SM; halo
  // kernels keep their per-k16-step descriptor offsets there) and the tile's bias slice (the
  // epilogue would otherwise wait on one L2 round trip per 8 columns)
  int* const ktab = reinterpret_cast<int*>(tiles + tile_area);
  float* const s_bias = reinterpret_cast<float*>(ktab + ((p.ktab_n + 3) & ~3));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * BLOCK_M, n0 = blockIdx.x * BLOCK_N;
  const int total_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int kb_begin = blockIdx.z * p.k_blocks_per_split;
  const int kb_end = min(total_kb, kb_begin + p.k_blocks_per_split);
  const int num_kb = max(0, kb_end - kb_begin);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], (A_GATHER ? 128u : 0u) + 1u);
      mbar_init(&empty_bar[s], 1u);
    }
    if (HALO) mbar_init(&halo_bar, 1u);
    fence_barrier_init();
    if (!A_GATHER) tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
  }
  if (A_GATHER) build_ktab(ktab, p.g, GKIND, p.gK);
  if (HALO) build_halo_tab<GKIND>(ktab, p);
  // band kernels: group j of this CTA is gv = blockIdx.y * BAND_GROUPS + j, numbered plane-major
  // (gv = plane * KY + ky) so that a CTA loads as few planes as possible; gv == bgroups is the bias
  // group, whose A is the ones block: 8 rows of {1, 0, ..., 0} read with LBO = SBO = 0, so that
  // product row 0 of the group is sum_pixels err[pixel][f], the gather's ones row
  int band_plo = 0, band_np = 0;
  uint8_t* const ones = halo + (size_t)STAGES * p.hbytes;
  if (BAND) {
    const int g0 = blockIdx.y * BAND_GROUPS, gl = min(g0 + BAND_GROUPS, p.bgroups) - 1;
    band_plo = g0 / p.g.KY;
    band_np = gl >= g0 ? gl / p.g.KY - band_plo + 1 : 0;
    if (threadIdx.x < 64)
      reinterpret_cast<__nv_bfloat16*>(ones)[threadIdx.x] =
          __float2bfloat16_rn((threadIdx.x & 7) == 0 ? 1.f : 0.f);
    fence_proxy_async_smem();
  }
  pdl_wait();      // everything above overlapped the previous kernel's tail; global reads start here
  if (HALO && threadIdx.x == 0) {
    // the windows of the tile's two 8x8 blocks
    mbar_arrive_expect_tx(&halo_bar, 2u * halo_tx_bytes<GKIND>(p));
#pragma unroll 1
    for (int h = 0; h < 2; ++h) load_halo<GKIND>(halo + h * p.hbytes, &tmap_a, &halo_bar, p, blockIdx.y * 2 + h);
  }
  if (threadIdx.x < BLOCK_N) {
    const int n = blockIdx.x * BLOCK_N + threadIdx.x;
    s_bias[threadIdx.x] = (p.bias && n < p.N) ? __ldg(p.bias + n) : 0.f;
  }
  __syncthreads();

  if (A_GATHER && threadIdx.x >= 128) {
    // ===================== gather producers (warpgroup 1) =====================
    const int t = threadIdx.x - 128;        // 0..127
    if (A_MODE == A_GATHER_K) {
      // tile row r = t is GEMM row m0 + t (a pixel); chunks run over the reduction index
      const int m = m0 + t;
      const PixCtx ctx = (GKIND == G_IM2COL) ? decode_out_pixel(p.gsrc, p.g, m, p.M)
                                             : decode_in_pixel(p.gsrc, p.g, m, p.M);
      if (GVEC == 2) {
        // asynchronous gather: issue the LDGSTS of a stage as soon as its slot is free; the
        // stage's full barrier is armed by the copies themselves
#pragma unroll 1
        for (int i = 0; i < num_kb; ++i) {
          const int s = i % STAGES; const uint32_t ph = (i / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          const uint32_t row_base = smem_u32(tiles + (size_t)s * STAGE_BYTES) + t * 128;
          gather_row_async<GKIND>(row_base, t & 7, ktab, p.g, ctx, (kb_begin + i) * BLOCK_K);
          cp_async_mbar_arrive_noinc(&full_bar[s]);
        }
      } else {
        uint4 v[8], nv[8];
        // software pipeline with ONE load site: iteration i issues the global loads of stage
        // i + 1 and then publishes stage i (whose loads were issued one iteration earlier)
#pragma unroll 1
        for (int i = -1; i < num_kb; ++i) {
          if (i + 1 < num_kb) {
            const int k0 = (kb_begin + i + 1) * BLOCK_K;
            gather_row<GKIND, GVEC>(nv, ktab, p.g, ctx, k0, p.gK);
          }
          if (i >= 0) {
            const int s = i % STAGES; const uint32_t ph = (i / STAGES) & 1;
            mbar_wait(&empty_bar[s], ph ^ 1);
            uint8_t* sa = tiles + (size_t)s * STAGE_BYTES;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8)
              *reinterpret_cast<uint4*>(sa + t * 128 + ((c8 ^ (t & 7)) << 4)) = v[c8];
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[s]);
          }
#pragma unroll
          for (int c8 = 0; c8 < 8; ++c8) v[c8] = nv[c8];
        }
      }
    } else {
      // A_GATHER_MN (conv wgrad): tile = [64 reduction rows (pixels)][128 m (kidx)];
      // thread -> reduction row kr = t % 64, 64-wide m block = t / 64 (8 chunks of 8 kidx)
      const int kr = t & 63, mblk = t >> 6;
      // only the 64-wide m block that contains index Kw carries the bias "ones" row
      const int kk0 = m0 + mblk * 64;
      const bool has_one = p.g.ones != nullptr && kk0 <= p.gK && p.gK < kk0 + 64;
      if (GVEC == 2) {
#pragma unroll 1
        for (int i = 0; i < num_kb; ++i) {
          const int s = i % STAGES; const uint32_t ph = (i / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int pix = (kb_begin + i) * BLOCK_K + kr;
          const PixCtx ctx = decode_out_pixel(p.gsrc, p.g, pix, p.K);
          const uint32_t row_base =
              smem_u32(tiles + (size_t)s * STAGE_BYTES) + mblk * 8192 + kr * 128;
          if (has_one) gather_row_async<G_IM2COL, true>(row_base, kr & 7, ktab, p.g, ctx, kk0);
          else gather_row_async<G_IM2COL, false>(row_base, kr & 7, ktab, p.g, ctx, kk0);
          cp_async_mbar_arrive_noinc(&full_bar[s]);
        }
      } else {
        uint4 v[8], nv[8];
#pragma unroll 1
        for (int i = -1; i < num_kb; ++i) {
          if (i + 1 < num_kb) {
            const int pix = (kb_begin + i + 1) * BLOCK_K + kr;
            const PixCtx ctx = decode_out_pixel(p.gsrc, p.g, pix, p.K);
            gather_row<G_IM2COL, GVEC>(nv, ktab, p.g, ctx, m0 + mblk * 64, p.gK);
          }
          if (i >= 0) {
            const int s = i % STAGES; const uint32_t ph = (i / STAGES) & 1;
            mbar_wait(&empty_bar[s], ph ^ 1);
            uint8_t* sa = tiles + (size_t)s * STAGE_BYTES;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8)
              *reinterpret_cast<uint4*>(sa + mblk * 8192 + kr * 128 + ((c8 ^ (kr & 7)) << 4)) = v[c8];
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[s]);
          }
#pragma unroll
          for (int c8 = 0; c8 < 8; ++c8) v[c8] = nv[c8];
        }
      }
    }
    return;
  }

  // ===================== warpgroup 0: TMA issue (thread 0), wgmma, epilogue =====================
  // TMA loads of k-block i into its stage; the slot is free (released by this thread below)
  auto issue_loads = [&](int i) {
    const int s = i % STAGES;
    uint8_t* sa = tiles + (size_t)s * STAGE_BYTES;
    uint8_t* sb = sa + A_STAGE;
    const int k0 = (kb_begin + i) * BLOCK_K;
    mbar_arrive_expect_tx(&full_bar[s], TX_BYTES + (BAND ? band_np * p.bw * p.bh * 16 : 0));
    if (BAND) {
      // the band of pixels k0 .. k0 + 63 (one image: (OH * OW) % 64 == 0), one box per plane;
      // output pixel (oy, ox) with tap (ky, kx) reads x[oy + ky - PT][ox + kx - PL]
      const ConvGeomU& g = p.g;
      const int img = g.OH * g.OW, n = k0 / img, rem = k0 - n * img, oy = rem / g.OW;
      const int ox = rem - oy * g.OW;
      uint8_t* const band = halo + (size_t)s * p.hbytes;
#pragma unroll 1
      for (int j = 0; j < band_np; ++j)
        tma_load_4d(band + j * p.bplane, &tmap_a, &full_bar[s], (band_plo + j) * 8, ox - g.PL,
                    oy - g.PT, n);
    } else if (A_MODE == A_IM2COL_K) {
      // conv fprop / stride-1 dgrad: tile rows = pixels m0 .. m0 + 127, k-block = 64
      // channels of ONE filter tap
      const ConvGeomU& g = p.g;
      const int tap = k0 / g.inner, c0 = k0 - tap * g.inner;
      const int ky = tap / g.KX, kx = tap - ky * g.KX;
      int w0, h0, n, ow, oh;
      if (GKIND == G_IM2COL) {
        const int q = m0 % g.OW; const int t2 = m0 / g.OW;
        const int pr = t2 % g.OH; n = t2 / g.OH;
        w0 = q * g.SX - g.PL; h0 = pr * g.SY - g.PT; ow = kx; oh = ky;
      } else {                                   // dgrad: correlation with the flipped filter
        const int ix = m0 % g.W; const int t2 = m0 / g.W;
        const int iy = t2 % g.H; n = t2 / g.H;
        w0 = ix - (g.KX - 1 - g.PL); h0 = iy - (g.KY - 1 - g.PT);
        ow = g.KX - 1 - kx; oh = g.KY - 1 - ky;
      }
      tma_load_im2col_4d(sa, &tmap_a, &full_bar[s], c0, w0, h0, n, (uint16_t)ow, (uint16_t)oh);
    } else if (A_MODE == A_TMA_K) {
      tma_load_2d(sa, &tmap_a, &full_bar[s], k0, m0);
    } else if (A_MODE == A_TMA_MN) {
      tma_load_2d(sa, &tmap_a, &full_bar[s], m0, k0);
      tma_load_2d(sa + 8192, &tmap_a, &full_bar[s], m0 + 64, k0);
    }
    if (B_MODE == B_TMA_K) {
      tma_load_2d(sb, &tmap_b, &full_bar[s], k0, n0);
    } else {
#pragma unroll
      for (int j = 0; j < (BLOCK_N + 63) / 64; ++j)
        tma_load_2d(sb + j * 8192, &tmap_b, &full_bar[s], n0 + j * 64, k0);
    }
  };

  float acc0[ACC], acc1[ACC];                 // rows 0-63 / 64-127 of the tile
  float acc2[BAND ? ACC : 1];                 // band kernels: the third group
#pragma unroll
  for (int j = 0; j < ACC; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
#pragma unroll
  for (int j = 0; j < (BAND ? ACC : 1); ++j) acc2[j] = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < STAGES && i < num_kb; ++i) issue_loads(i);
  const uint32_t halo_sa = smem_u32(halo);
  const uint32_t halo_sbo = (8 + p.g.KX - 1) * 16;       // one halo row = the next 8 tile rows
  if (HALO) mbar_wait(&halo_bar, 0);
  // band kernels: byte offset of each group's slot-0 core matrix for pixel 0 (ones: the group
  // reads the ones block), of each k16 step's first pixel, and between its two 8-pixel halves
  // (the next 8 pixels of the row, or the next band row when OW = 8)
  uint32_t band_goff[BAND_GROUPS], band_soff[BLOCK_K / 16], band_kstr = 0;
  bool band_one[BAND_GROUPS];
  if (BAND) {
    const ConvGeomU& g = p.g;
    const int owb = min(g.OW, 64);
#pragma unroll
    for (int j = 0; j < BAND_GROUPS; ++j) {
      const int gv = blockIdx.y * BAND_GROUPS + j, pl = gv / g.KY, ky = gv - pl * g.KY;
      band_one[j] = gv >= p.bgroups;
      band_goff[j] = band_one[j] ? 0u : (uint32_t)((pl - band_plo) * p.bplane + ky * p.bw * 16);
    }
#pragma unroll
    for (int k = 0; k < BLOCK_K / 16; ++k) {
      const int r = (16 * k) / owb, c = 16 * k - r * owb;
      band_soff[k] = (uint32_t)((r * p.bw + c) * 16);
    }
    band_kstr = owb == 8 ? p.bw * 16 : 128;
  }
  const uint64_t ones_desc = make_smem_desc_interleave(smem_u32(ones), 0, 0);
#pragma unroll 1
  for (int i = 0; i < num_kb; ++i) {
    const int s = i % STAGES; const uint32_t ph = (i / STAGES) & 1;
    mbar_wait(&full_bar[s], ph);
    if (A_GATHER && GVEC == 2) fence_proxy_async_smem();   // LDGSTS data -> async proxy
    const uint32_t sa = smem_u32(tiles + (size_t)s * STAGE_BYTES);
    const uint32_t sb = sa + A_STAGE;
    const uint32_t band = halo_sa + s * p.hbytes;
    wg_fence_regs(acc0); wg_fence_regs(acc1);
    if (BAND) wg_fence_regs(acc2);
    wg_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / 16; ++k) {
      // K-major: 16 bf16 = 32 B along the swizzled row. MN-major: 16 k-rows = 2 atoms.
      // The 64-row halves of A are 8192 bytes apart in both layouts.
      uint64_t da0, da1, da2 = 0;
      if (BAND) {
        // MN-major, no swizzle: SBO = 16 bytes between the kx slots along M, LBO between the two
        // 8-pixel halves along K
        uint64_t d[BAND_GROUPS];
#pragma unroll
        for (int j = 0; j < BAND_GROUPS; ++j)
          d[j] = band_one[j] ? ones_desc
                             : make_smem_desc_interleave(band + band_goff[j] + band_soff[k], band_kstr, 16);
        da0 = d[0]; da1 = d[1]; da2 = d[2];
      } else if (HALO) {
        const uint32_t e = (uint32_t)ktab[(kb_begin + i) * (BLOCK_K / 16) + k];
        const uint32_t a = halo_sa + (e & 0xFFFFu);
        da0 = make_smem_desc_interleave(a, e >> 16, halo_sbo);
        da1 = make_smem_desc_interleave(a + p.hbytes, e >> 16, halo_sbo);
      } else {
        da0 = A_MN ? make_smem_desc(sa + k * 2048, 8192, 1024) : make_smem_desc(sa + k * 32, 16, 1024);
        da1 = A_MN ? make_smem_desc(sa + 8192 + k * 2048, 8192, 1024)
                   : make_smem_desc(sa + 8192 + k * 32, 16, 1024);
      }
      const uint64_t db = B_MN ? make_smem_desc(sb + k * 2048, 8192, 1024)
                               : make_smem_desc(sb + k * 32, 16, 1024);
      wgmma_bf16<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc0, da0, db, 1);
      wgmma_bf16<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc1, da1, db, 1);
      if constexpr (BAND) wgmma_bf16<BLOCK_N, 1, 1>(acc2, da2, db, 1);
    }
    wg_commit();
    wg_fence_regs(acc0); wg_fence_regs(acc1);
    if (BAND) wg_fence_regs(acc2);
    wg_wait<1>();                               // the MMAs of k-block i - 1 have retired
    if (i > 0 && threadIdx.x == 0) {
      const int sp = (i - 1) % STAGES;
      mbar_arrive(&empty_bar[sp]);
      if (i - 1 + STAGES < num_kb) issue_loads(i - 1 + STAGES);
    }
  }
  wg_wait<0>();
  wg_fence_regs(acc0); wg_fence_regs(acc1);
  if constexpr (BAND) {
    wg_fence_regs(acc2);
    band_epilogue<BLOCK_N>(p, reinterpret_cast<float*>(tiles), acc0, acc1, acc2);
    return;
  }

  // ===================== epilogue =====================
  // The accumulator fragments go through shared memory (the ring is idle: every k-block has been
  // consumed) so that thread t owns row m0 + t.
  float* const stg = reinterpret_cast<float*>(tiles);
  {
    const int r0 = 16 * warp + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        *reinterpret_cast<float2*>(stg + (r0 + 8 * hh) * SROW + 8 * i + cq) =
            make_float2(acc0[4 * i + 2 * hh], acc0[4 * i + 2 * hh + 1]);
        *reinterpret_cast<float2*>(stg + (64 + r0 + 8 * hh) * SROW + 8 * i + cq) =
            make_float2(acc1[4 * i + 2 * hh], acc1[4 * i + 2 * hh + 1]);
      }
    }
  }
  named_bar_sync(1, 128);
  const int row = HALO ? halo_row<GKIND>(p, blockIdx.y * 2 + (threadIdx.x >> 6), threadIdx.x & 63)
                       : m0 + (int)threadIdx.x;
  epilogue_row(p, row, stg + threadIdx.x * SROW, s_bias, n0, 0, BLOCK_N, blockIdx.z);
}

// ---- persistent halo conv: the A_HALO geometries with N <= 64 (dgrad: 16 < C <= 64) and a filter
// that fits shared memory. A work item is one 8x8 block of output (dgrad: input) pixels x BLOCK_N
// columns: one m64 x BLOCK_N
// accumulator chain over every k16 step of the reduction, with the same per-step halo offsets
// (build_halo_tab) in the same order as A_HALO, so the results are bit-identical to it. Each CTA
// loads its BLOCK_N columns of B into shared memory once and keeps them for all its items, instead
// of streaming the whole filter through a ring per 128-row tile. Items are taken in a static stride,
// item = blockIdx.x + j * gridDim.x; the column tile is item % ntiles, the same for every item of a
// CTA because gridDim.x is a multiple of ntiles. Thread 0 keeps PH_STAGES halos in flight: the halo
// of item j + PH_STAGES is requested as soon as the MMAs of item j have retired, so its TMA overlaps
// the epilogue and the following items. One warpgroup per CTA; the several CTAs that fit an SM
// overlap one CTA's epilogue with another's MMAs. Resident B, one tile of BLOCK_N * 128 bytes per
// k-block of 64 reduction indices:
//   fprop, B = w_lp [F][ldw] (K-major): SW128 tiles [BLOCK_N rows][64], as in gemm_umma_k's ring;
//   dgrad, B = wd_lp [Kd][ldc] (MN-major, BLOCK_N = 32): SW64 tiles [64 k-rows][32 columns], one
//   TMA box {32, 64} each. A 64-byte row holds the 32 columns of one k-row, 8 k-rows make one
//   512-byte swizzle atom (SBO), and a k16 step is two atoms. The SW128 MN-major tiles of
//   gemm_umma_k are 64 columns wide, so C = 32 would issue N = 64; this issues N = 32.
constexpr int PH_STAGES = 4;
constexpr int PERSIST_SMEM_MAX = 226 * 1024;     // + the static barriers <= 227 KB per block

__host__ __device__ __forceinline__ int persist_b_bytes(const GemmParams& p, int bn) {
  return (p.K + BLOCK_K - 1) / BLOCK_K * bn * 128;
}
// dynamic shared memory of conv_halo_persist_k: alignment slack, resident B, the halo ring, the
// fp32 staging of one item, the per-k16-step halo offsets, the bias slice
__host__ __device__ __forceinline__ int persist_smem_bytes(const GemmParams& p, int bn) {
  return 1024 + persist_b_bytes(p, bn) + PH_STAGES * p.hbytes + 64 * (bn + 4) * 4 +
         ((p.ktab_n + 3) & ~3) * 4 + bn * 4;
}

template <int BLOCK_N, int GKIND>
__global__ void __launch_bounds__(128)
conv_halo_persist_k(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const GemmParams p) {
  pdl_trigger();
  constexpr int ACC = BLOCK_N / 2;
  constexpr int SROW = BLOCK_N + 4;
  constexpr bool DGRAD = GKIND == G_DGRAD;
  static_assert(!DGRAD || BLOCK_N == 32, "dgrad B tiles are one 64-byte swizzle atom wide");
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t b_bar;
  __shared__ __align__(8) uint64_t full_bar[PH_STAGES];

  uint8_t* const bres = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  uint8_t* const halo = bres + persist_b_bytes(p, BLOCK_N);
  float* const stg = reinterpret_cast<float*>(halo + PH_STAGES * p.hbytes);
  int* const tab = reinterpret_cast<int*>(stg + 64 * SROW);
  float* const s_bias = reinterpret_cast<float*>(tab + ((p.ktab_n + 3) & ~3));

  const int ntiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int n0 = (int)(blockIdx.x % ntiles) * BLOCK_N;
  const int items = p.g.N * p.hnby * p.hnbx * ntiles;
  const int nj = (items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const uint32_t hx = halo_tx_bytes<GKIND>(p);

  if (threadIdx.x == 0) {
    mbar_init(&b_bar, 1u);
    for (int s = 0; s < PH_STAGES; ++s) mbar_init(&full_bar[s], 1u);
    fence_barrier_init();
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
  }
  build_halo_tab<GKIND>(tab, p);
  pdl_wait();      // everything above overlapped the previous kernel's tail; global reads start here
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&b_bar, (uint32_t)persist_b_bytes(p, BLOCK_N));
#pragma unroll 1
    for (int i = 0; i < kb; ++i) {
      if (DGRAD) tma_load_2d(bres + i * (BLOCK_N * 128), &tmap_b, &b_bar, n0, i * BLOCK_K);
      else tma_load_2d(bres + i * (BLOCK_N * 128), &tmap_b, &b_bar, i * BLOCK_K, n0);
    }
#pragma unroll 1
    for (int j = 0; j < PH_STAGES && j < nj; ++j) {
      mbar_arrive_expect_tx(&full_bar[j], hx);
      load_halo<GKIND>(halo + j * p.hbytes, &tmap_a, &full_bar[j], p,
                       ((int)blockIdx.x + j * (int)gridDim.x) / ntiles);
    }
  }
  if (threadIdx.x < BLOCK_N) {
    const int n = n0 + threadIdx.x;
    s_bias[threadIdx.x] = (p.bias && n < p.N) ? __ldg(p.bias + n) : 0.f;
  }
  __syncthreads();
  mbar_wait(&b_bar, 0);

  const uint32_t bres_sa = smem_u32(bres), halo_sa = smem_u32(halo);
  const uint32_t halo_sbo = (8 + p.g.KX - 1) * 16;       // one halo row = the next 8 block rows
  const int r = threadIdx.x & 63, half = threadIdx.x >> 6;  // epilogue: row and column half
#pragma unroll 1
  for (int j = 0; j < nj; ++j) {
    const int s = j % PH_STAGES, item = (int)blockIdx.x + j * (int)gridDim.x;
    const uint32_t hs = halo_sa + s * p.hbytes;
    float acc[ACC];
#pragma unroll
    for (int e = 0; e < ACC; ++e) acc[e] = 0.f;
    mbar_wait(&full_bar[s], (j / PH_STAGES) & 1);
    wg_fence_regs(acc);
    wg_fence();
#pragma unroll 1
    for (int i = 0; i < kb; ++i) {
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        const int step = i * (BLOCK_K / 16) + k;
        const uint32_t e = (uint32_t)tab[step];
        const uint64_t da = make_smem_desc_interleave(hs + (e & 0xFFFFu), e >> 16, halo_sbo);
        const uint64_t db = DGRAD ? make_smem_desc(bres_sa + i * (BLOCK_N * 128) + k * 1024, 0, 512, SW64)
                                  : make_smem_desc(bres_sa + i * (BLOCK_N * 128) + k * 32, 16, 1024);
        wgmma_bf16<BLOCK_N, 0, DGRAD ? 1 : 0>(acc, da, db, 1);
      }
    }
    wg_commit();
    wg_fence_regs(acc);
    wg_wait<0>();
    wg_fence_regs(acc);
    if (threadIdx.x == 0 && j + PH_STAGES < nj) {   // slot s is free: the halo of item j + PH_STAGES
      mbar_arrive_expect_tx(&full_bar[s], hx);
      load_halo<GKIND>(halo + s * p.hbytes, &tmap_a, &full_bar[s], p, (item + PH_STAGES * (int)gridDim.x) / ntiles);
    }
    if (j > 0) named_bar_sync(1, 128);               // the previous item's staging has been read
    stage_acc<BLOCK_N>(stg, 0, acc);
    named_bar_sync(1, 128);
    epilogue_row<false>(p, halo_row<GKIND>(p, item / ntiles, r), stg + r * SROW, s_bias, n0,
                        half * (BLOCK_N / 2), (half + 1) * (BLOCK_N / 2), 0);
  }
}

// ------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 tensor map: inner dim `inner` (contiguous), outer dim `outer`, row pitch ld elements,
// box {64, box_rows} with SWIZZLE_128B, or {32, box_rows} with SWIZZLE_64B (box_inner = 32: the
// dgrad B tiles of conv_halo_persist_k), OOB -> zeros.
static int make_map(CUtensorMap* m, const void* ptr, long long inner, long long outer, long long ld,
                    int box_rows, int box_inner = 64) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -1;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)(ld * 2)};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   box_inner == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

// ---- im2col-mode tensor map over an NHWC bf16 tensor [N][H][W][C] --------------------------------
// Filter-window base positions along w run from lower_w to W + upper_w (exclusive) in steps of the
// traversal stride; upper_* are chosen by the callers so that exactly OW x OH positions exist.
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeIm2colFn get_encode_im2col() {
  static EncodeIm2colFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return nullptr;
    fn = reinterpret_cast<EncodeIm2colFn>(p);
  }
  return fn;
}
static int make_map_im2col(CUtensorMap* m, const void* ptr, int N, int H, int W, int C, int lower_w,
                           int lower_h, int upper_w, int upper_h, int stride_w, int stride_h, int pixels) {
  EncodeIm2colFn enc = get_encode_im2col();
  if (!enc) return -1;
  if (lower_w < -128 || lower_h < -128 || upper_w < -128 || upper_h < -128 || lower_w > 127 ||
      lower_h > 127 || upper_w > 127 || upper_h > 127 || stride_w > 8 || stride_h > 8)
    return -7;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lower[2] = {lower_w, lower_h};
  int upper[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1u, (cuuint32_t)stride_w, (cuuint32_t)stride_h, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower,
                   upper, 64u, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}
static long long g_im2col_launches = 0;
long long im2col_tma_launches() { return g_im2col_launches; }
// ZNICZ_IM2COL_TMA=0 keeps the LDGSTS gather producers (A/B measurements, fallback)
static bool im2col_tma_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("ZNICZ_IM2COL_TMA"); on = (e && atoi(e) == 0) ? 0 : 1; }
  return on != 0;
}

// ---- A_HALO selection: a 4-D map over the NHWC source (x for fprop, err_out for dgrad) whose box
// is one 8-channel plane of a block's halo, {8, 8 + KX - 1, 8 + KY - 1, 1}, no swizzle
static long long g_halo_launches = 0;
long long conv_halo_launches() { return g_halo_launches; }
// ZNICZ_CONV_HALO=0 keeps the tap-mode LDGSTS gather for the shapes the halo kernel serves
static bool conv_halo_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("ZNICZ_CONV_HALO"); on = (e && atoi(e) == 0) ? 0 : 1; }
  return on != 0;
}
// Tap-mode geometry (set_tap_mode) the halo kernel serves: unit stride, 8 / 16 / 32 inner channels
// (tpk >= 2), a halo that fits HALO_MAX_BYTES. dgrad with 8 channels stays on the gather: its
// flipped taps would need a negative LBO between the two taps of a k16 step.
static bool halo_eligible(GemmParams& p, bool dgrad) {
  const ConvGeomU& g = p.g;
  if (!conv_halo_enabled() || g.SY != 1 || g.SX != 1 || g.tpk < 2 || (dgrad && g.tpk == 8)) return false;
  if (8 + g.KX - 1 > 256 || 8 + g.KY - 1 > 256) return false;        // TMA box extent
  p.hbytes = (g.inner / 8) * halo_plane_bytes(g);
  if (p.hbytes > HALO_MAX_BYTES) return false;
  const int PH = dgrad ? g.H : g.OH, PW = dgrad ? g.W : g.OW;
  p.hnby = (PH + 7) / 8; p.hnbx = (PW + 7) / 8;
  return (long long)g.N * p.hnby * p.hnbx < (1LL << 31);
}
// The conv weight gradient (A_HALO_MN) of the same tap-mode geometries, with F <= 64 (one BLOCK_N
// = 64 tile: three groups of accumulators fit the registers), KX <= 8 (one group's 8 kx slots),
// k-blocks of whole output rows (OW = 8 / 16 / 32 / 64) or 64-pixel row segments (OW % 64 == 0)
// that never straddle two images, and a band that fits BAND_MAX_BYTES per stage. Fills the band
// fields of p; the group count includes the bias group when p.bias_out is set.
static bool band_eligible(GemmParams& p) {
  const ConvGeomU& g = p.g;
  if (!conv_halo_enabled() || g.SY != 1 || g.SX != 1 || g.tpk < 2 || g.F > 64 || g.KX > 8) return false;
  const bool rows = g.OW % 8 == 0 && 64 % g.OW == 0;
  if ((!rows && g.OW % 64) || (g.OH * g.OW) % 64) return false;
  p.bw = (rows ? g.OW : 64) + g.KX - 1;
  p.bh = (rows ? 64 / g.OW : 1) + g.KY - 1;
  if (p.bw > 256 || p.bh > 256) return false;                       // TMA box extent
  p.bplane = (p.bw * p.bh * 16 + 127) & ~127;
  p.bgroups = g.KY * (g.C / 8);
  p.bvgroups = p.bgroups + (p.bias_out ? 1 : 0);
  int np = 0;                  // planes of the widest CTA (groups are numbered plane * KY + ky)
  for (int g0 = 0; g0 < p.bgroups; g0 += BAND_GROUPS)
    np = std::max(np, (std::min(g0 + BAND_GROUPS, p.bgroups) - 1) / g.KY - g0 / g.KY + 1);
  // slots >= KX of the last pixels read up to (8 - KX) * 16 bytes past the last plane
  p.hbytes = np * p.bplane + 128;
  return p.hbytes <= BAND_MAX_BYTES;
}
// ZNICZ_CONV_HALO_PERSIST=0 runs the shapes that conv_halo_persist_k serves on A_HALO instead
static bool halo_persist_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("ZNICZ_CONV_HALO_PERSIST"); on = (e && atoi(e) == 0) ? 0 : 1; }
  return on != 0;
}
// The persistent kernel's column tile for an A_HALO shape (p from halo_eligible) with N columns,
// and the shared memory it needs; 0 when it does not serve the shape: N > 64, an output other than
// bf16 without beta (see epilogue_row<false>), or a resident B and halo ring that do not fit.
// p.ktab_n is set to the k16 steps (build_halo_tab).
static int persist_bn(GemmParams& p, int& smem) {
  if (!halo_persist_enabled() || p.N > 64 || !p.out_bf16 || p.beta != 0.f) return 0;
  const int bn = p.N <= 16 ? 16 : 32;      // N = 64: two 32-column items per block, more items
  p.ktab_n = (p.K + BLOCK_K - 1) / BLOCK_K * (BLOCK_K / 16);
  smem = persist_smem_bytes(p, bn);
  return smem <= PERSIST_SMEM_MAX ? bn : 0;
}
// Grid: as many CTAs as fit at once (occupancy at this shared-memory size), reduced to the fewest
// that still give every CTA the same number of items +- 1 in as many rounds (fewer CTAs load B
// fewer times), rounded up to a multiple of the column tiles.
template <int BN, int GK>
static int launch_persist(const CUtensorMap& th, const CUtensorMap& tb, const GemmParams& p, int smem,
                          cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_halo_persist_k<BN, GK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         PERSIST_SMEM_MAX);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  int occ = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, conv_halo_persist_k<BN, GK>, 128, smem);
  if (e != cudaSuccess) return (int)e;
  if (occ < 1) return -6;
  const long long ntiles = (p.N + BN - 1) / BN, items = (long long)p.g.N * p.hnby * p.hnbx * ntiles;
  const long long slots = (long long)occ * num_sms(), rounds = (items + slots - 1) / slots;
  long long grid = (items + rounds - 1) / rounds;
  grid = std::min(items, (grid + ntiles - 1) / ntiles * ntiles);
  launch_k(conv_halo_persist_k<BN, GK>, dim3((unsigned)grid), 128, smem, st, th, tb, p);
  return (int)cudaGetLastError();
}

static int make_map_halo(CUtensorMap* m, const void* ptr, int N, int H, int W, int C, int KY, int KX,
                         int box_w = 0, int box_h = 0) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -1;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  // box {8 channels, 8 + KX - 1, 8 + KY - 1, 1} (A_HALO) or {8, box_w, box_h, 1} (a band)
  cuuint32_t box[4] = {8u, (cuuint32_t)(box_w ? box_w : 8 + KX - 1), (cuuint32_t)(box_h ? box_h : 8 + KY - 1), 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

template <int BN, int AM, int BM, int GK, int GV, int NS>
static int launch_stages(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p_in, dim3 grid,
                         cudaStream_t st) {
  constexpr int ring = NS * (a_stage_bytes<AM>() + b_bytes<BN, BM>()) + 1024;
  constexpr bool gather = (AM == A_GATHER_K || AM == A_GATHER_MN);
  constexpr bool halo = (AM == A_HALO);
  constexpr bool band = (AM == A_HALO_MN);
  // must match the kernel's tile area: halo kernels add two halos behind the ring, band kernels a
  // ring of bands and the ones block; the epilogue staging of both may need more
  constexpr int area_max = halo ? std::max(ring + 2 * HALO_MAX_BYTES, stage_f32_bytes<BN>() + 1024)
                           : band ? std::max(ring + NS * BAND_MAX_BYTES + 128, band_f32_bytes<BN>() + 1024)
                                  : ring;
  constexpr int smem_max = area_max + (gather || halo ? KTAB * 4 : 0) + BN * 4 + 16;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_umma_k<BN, AM, BM, GK, GV, NS>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  GemmParams p = p_in;
  p.ktab_n = 0;
  if (gather) {       // must match build_ktab()
    const int step = p.g.vec ? 8 : 1;
    p.ktab_n = p.g.tpk > 0 ? p.g.ntaps : std::min(KTAB, (p.gK + step - 1) / step);
  }
  if (halo) p.ktab_n = p.k_blocks_per_split * (BLOCK_K / 16);    // build_halo_tab(): one per k16 step
  const int area = halo ? std::max(ring + 2 * p.hbytes, stage_f32_bytes<BN>() + 1024)
                   : band ? std::max(ring + NS * p.hbytes + 128, band_f32_bytes<BN>() + 1024)
                          : ring;
  const int smem = area + ((p.ktab_n + 3) & ~3) * 4 + BN * 4;
  launch_k(gemm_umma_k<BN, AM, BM, GK, GV, NS>, grid, kthreads<AM>(), smem, st, ta, tb, p);
  return (int)cudaGetLastError();
}

template <int BN, int AM, int BM, int GK, int GV>
static int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int splits,
                      cudaStream_t st) {
  // halo kernels: one tile = two 8x8 pixel blocks, numbered over (image, block row, block column)
  // band kernels: BAND_GROUPS (plane, ky) groups per CTA
  const int m_tiles = AM == A_HALO ? (p.g.N * p.hnby * p.hnbx + 1) / 2
                      : AM == A_HALO_MN ? (p.bvgroups + BAND_GROUPS - 1) / BAND_GROUPS
                                        : (p.M + BLOCK_M - 1) / BLOCK_M;
  dim3 grid((p.N + BN - 1) / BN, m_tiles, splits);
  // Short reductions (K <= 4 k-blocks, e.g. a 5x5 first layer on 8 padded channels) in grids of
  // several waves: a 3-stage ring already holds almost the whole K and is small enough for a
  // third CTA per SM (these kernels are latency bound).
  if constexpr (AM == A_GATHER_K && GV == 2 && BN <= 64) {
    const long long ctas = (long long)grid.x * grid.y * grid.z;
    static int s3 = -1;
    if (s3 < 0) { const char* e = getenv("ZNICZ_UMMA_S3"); s3 = e ? atoi(e) : 1; }
    if (s3 && p.k_blocks_per_split <= 4 && ctas > 2 * num_sms())
      return launch_stages<BN, AM, BM, GK, GV, 3>(ta, tb, p, grid, st);
  }
  // Halo kernels keep only B in the ring, and the MMAs of a k-block are a few hundred cycles: with
  // 4 stages a 13-k-block reduction (5x5 x 32 channels) waits on ~3 serial refill round trips.
  // 8 B stages halve that; short reductions keep 4 stages and their CTAs per SM.
  // Band kernels likewise: an 8-stage ring of err tiles and bands for reductions longer than 4.
  if constexpr (AM == A_HALO || AM == A_HALO_MN) {
    if (p.k_blocks_per_split > STAGES_DEFAULT) return launch_stages<BN, AM, BM, GK, GV, 8>(ta, tb, p, grid, st);
  }
  return launch_stages<BN, AM, BM, GK, GV, STAGES_DEFAULT>(ta, tb, p, grid, st);
}

// B K-major: BLOCK_N in {16, 32, 64, 128}; B MN-major: {64, 128}
template <int AM, int BM, int GK, int GV>
static int launch_bn(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                     int splits, cudaStream_t st) {
  if constexpr (BM == B_TMA_K) {
    switch (bn) {
      case 16: return launch_cfg<16, AM, BM, GK, GV>(ta, tb, p, splits, st);
      case 32: return launch_cfg<32, AM, BM, GK, GV>(ta, tb, p, splits, st);
      case 64: return launch_cfg<64, AM, BM, GK, GV>(ta, tb, p, splits, st);
      case 128: return launch_cfg<128, AM, BM, GK, GV>(ta, tb, p, splits, st);
      default: return -2;
    }
  } else {
    switch (bn) {
      case 64: return launch_cfg<64, AM, BM, GK, GV>(ta, tb, p, splits, st);
      case 128: return launch_cfg<128, AM, BM, GK, GV>(ta, tb, p, splits, st);
      default: return -2;
    }
  }
}

static int pick_bn(int N) { return N <= 16 ? 16 : (N <= 32 ? 32 : (N <= 64 ? 64 : 128)); }

int pair_wgrad_splits(int, int, int, int);      // gemm_pair.cu

int umma_pick_splits(int M, int N, int K, int max_splits) {
  {
    // conv wgrad shapes served by the persistent kernel (gemm_pair.cu) want ~one work item per SM
    const int sp = pair_wgrad_splits(M, N, K, max_splits);
    if (sp > 0) return sp;
  }
  int bn = pick_bn(N);
  if (bn < 64) bn = 64;
  long long tiles = (long long)((M + BLOCK_M - 1) / BLOCK_M) * ((N + bn - 1) / bn);
  int kb = (K + BLOCK_K - 1) / BLOCK_K;
  int s = (int)((num_sms() + tiles - 1) / tiles);
  if (s > kb) s = kb;
  if (s > max_splits) s = max_splits;
  return s < 1 ? 1 : s;
}

// Dense GEMM. a_mn = 0: A stored [M][lda] (K contiguous); 1: A stored [K][lda] (M contiguous).
// b_mn = 0: B stored [N][ldb] (K contiguous); 1: B stored [K][ldb] (N contiguous).
// Returns 0 on success; non-zero = not launched (caller must fall back loudly).
int launch_gemm_umma(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn,
                     void* out, int out_bf16, long long ldo, int out_trans, int M, int N, int K,
                     const float* bias, int act, float alpha, float beta, int splits,
                     long long split_stride, cudaStream_t st) {
  if ((lda % 8) || (ldb % 8) || ((uintptr_t)a & 15) || ((uintptr_t)b & 15)) return -3;
  CUtensorMap ta, tb;
  int bn = pick_bn(N);
  if (b_mn && bn < 64) bn = 64;
  int r;
  if (a_mn) r = make_map(&ta, a, M, K, lda, 64); else r = make_map(&ta, a, K, M, lda, BLOCK_M);
  if (r) return r;
  if (b_mn) r = make_map(&tb, b, N, K, ldb, 64); else r = make_map(&tb, b, K, N, ldb, bn);
  if (r) return r;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  int total_kb = (K + BLOCK_K - 1) / BLOCK_K;
  if (splits < 1) splits = 1;
  p.k_blocks_per_split = (total_kb + splits - 1) / splits;
  splits = (total_kb + p.k_blocks_per_split - 1) / p.k_blocks_per_split;
  p.out = out; p.out_bf16 = out_bf16; p.ldo = ldo; p.out_trans = out_trans;
  p.bias = bias; p.act = act; p.alpha = alpha; p.beta = beta; p.split_stride = split_stride;
  p.gather_kind = G_NONE;
  if (!a_mn && !b_mn) return launch_bn<A_TMA_K, B_TMA_K, 0, 0>(bn, ta, tb, p, splits, st);
  // MN-major B tiles are built from 64-wide swizzle atoms: never go below UMMA_N = 64 there
  if (!a_mn && b_mn) return launch_bn<A_TMA_K, B_TMA_MN, 0, 0>(bn, ta, tb, p, splits, st);
  if (a_mn && !b_mn) return launch_bn<A_TMA_MN, B_TMA_K, 0, 0>(bn, ta, tb, p, splits, st);
  return launch_bn<A_TMA_MN, B_TMA_MN, 0, 0>(bn, ta, tb, p, splits, st);
}

static ConvGeomU geom(int N, int H, int W, int C, int OH, int OW, int F, int KY, int KX, int SY, int SX,
                      int PT, int PL, int vec) {
  ConvGeomU g{N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL, vec, 0, KY * KX, 0};
  return g;
}
// Enable the tap-mode gather when the inner (channel) extent tiles a 64-wide reduction block.
static bool set_tap_mode(ConvGeomU& g, int inner, bool dgrad) {
  g.tpk = 0; g.inner = inner;
  if (!g.vec || (inner % 8) || g.KY * g.KX > KTAB) return false;
  if (dgrad && (g.SY != 1 || g.SX != 1)) return false;
  if (inner >= 64) { if (inner % 64) return false; g.tpk = 1; return true; }
  if (64 % inner) return false;
  g.tpk = 64 / inner;
  return true;
}

int launch_conv_fprop_pair(const void*, const void*, long long, const float*, void*, int, int, int, int, int,
                           int, int, int, int, int, int, int, int, int, cudaStream_t);
int launch_conv_dgrad_pair(const void*, const void*, long long, void*, int, int, int, int, int, int, int, int,
                           int, int, int, float, const void*, int, cudaStream_t);
int launch_conv_wgrad_pair(const void*, const void*, float*, int, int, int, int, int, int, int, int, int, int,
                           int, int, int, int, cudaStream_t);
int pair_wgrad_splits(int, int, int, int);
static long long g_pair_conv_launches = 0;
long long conv_pair_launches() { return g_pair_conv_launches; }

// out[pix, f] = act(im2col(x)[pix, :] . w_lp[f, :] + bias[f]); w_lp stored [F][ldw] bf16 (ldw % 8 == 0)
int launch_conv_fprop_umma(const void* x, const void* w_lp, long long ldw, const float* bias, void* out,
                           int out_bf16, int N, int H, int W, int C, int OH, int OW, int F, int KY, int KX,
                           int SY, int SX, int PT, int PL, int act, cudaStream_t st) {
  if ((ldw % 8) || ((uintptr_t)w_lp & 15) || ((uintptr_t)x & 15)) return -3;
  if (out_bf16 && launch_conv_fprop_pair(x, w_lp, ldw, bias, out, N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT,
                                         PL, act, st) == 0) {
    ++g_pair_conv_launches;        // large layer: persistent kernel, A by TMA im2col
    return 0;
  }
  int Kw = KY * KX * C;
  if ((C % 8 == 0 ? (Kw + 7) / 8 : Kw) > KTAB || KY > 255 || KX > 255) return -4;
  CUtensorMap ta, tb;
  int bn = pick_bn(F);
  int r = make_map(&tb, w_lp, ldw, F, ldw, bn);
  if (r) return r;
  ta = tb;
  GemmParams p{};
  p.M = N * OH * OW; p.N = F; p.K = Kw;
  p.k_blocks_per_split = (Kw + BLOCK_K - 1) / BLOCK_K;
  p.out = out; p.out_bf16 = out_bf16; p.ldo = F; p.out_trans = 0;
  p.bias = bias; p.act = act; p.alpha = 1.f; p.beta = 0.f; p.split_stride = 0;
  p.gsrc = (const __nv_bfloat16*)x; p.g = geom(N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL, C % 8 == 0);
  p.gather_kind = G_IM2COL; p.gK = Kw;
  if (C % 64 == 0 && im2col_tma_enabled()) {
    // A operand by TMA im2col: window bases -PL .. W + upper_w, OW x OH of them
    CUtensorMap ti;
    if (make_map_im2col(&ti, x, N, H, W, C, -PL, -PT, (OW - 1) * SX + 1 - PL - W,
                        (OH - 1) * SY + 1 - PT - H, SX, SY, BLOCK_M) == 0) {
      p.g.inner = C;
      ++g_im2col_launches;
      return launch_bn<A_IM2COL_K, B_TMA_K, G_IM2COL, 0>(bn, ti, tb, p, 1, st);
    }
  }
  if (set_tap_mode(p.g, C, false)) {
    if (halo_eligible(p, false)) {
      CUtensorMap th;
      r = make_map_halo(&th, x, N, H, W, C, KY, KX);
      if (r) return r;
      ++g_halo_launches;
      int smem = 0;
      if (const int pbn = persist_bn(p, smem)) {
        CUtensorMap tp;                          // B box {64, pbn}
        r = make_map(&tp, w_lp, ldw, F, ldw, pbn);
        if (r) return r;
        return pbn == 16 ? launch_persist<16, G_IM2COL>(th, tp, p, smem, st)
                         : launch_persist<32, G_IM2COL>(th, tp, p, smem, st);
      }
      return launch_bn<A_HALO, B_TMA_K, G_IM2COL, 0>(bn, th, tb, p, 1, st);
    }
    return launch_bn<A_GATHER_K, B_TMA_K, G_IM2COL, 2>(bn, ta, tb, p, 1, st);
  }
  if (C % 8 == 0) return launch_bn<A_GATHER_K, B_TMA_K, G_IM2COL, 1>(bn, ta, tb, p, 1, st);
  return launch_bn<A_GATHER_K, B_TMA_K, G_IM2COL, 0>(bn, ta, tb, p, 1, st);
}

// err_in[ipix, c] = alpha * sum_{tap,f} gather(err_out) * wd_lp[(tap,f), c] + beta * err_in
// wd_lp stored [KY*KX*F][ldc] bf16 (ldc % 8 == 0, zero padded columns)
int launch_conv_dgrad_umma(const void* err_out, const void* wd_lp, long long ldc, void* err_in,
                           int ei_bf16, int N, int H, int W, int C, int OH, int OW, int F, int KY, int KX,
                           int SY, int SX, int PT, int PL, float alpha, float beta, const void* dmul,
                           int dact, cudaStream_t st) {
  // the folded derivative needs the inline bf16 epilogue mode (row-major bf16 output, no beta)
  if (dmul && (!ei_bf16 || beta != 0.f || ((uintptr_t)dmul & 15))) return -5;
  if ((ldc % 8) || ((uintptr_t)wd_lp & 15) || ((uintptr_t)err_out & 15)) return -3;
  if (ei_bf16 && beta == 0.f && SY == 1 && SX == 1 &&
      launch_conv_dgrad_pair(err_out, wd_lp, ldc, err_in, N, H, W, C, OH, OW, F, KY, KX, PT, PL, alpha, dmul,
                             dact, st) == 0) {
    ++g_pair_conv_launches;
    return 0;
  }
  int Kd = KY * KX * F;
  if ((F % 8 == 0 ? (Kd + 7) / 8 : Kd) > KTAB || KY > 255 || KX > 255) return -4;
  CUtensorMap ta, tb;
  int bn = pick_bn(C);
  if (bn < 64) bn = 64;
  int r = make_map(&tb, wd_lp, ldc, Kd, ldc, 64);
  if (r) return r;
  ta = tb;
  GemmParams p{};
  p.M = N * H * W; p.N = C; p.K = Kd;
  p.k_blocks_per_split = (Kd + BLOCK_K - 1) / BLOCK_K;
  p.out = err_in; p.out_bf16 = ei_bf16; p.ldo = C; p.out_trans = 0;
  p.bias = nullptr; p.act = 0; p.alpha = alpha; p.beta = beta; p.split_stride = 0;
  p.gsrc = (const __nv_bfloat16*)err_out;
  p.g = geom(N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL, F % 8 == 0);
  p.gather_kind = G_DGRAD; p.gK = Kd;
  p.dmul = (const __nv_bfloat16*)dmul; p.dact = dmul ? dact : 0;
  if (F % 64 == 0 && SY == 1 && SX == 1 && im2col_tma_enabled()) {
    // unit stride: dgrad is a correlation of err_out with the flipped filter; W x H window bases
    // starting at -(K - 1 - pad) over the [N][OH][OW][F] tensor
    CUtensorMap ti;
    const int lw = -(KX - 1 - PL), lh = -(KY - 1 - PT);
    if (make_map_im2col(&ti, err_out, N, OH, OW, F, lw, lh, W + lw - OW, H + lh - OH, 1, 1,
                        BLOCK_M) == 0) {
      p.g.inner = F;
      ++g_im2col_launches;
      return launch_bn<A_IM2COL_K, B_TMA_MN, G_DGRAD, 0>(bn, ti, tb, p, 1, st);
    }
  }
  if (set_tap_mode(p.g, F, true)) {
    if (halo_eligible(p, true)) {
      CUtensorMap th;
      r = make_map_halo(&th, err_out, N, OH, OW, F, KY, KX);
      if (r) return r;
      ++g_halo_launches;
      int smem = 0;
      if (persist_bn(p, smem) == 32) {          // C <= 16 keeps A_HALO (B tiles are 32 columns)
        CUtensorMap tp;                          // B box {32, 64}, SWIZZLE_64B
        r = make_map(&tp, wd_lp, ldc, Kd, ldc, BLOCK_K, 32);
        if (r) return r;
        return launch_persist<32, G_DGRAD>(th, tp, p, smem, st);
      }
      return launch_bn<A_HALO, B_TMA_MN, G_DGRAD, 0>(bn, th, tb, p, 1, st);
    }
    return launch_bn<A_GATHER_K, B_TMA_MN, G_DGRAD, 2>(bn, ta, tb, p, 1, st);
  }
  if (F % 8 == 0) return launch_bn<A_GATHER_K, B_TMA_MN, G_DGRAD, 1>(bn, ta, tb, p, 1, st);
  return launch_bn<A_GATHER_K, B_TMA_MN, G_DGRAD, 0>(bn, ta, tb, p, 1, st);
}

// partials[z][f][kidx] = sum_{pix in split z} err_out[pix, f] * im2col(x)[pix, kidx]
// (computed as D[kidx, f] with the im2col operand on the 128-wide M side, stored transposed)
__device__ __align__(16) unsigned short zn_ones_bf16[8] = {0x3F80, 0, 0, 0, 0, 0, 0, 0};

// Returns 0, or 1 when ``bias_parts`` [splits][F] was filled with the per-split column sums of
// err_out as well (tap-mode gather and Kw % 128 != 0, i.e. the last M tile has a spare row).
int launch_conv_wgrad_umma(const void* err_out, const void* x, float* partials, int splits, int N, int H,
                           int W, int C, int OH, int OW, int F, int KY, int KX, int SY, int SX, int PT,
                           int PL, float* bias_parts, cudaStream_t st) {
  if ((F % 8) || ((uintptr_t)err_out & 15) || ((uintptr_t)x & 15)) return -3;
  if (launch_conv_wgrad_pair(err_out, x, partials, splits, N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL,
                             st) == 0) {
    ++g_pair_conv_launches;        // (no bias row: the caller falls back to the column-sum kernel)
    return 0;
  }
  int Kw = KY * KX * C, P = N * OH * OW;
  if ((C % 8 == 0 ? (Kw + 7) / 8 : Kw) > KTAB || KY > 255 || KX > 255) return -4;
  CUtensorMap ta, tb;
  int bn = pick_bn(F);
  if (bn < 64) bn = 64;
  int r = make_map(&tb, err_out, F, P, F, 64);
  if (r) return r;
  ta = tb;
  GemmParams p{};
  p.M = Kw; p.N = F; p.K = P;
  int total_kb = (P + BLOCK_K - 1) / BLOCK_K;
  if (splits < 1) splits = 1;
  p.k_blocks_per_split = (total_kb + splits - 1) / splits;
  p.out = partials; p.out_bf16 = 0; p.ldo = Kw; p.out_trans = 1;
  p.bias = nullptr; p.act = 0; p.alpha = 1.f; p.beta = 0.f; p.split_stride = (long long)F * Kw;
  p.gsrc = (const __nv_bfloat16*)x; p.g = geom(N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL, C % 8 == 0);
  p.gather_kind = G_IM2COL; p.gK = Kw;
  if (set_tap_mode(p.g, C, false)) {
    bool row = bias_parts != nullptr && (Kw % BLOCK_M) != 0;
    if (row) {
      static void* ones = nullptr;
      if (!ones && cudaGetSymbolAddress(&ones, zn_ones_bf16) != cudaSuccess) ones = nullptr;
      row = ones != nullptr;
      if (row) { p.g.ones = (const __nv_bfloat16*)ones; p.bias_out = bias_parts; }
    }
    if (bn == 64 && band_eligible(p)) {
      // the same products in the same pixel order as the gather below (and the bias row exactly
      // where it would have one), from one band of x per k-block instead of a gather per tap
      CUtensorMap th;
      r = make_map_halo(&th, x, N, H, W, C, KY, KX, p.bw, p.bh);
      if (r) return r;
      ++g_halo_launches;
      r = launch_cfg<64, A_HALO_MN, B_TMA_MN, G_IM2COL, 0>(th, tb, p, splits, st);
      return (r == 0 && row) ? 1 : r;
    }
    r = launch_bn<A_GATHER_MN, B_TMA_MN, G_IM2COL, 2>(bn, ta, tb, p, splits, st);
    return (r == 0 && row) ? 1 : r;
  }
  if (C % 8 == 0) return launch_bn<A_GATHER_MN, B_TMA_MN, G_IM2COL, 1>(bn, ta, tb, p, splits, st);
  return launch_bn<A_GATHER_MN, B_TMA_MN, G_IM2COL, 0>(bn, ta, tb, p, splits, st);
}

}  // namespace zn
