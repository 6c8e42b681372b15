// Dense GEMM for large shapes, persistent warp-specialised form (sm_90a):
//
//   D[M, N] = act(alpha * sum_k A[m, k] * B[n, k] + bias[n])        A, B bf16, D bf16 / fp32
//
// * one CTA per SM loops over 128 x BN output tiles (grouped raster: 8 M-tiles x all N-tiles per
//   group, so a wave re-reads A and B from L2);
// * warpgroup 0 is the producer (one thread issues the TMA loads of a deep ring: 4 x 48 KB stages
//   at BN = 256, 6 x 32 KB at BN = 128) and hands its registers to the two MMA warpgroups;
// * warpgroups 1 and 2 each own 64 rows of the tile: wgmma m64 x BN x k16 with the fp32
//   accumulators in registers, then the epilogue (bias / activation / f' -> swizzled smem -> TMA
//   store, two staging buffers so the store of one chunk overlaps the next);
// * the ring runs ahead across tiles: the loads of tile t + 1 are in flight during the epilogue
//   of tile t.
//
// Used for the large fully-connected layers and convolutions; skinny / small shapes stay on
// gemm_umma.cu.
//
// fp8 operand mode (AM_FP8, BN = 128 only): A [M][K] and B [N][K] hold e4m3 codes with one fp32
// scale per row and 128-element k-block (scales [KB][rows rounded up to 128], written by fp8.cu):
//
//   D[m, n] = act(alpha * sum_kb sA[kb][m] sB[kb][n] P_kb[m, n] + bias[n])
//
// One stage is one k-block (128 e4m3 = one 128-byte SW128 row); the producer also fetches the
// stage's 2 x 128 scales with two bulk copies. Each MMA warpgroup issues four wgmma m64n128k32
// e4m3 into a temporary fragment P_kb (the tensor core's partial sums never span more than one
// k-block), waits, and promotes sA sB P_kb into its fp32 accumulators with one FMA per element.
// Any M, N, K >= 1: the tails arrive as TMA zero fill.
#include "common.cuh"
#include "umma.cuh"
#include <stdlib.h>
#include <utility>

namespace zn {

using namespace umma;

namespace pr {

constexpr int BM = 128;                 // rows per tile (two 64-row MMA warpgroups)
constexpr int BK = 64;                  // bf16 elements = 128 bytes = one SW128 row
constexpr int A_BYTES = BM * 128;
constexpr int EPI_BUF = 128 * 128;      // 128 rows x 128 bytes per staging buffer
constexpr int THREADS = 384;

// A operand: dense [M][K] tile, or the implicit-GEMM operand of a convolution fetched by TMA in
// im2col mode (one [128 pixels x 64 channels] box per k-block): fprop = im2col(x), dgrad
// (unit stride) = windows of err_out for the flipped filter.
enum { AM_DENSE = 0, AM_IM2COL_FPROP = 1, AM_IM2COL_DGRAD = 2,
       AM_DENSE_MN = 3,            // A stored [K][M] (M contiguous): err^T of the weight-gradient GEMMs
       AM_FP8 = 4 };               // A, B: block-scaled e4m3 [rows][K] (see the top of the file)
// B operand: K-major tile, MN-major tile ([K][N], N contiguous), or - conv wgrad - the im2col
// operand as MN-major blocks fetched by TMA im2col ([64 pixels][64 channels of one tap])
enum { BM_K = 0, BM_MN = 1, BM_IM2COL_MN = 2 };

struct ConvP { int H, W, OH, OW, KY, KX, SY, SX, PT, PL, inner; };

struct Params {
  int M, N, K;
  const float* bias; int act; float alpha;
  int tiles_m, tiles_n;
  int splits, kb_per_split;       // split-K over the reduction (fp32 partials [splits][M][N])
  ConvP g;
  const __nv_bfloat16* dmul; int dact; long long ldo;   // dgrad: out *= f'(dmul[row][col])
  const float* sa; const float* sb;                      // fp8: scales [KB][sa_pitch], [KB][sb_pitch]
  int sa_pitch, sb_pitch;
};

__device__ __forceinline__ void tma_store_wait_read(int keep) {
  if (keep == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  else asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}

// grouped raster: GM consecutive M-tiles share a sweep over all N-tiles
__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int& tm, int& tn) {
  constexpr int GM = 8;
  const int per_group = GM * tiles_n;
  const int g = t / per_group, r = t - g * per_group;
  const int m0 = g * GM;
  const int gm = min(GM, tiles_m - m0);
  tn = r / gm;
  tm = m0 + (r - tn * gm);
}

template <typename F, int... I>
__device__ __forceinline__ void static_for(std::integer_sequence<int, I...>, F&& f) {
  (f(std::integral_constant<int, I>{}), ...);
}

template <int BN, int AMODE = AM_DENSE>
__host__ __device__ constexpr int pair_stages() { return AMODE == AM_FP8 ? 5 : (BN == 256 ? 4 : 6); }
// dynamic shared memory: stages, two epilogue staging buffers, fp8 scales (1 KB per stage), alignment
template <int BN, int AMODE>
__host__ __device__ constexpr int pair_smem() {
  return pair_stages<BN, AMODE>() * (A_BYTES + BN * 128 + (AMODE == AM_FP8 ? 1024 : 0)) + 2 * EPI_BUF +
         1024;
}

template <int BN, bool OUT_F32, int AMODE = AM_DENSE, int BMODE = BM_K>
__global__ void __launch_bounds__(THREADS, 1)
gemm_pair_k(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_c, const Params p) {
  constexpr int B_BYTES = BN * 128;
  constexpr int STAGE = A_BYTES + B_BYTES;
  constexpr int NST = pair_stages<BN, AMODE>();
  constexpr int EPI_COLS = OUT_F32 ? 32 : 64;          // 128-byte staging rows
  constexpr int NCHUNK = BN / EPI_COLS;
  constexpr int ESZ = OUT_F32 ? 4 : 2;
  constexpr bool A_MN = (AMODE == AM_DENSE_MN);
  constexpr bool B_MN = (BMODE != BM_K);
  constexpr bool FP8 = (AMODE == AM_FP8);
  constexpr int KSTEP = FP8 ? 128 : BK;                 // reduction elements per stage
  static_assert(!FP8 || (BN == 128 && BMODE == BM_K), "fp8 mode: BN = 128, K-major B");

  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[NST];
  __shared__ __align__(8) uint64_t empty_bar[NST];

  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* epi = tiles + (size_t)NST * STAGE;          // 2 x EPI_BUF, 1024-byte aligned
  uint8_t* scl = epi + 2 * EPI_BUF;                    // fp8: per stage sA[128] then sB[128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int splits = p.splits > 1 ? p.splits : 1;
  const int num_tiles = p.tiles_m * p.tiles_n * splits;      // work items (tile, k-split)
  const int total_kb = (p.K + KSTEP - 1) / KSTEP;

  if (threadIdx.x == 0) {
    // fp8 mode: every consumer warp releases the stage (it also read the stage's scales)
    for (int s = 0; s < NST; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], FP8 ? 8u : 2u); }
    fence_barrier_init();
    tma_prefetch_desc(&tmap_a); tma_prefetch_desc(&tmap_b); tma_prefetch_desc(&tmap_c);
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== producer warpgroup =====================
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int tm, tn;
        tile_coords(t / splits, p.tiles_m, p.tiles_n, tm, tn);
        const int split = t % splits;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = splits > 1 ? min(total_kb, kb0 + p.kb_per_split) : total_kb;
        const int m0 = tm * BM, n0 = tn * BN;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % NST; const uint32_t ph = (it / NST) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = tiles + (size_t)s * STAGE;
          uint32_t tx = STAGE;
          int nblk = BN / 64;                  // 64-wide B blocks (im2col B only)
          if (BMODE == BM_IM2COL_MN) {
            // blocks past the last reduction-weight index are not fetched
            const int left = p.N - n0;
            nblk = left <= 0 ? 0 : min(BN / 64, (left + 63) / 64);
            tx = A_BYTES + (uint32_t)nblk * 8192u;
          }
          if (FP8) tx += 1024;
          mbar_arrive_expect_tx(&full_bar[s], tx);
          if (FP8) {
            tma_load_2d(sa, &tmap_a, &full_bar[s], kb * KSTEP, m0);
            bulk_load(scl + s * 1024, p.sa + (long long)kb * p.sa_pitch + m0, 512, &full_bar[s]);
            bulk_load(scl + s * 1024 + 512, p.sb + (long long)kb * p.sb_pitch + n0, 512, &full_bar[s]);
          } else if (AMODE == AM_DENSE) {
            tma_load_2d(sa, &tmap_a, &full_bar[s], kb * BK, m0);
          } else if (AMODE == AM_DENSE_MN) {
            // A stored [K][M]: two [64 k][64 m] boxes for the tile's 128 rows
            tma_load_2d(sa, &tmap_a, &full_bar[s], m0, kb * BK);
            tma_load_2d(sa + 8192, &tmap_a, &full_bar[s], m0 + 64, kb * BK);
          } else {
            // the tile's 128 pixels start at m0; k-block = 64 channels of one filter tap
            const ConvP& g = p.g;
            const int k0 = kb * BK;
            const int tap = k0 / g.inner, c0 = k0 - tap * g.inner;
            const int ky = tap / g.KX, kx = tap - ky * g.KX;
            int w0, h0, n, ow, oh;
            if (AMODE == AM_IM2COL_FPROP) {
              const int q = m0 % g.OW; const int t2 = m0 / g.OW;
              const int pr = t2 % g.OH; n = t2 / g.OH;
              w0 = q * g.SX - g.PL; h0 = pr * g.SY - g.PT; ow = kx; oh = ky;
            } else {
              const int ix = m0 % g.W; const int t2 = m0 / g.W;
              const int iy = t2 % g.H; n = t2 / g.H;
              w0 = ix - (g.KX - 1 - g.PL); h0 = iy - (g.KY - 1 - g.PT);
              ow = g.KX - 1 - kx; oh = g.KY - 1 - ky;
            }
            tma_load_im2col_4d(sa, &tmap_a, &full_bar[s], c0, w0, h0, n, (uint16_t)ow, (uint16_t)oh);
          }
          if (BMODE == BM_K) {
            tma_load_2d(sa + A_BYTES, &tmap_b, &full_bar[s], kb * KSTEP, n0);
          } else if (BMODE == BM_MN) {
            // B stored [K][N] (N contiguous): 64 x 64 boxes, one per 64 columns of the tile
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_2d(sa + A_BYTES + j * 8192, &tmap_b, &full_bar[s], n0 + j * 64, kb * BK);
          } else {
            // conv wgrad: reduction = pixels kb * 64 .., N = (tap, channel); one im2col box of
            // [64 pixels][64 channels] per 64-wide N block
            const ConvP& g = p.g;
            const int pix0 = kb * BK;
            const int q = pix0 % g.OW; const int t2 = pix0 / g.OW;
            const int pr = t2 % g.OH; const int n = t2 / g.OH;
            const int w0 = q * g.SX - g.PL, h0 = pr * g.SY - g.PT;
            for (int j = 0; j < nblk; ++j) {
              const int kidx0 = n0 + j * 64;
              const int tap = kidx0 / g.inner, c0 = kidx0 - tap * g.inner;
              tma_load_im2col_4d(sa + A_BYTES + j * 8192, &tmap_b, &full_bar[s], c0, w0, h0, n,
                                 (uint16_t)(tap % g.KX), (uint16_t)(tap / g.KX));
            }
          }
        }
      }
    }
    return;
  }

  // ===================== MMA warpgroups 1, 2: rows 64 (wg - 1) .. + 63 of the tile =============
  reg_alloc<232>();
  const int half = wg - 1;
  const int et = threadIdx.x - 128;                     // 0..255: consumer thread
  const int wq = warp & 3;                              // warp within the warpgroup
  const int lr = half * 64 + 16 * wq + (lane >> 2);     // tile row of fragment rows h = 0 (+8 for h = 1)
  const int cq = 2 * (lane & 3);
  uint32_t it = 0, chunk_no = 0;
  float acc[BN / 2];
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    int tm, tn;
    tile_coords(t / splits, p.tiles_m, p.tiles_n, tm, tn);
    const int split = t % splits;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = splits > 1 ? min(total_kb, kb0 + p.kb_per_split) : total_kb;
    const int m0 = tm * BM, n0 = tn * BN;
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    if constexpr (FP8) {
      float tmp[BN / 2];
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % NST; const uint32_t ph = (it / NST) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sa = smem_u32(tiles + (size_t)s * STAGE) + half * 8192;
        const uint32_t sb = smem_u32(tiles + (size_t)s * STAGE) + A_BYTES;
        const float* ss = reinterpret_cast<const float*>(scl + s * 1024);
        wg_fence();
        const uint64_t da = make_smem_desc(sa, 16, 1024), db = make_smem_desc(sb, 16, 1024);
#pragma unroll
        for (int k = 0; k < 4; ++k)        // P_kb = sum of four k32 products, from zero
          wgmma_e4m3_n128(tmp, da + 2 * k, db + 2 * k, k > 0);   // +32 bytes per k32 step
        wg_commit();
        wg_wait<0>();
        wg_fence_regs(tmp);
        const float a0 = ss[lr], a1 = ss[lr + 8];
        // (scales of B read inside the loop: holding all 32 across the wait spills)
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const float2 b = *reinterpret_cast<const float2*>(ss + 128 + 8 * i + cq);
          acc[4 * i + 0] = fmaf(a0 * b.x, tmp[4 * i + 0], acc[4 * i + 0]);
          acc[4 * i + 1] = fmaf(a0 * b.y, tmp[4 * i + 1], acc[4 * i + 1]);
          acc[4 * i + 2] = fmaf(a1 * b.x, tmp[4 * i + 2], acc[4 * i + 2]);
          acc[4 * i + 3] = fmaf(a1 * b.y, tmp[4 * i + 3], acc[4 * i + 3]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      }
    } else {
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % NST; const uint32_t ph = (it / NST) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint32_t sa = smem_u32(tiles + (size_t)s * STAGE) + half * 8192;
      const uint32_t sb = smem_u32(tiles + (size_t)s * STAGE) + A_BYTES;
      wg_fence_regs(acc);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t da = A_MN ? make_smem_desc(sa + k * 2048, 8192, 1024)
                                 : make_smem_desc(sa + k * 32, 16, 1024);
        const uint64_t db = B_MN ? make_smem_desc(sb + k * 2048, 8192, 1024)
                                 : make_smem_desc(sb + k * 32, 16, 1024);
        wgmma_bf16<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, 1);
      }
      wg_commit();
      wg_fence_regs(acc);
      wg_wait<1>();                                     // the previous k-block's MMAs retired
      if (kb > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % NST]);
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (kb1 > kb0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % NST]);
    }

    // ---- epilogue: registers -> swizzled staging chunk -> one TMA store per chunk ----
    // split-K partial s lives at rows [s * M, (s + 1) * M) of the output map
    const bool store_ok = m0 < p.M;
    const int row0 = split * p.M + m0;
    // (chunk index as a compile-time constant: the accumulator array stays in registers)
    static_for(std::make_integer_sequence<int, NCHUNK>{}, [&](auto cc_) {
      constexpr int c = decltype(cc_)::value;
      uint8_t* buf = epi + (chunk_no & 1) * EPI_BUF;
      // the TMA store that read this buffer two chunks ago must be done with it
      if (et == 0) tma_store_wait_read(1);
      named_bar_sync(1, 256);
      // this chunk's accumulators (compile-time indices), then a rolled loop over them: the
      // activation / derivative code is emitted once, not once per element
      float v[EPI_COLS / 2];
#pragma unroll
      for (int k = 0; k < EPI_COLS / 2; ++k) v[k] = acc[c * (EPI_COLS / 2) + k];
#pragma unroll 1
      for (int q = 0; q < EPI_COLS / 4; ++q) {
        const int ii = q >> 1, h = q & 1;               // register pair 4 ii + 2 h (+1)
        const int cc = ii * 8 + cq;                     // column inside the chunk
        const int n = n0 + c * EPI_COLS + cc;
        const int r = lr + 8 * h;
        const float b0 = (p.bias != nullptr && n < p.N) ? __ldg(p.bias + n) : 0.f;
        const float b1 = (p.bias != nullptr && n + 1 < p.N) ? __ldg(p.bias + n + 1) : 0.f;
        float v0 = act_fwd5_fast(p.act, fmaf(v[2 * q], p.alpha, b0));
        float v1 = act_fwd5_fast(p.act, fmaf(v[2 * q + 1], p.alpha, b1));
        const int byte = cc * ESZ;
        uint8_t* dst = buf + r * 128 + (((byte >> 4) ^ (r & 7)) << 4) + (byte & 15);
        if (OUT_F32) {
          *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
        } else {
          const int row = m0 + r;
          if (p.dmul != nullptr && row < p.M) {
            // err_input *= f'(x): x has the layout of the output (row pitch ldo)
            const __nv_bfloat16* dx = p.dmul + (long long)row * p.ldo + n;
            if (n < p.N) v0 *= act_deriv(p.dact, 0.f, __bfloat162float(dx[0]));
            if (n + 1 < p.N) v1 *= act_deriv(p.dact, 0.f, __bfloat162float(dx[1]));
          }
          *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 256);
      if (et == 0) {
        if (store_ok) tma_store_2d(&tmap_c, buf, n0 + c * EPI_COLS, row0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      ++chunk_no;
    });
  }
  if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &qr) != cudaSuccess || !q)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(q);
  }
  return fn;
}
// 2-D map, inner dim contiguous, row pitch `ld` elements, box {box_inner, box_rows}, SWIZZLE_128B
static int make_map(CUtensorMap* m, const void* ptr, CUtensorMapDataType dt, int esize, long long inner,
                    long long outer, long long ld, int box_inner, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -1;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)(ld * esize)};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

template <int BN, bool OUT_F32, int AMODE = AM_DENSE, int BMODE = BM_K>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const Params& p,
                  cudaStream_t st) {
  constexpr int smem = pair_smem<BN, AMODE>();
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_pair_k<BN, OUT_F32, AMODE, BMODE>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int tiles = p.tiles_m * p.tiles_n * (p.splits > 1 ? p.splits : 1);
  const int ctas = tiles < num_sms() ? tiles : num_sms();
  gemm_pair_k<BN, OUT_F32, AMODE, BMODE><<<dim3(ctas), dim3(THREADS), smem, st>>>(ta, tb, tc, p);
  return (int)cudaGetLastError();
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// im2col-mode map over NHWC bf16 [N][H][W][C]: 128 window positions x 64 channels per load
static int make_map_im2col(CUtensorMap* m, const void* ptr, int N, int H, int W, int C, int lower_w,
                           int lower_h, int upper_w, int upper_h, int stride_w, int stride_h,
                           int pixels = BM) {
  static EncodeIm2colFn enc = nullptr;
  if (!enc) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &q, cudaEnableDefault, &qr) != cudaSuccess || !q)
      return -1;
    enc = reinterpret_cast<EncodeIm2colFn>(q);
  }
  const int v[6] = {lower_w, lower_h, upper_w, upper_h, 0, 0};
  for (int i = 0; i < 4; ++i) if (v[i] < -128 || v[i] > 127) return -7;
  if (stride_w > 8 || stride_h > 8) return -7;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lower[2] = {lower_w, lower_h};
  int upper[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1u, (cuuint32_t)stride_w, (cuuint32_t)stride_h, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower,
                   upper, 64u, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}
static bool conv_pair_enabled() {
  static int on = -1;
  if (on < 0) { const char* e = getenv("ZNICZ_CONV_PAIR"); on = (e && atoi(e) == 0) ? 0 : 1; }
  return on != 0;
}

static long long g_fp8_launches = 0;

}  // namespace pr

// Convolution forward as an implicit GEMM on the persistent kernel: A = im2col(x) by TMA
// (im2col mode), B = w_lp [F][ldw] (K = (tap, c) contiguous). out[pix][f] = act(. + bias[f]).
// Returns 0 when launched, non-zero when the geometry is not served here (caller falls back).
int launch_conv_fprop_pair(const void* x, const void* w_lp, long long ldw, const float* bias, void* out,
                           int N, int H, int W, int C, int OH, int OW, int F, int KY, int KX, int SY,
                           int SX, int PT, int PL, int act, cudaStream_t st) {
  using namespace pr;
  if (!conv_pair_enabled()) return -8;
  const int M = N * OH * OW, K = KY * KX * C;
  if ((C % 64) || F < 128 || (F % 8) || M < 1024 || (ldw % 8)) return -6;
  if (((uintptr_t)x & 15) || ((uintptr_t)w_lp & 15) || ((uintptr_t)out & 15)) return -3;
  const int bn = (F % 256 == 0) ? 256 : 128;
  CUtensorMap ta, tb, tc;
  int r = make_map_im2col(&ta, x, N, H, W, C, -PL, -PT, (OW - 1) * SX + 1 - PL - W,
                          (OH - 1) * SY + 1 - PT - H, SX, SY);
  if (r) return r;
  r = make_map(&tb, w_lp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, F, ldw, 64, bn);
  if (r) return r;
  r = make_map(&tc, out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, F, M, F, 64, BM);
  if (r) return r;
  Params p{};
  p.M = M; p.N = F; p.K = K; p.bias = bias; p.act = act; p.alpha = 1.f;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = (F + bn - 1) / bn;
  p.g = ConvP{H, W, OH, OW, KY, KX, SY, SX, PT, PL, C};
  p.ldo = F;
  p.splits = 1; p.kb_per_split = (K + BK - 1) / BK;
  return bn == 256 ? launch<256, false, AM_IM2COL_FPROP, BM_K>(ta, tb, tc, p, st)
                   : launch<128, false, AM_IM2COL_FPROP, BM_K>(ta, tb, tc, p, st);
}

// Unit-stride conv dgrad on the same kernel: A = windows of err_out [N][OH][OW][F] for the flipped
// filter (TMA im2col), B = wd_lp [(tap, f)][ldc] (N = input channels contiguous),
// err_in[ipix][c] = alpha * (.) (* f'(dmul)).
int launch_conv_dgrad_pair(const void* err_out, const void* wd_lp, long long ldc, void* err_in, int N,
                           int H, int W, int C, int OH, int OW, int F, int KY, int KX, int PT, int PL,
                           float alpha, const void* dmul, int dact, cudaStream_t st) {
  using namespace pr;
  if (!conv_pair_enabled()) return -8;
  const int M = N * H * W, K = KY * KX * F;
  if ((F % 64) || C < 128 || (C % 8) || M < 1024 || (ldc % 8)) return -6;
  if (((uintptr_t)err_out & 15) || ((uintptr_t)wd_lp & 15) || ((uintptr_t)err_in & 15)) return -3;
  const int bn = (C % 256 == 0) ? 256 : 128;
  CUtensorMap ta, tb, tc;
  const int lw = -(KX - 1 - PL), lh = -(KY - 1 - PT);
  int r = make_map_im2col(&ta, err_out, N, OH, OW, F, lw, lh, W + lw - OW, H + lh - OH, 1, 1);
  if (r) return r;
  // B stored [K][ldc]: inner dim = N (channels), boxes of 64 x 64
  r = make_map(&tb, wd_lp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ldc, K, ldc, 64, 64);
  if (r) return r;
  r = make_map(&tc, err_in, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, C, M, C, 64, BM);
  if (r) return r;
  Params p{};
  p.M = M; p.N = C; p.K = K; p.bias = nullptr; p.act = 0; p.alpha = alpha;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = (C + bn - 1) / bn;
  p.g = ConvP{H, W, OH, OW, KY, KX, 1, 1, PT, PL, F};
  p.dmul = (const __nv_bfloat16*)dmul; p.dact = dmul ? dact : 0; p.ldo = C;
  p.splits = 1; p.kb_per_split = (K + BK - 1) / BK;
  return bn == 256 ? launch<256, false, AM_IM2COL_DGRAD, BM_MN>(ta, tb, tc, p, st)
                   : launch<128, false, AM_IM2COL_DGRAD, BM_MN>(ta, tb, tc, p, st);
}

bool conv_pair_on() { return pr::conv_pair_enabled(); }

// Conv weight gradient on the persistent kernel: partials[s][f][kidx] (fp32) = sum over the pixels of
// split s of err_out[pix][f] * im2col(x)[pix][kidx]. A = err_out^T (stored [pix][F]: MN-major),
// B = im2col(x) as MN-major [64 pixels][64 channels] boxes (TMA im2col); the output is already in
// the weights' [F][Kw] layout - no transposed store. F % 128 == 0, C % 64 == 0.
int launch_conv_wgrad_pair(const void* err_out, const void* x, float* partials, int splits, int N, int H,
                           int W, int C, int OH, int OW, int F, int KY, int KX, int SY, int SX, int PT,
                           int PL, cudaStream_t st) {
  using namespace pr;
  if (!conv_pair_enabled()) return -8;
  const int Kw = KY * KX * C, P = N * OH * OW;
  if ((C % 64) || (F % 128) || F < 128 || Kw < 128 || P < 4096) return -6;
  if (((uintptr_t)err_out & 15) || ((uintptr_t)x & 15) || ((uintptr_t)partials & 15)) return -3;
  const int bn = Kw >= 256 ? 256 : 128;
  const int total_kb = (P + BK - 1) / BK;
  if (splits < 1) splits = 1;
  const int kbs = (total_kb + splits - 1) / splits;
  if ((long long)(splits - 1) * kbs >= total_kb) return -6;      // an empty split: not here
  CUtensorMap ta, tb, tc;
  int r = make_map(&ta, err_out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, F, P, F, 64, 64);
  if (r) return r;
  r = make_map_im2col(&tb, x, N, H, W, C, -PL, -PT, (OW - 1) * SX + 1 - PL - W,
                      (OH - 1) * SY + 1 - PT - H, SX, SY, 64);
  if (r) return r;
  r = make_map(&tc, partials, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, Kw, (long long)splits * F, Kw, 32, BM);
  if (r) return r;
  Params p{};
  p.M = F; p.N = Kw; p.K = P; p.bias = nullptr; p.act = 0; p.alpha = 1.f;
  p.tiles_m = (F + BM - 1) / BM;
  p.tiles_n = (Kw + bn - 1) / bn;
  p.splits = splits; p.kb_per_split = kbs;
  p.g = ConvP{H, W, OH, OW, KY, KX, SY, SX, PT, PL, C};
  p.ldo = Kw;
  return bn == 256 ? launch<256, true, AM_DENSE_MN, BM_IM2COL_MN>(ta, tb, tc, p, st)
                   : launch<128, true, AM_DENSE_MN, BM_IM2COL_MN>(ta, tb, tc, p, st);
}
// splits that give the CTAs of the persistent kernel ~1 work item each (0: shape not served)
int pair_wgrad_splits(int Kw, int F, int P, int max_splits) {
  using namespace pr;
  if (!conv_pair_enabled() || (Kw % 64) || (F % 128) || F < 128 || Kw < 128 || P < 4096) return 0;
  const int bn = Kw >= 256 ? 256 : 128;
  const long long tiles = (long long)((F + BM - 1) / BM) * ((Kw + bn - 1) / bn);
  int s = (int)((num_sms() + tiles - 1) / tiles);
  const int total_kb = (P + BK - 1) / BK;
  if (s > total_kb / 8) s = total_kb / 8;
  if (s > max_splits) s = max_splits;
  return s < 1 ? 1 : s;
}

// Fully-connected weight gradient: out[n_out][n_in] (fp32) = err^T . x with err stored
// [batch][n_out] and x stored [batch][n_in] (both MN-major operands, K = batch).
int launch_fc_wgrad_pair(const void* err, long long lde, const void* x, long long ldx, float* out,
                         long long ldo, int n_out, int n_in, int batch, cudaStream_t st) {
  using namespace pr;
  if (!conv_pair_enabled()) return -8;
  if (n_out < 256 || n_in < 256 || (lde % 8) || (ldx % 8) || (ldo % 4) || batch < 64) return -6;
  if (((uintptr_t)err & 15) || ((uintptr_t)x & 15) || ((uintptr_t)out & 15)) return -3;
  const int bn = 256;
  CUtensorMap ta, tb, tc;
  int r = make_map(&ta, err, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, n_out, batch, lde, 64, 64);
  if (r) return r;
  r = make_map(&tb, x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, n_in, batch, ldx, 64, 64);
  if (r) return r;
  r = make_map(&tc, out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, n_in, n_out, ldo, 32, BM);
  if (r) return r;
  Params p{};
  p.M = n_out; p.N = n_in; p.K = batch; p.alpha = 1.f;
  p.tiles_m = (n_out + BM - 1) / BM;
  p.tiles_n = (n_in + bn - 1) / bn;
  p.splits = 1; p.kb_per_split = (batch + BK - 1) / BK;
  p.ldo = ldo;
  return launch<256, true, AM_DENSE_MN, BM_MN>(ta, tb, tc, p, st);
}

// a [M][lda] bf16, b [N][ldb] bf16 (both K contiguous), out [M][ldo] bf16 or fp32.
// Returns 0, or non-zero when the shape / alignment is not served by this kernel (nothing launched).
int launch_gemm_pair(const void* a, long long lda, const void* b, long long ldb, void* out, int out_f32,
                     long long ldo, int M, int N, int K, const float* bias, int act, float alpha,
                     cudaStream_t st) {
  using namespace pr;
  const int esz = out_f32 ? 4 : 2;
  if ((lda % 8) || (ldb % 8) || ((uintptr_t)a & 15) || ((uintptr_t)b & 15)) return -3;
  if (((ldo * esz) % 16) || ((uintptr_t)out & 15)) return -3;
  if (M < 256 || N < 128 || K < 64) return -6;                // skinny / tiny: gemm_umma.cu
  const int bn = (N % 256 == 0 || N >= 1024) ? 256 : 128;
  CUtensorMap ta, tb, tc;
  int r = make_map(&ta, a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, M, lda, 64, BM);
  if (r) return r;
  r = make_map(&tb, b, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, K, N, ldb, 64, bn);
  if (r) return r;
  r = make_map(&tc, out, out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, esz,
               N, M, ldo, out_f32 ? 32 : 64, BM);
  if (r) return r;
  Params p{};
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.act = act; p.alpha = alpha;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = (N + bn - 1) / bn;
  p.splits = 1; p.kb_per_split = (K + BK - 1) / BK;
  if (bn == 256) return out_f32 ? launch<256, true>(ta, tb, tc, p, st) : launch<256, false>(ta, tb, tc, p, st);
  return out_f32 ? launch<128, true>(ta, tb, tc, p, st) : launch<128, false>(ta, tb, tc, p, st);
}

// Block-scaled fp8 GEMM (AM_FP8 mode): out[M][ldo] (bf16 or fp32) = act(alpha * A . B^T + bias),
// a [M][lda] and b [N][ldb] e4m3 codes (K contiguous), sa [ceil(K / 128)][round_up(M, 128)] and
// sb [ceil(K / 128)][round_up(N, 128)] their fp32 scales. Any M, N, K >= 1. Returns 0, or non-zero
// when the shape / alignment is refused (nothing launched).
int launch_gemm_fp8_block(const void* a, long long lda, const float* sa, const void* b, long long ldb,
                          const float* sb, void* out, int out_f32, long long ldo, int M, int N, int K,
                          const float* bias, int act, float alpha, cudaStream_t st) {
  using namespace pr;
  const int esz = out_f32 ? 4 : 2;
  if (M < 1 || N < 1 || K < 1 || lda < K || ldb < K || ldo < N) return -6;
  if ((lda % 16) || (ldb % 16) || ((uintptr_t)a & 15) || ((uintptr_t)b & 15)) return -3;
  if (((uintptr_t)sa & 15) || ((uintptr_t)sb & 15) || !sa || !sb) return -3;
  if (((ldo * esz) % 16) || ((uintptr_t)out & 15)) return -3;
  constexpr int bn = 128;
  CUtensorMap ta, tb, tc;
  int r = make_map(&ta, a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, K, M, lda, 128, BM);
  if (r) return r;
  r = make_map(&tb, b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, K, N, ldb, 128, bn);
  if (r) return r;
  r = make_map(&tc, out, out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, esz,
               N, M, ldo, out_f32 ? 32 : 64, BM);
  if (r) return r;
  Params p{};
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.act = act; p.alpha = alpha;
  p.tiles_m = (M + BM - 1) / BM;
  p.tiles_n = (N + bn - 1) / bn;
  p.splits = 1; p.kb_per_split = (K + 127) / 128;
  p.ldo = ldo;
  p.sa = sa; p.sb = sb;
  p.sa_pitch = p.tiles_m * BM; p.sb_pitch = p.tiles_n * bn;
  r = out_f32 ? launch<128, true, AM_FP8, BM_K>(ta, tb, tc, p, st)
              : launch<128, false, AM_FP8, BM_K>(ta, tb, tc, p, st);
  if (r == 0) ++g_fp8_launches;
  return r;
}
long long fp8_gemm_launches() { return pr::g_fp8_launches; }

}  // namespace zn
