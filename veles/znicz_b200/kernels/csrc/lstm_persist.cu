// Persistent LSTM sequence kernels (sm_90a): the whole time loop of an LSTM layer in ONE launch.
//
//   forward   z_t = [x_t | h_{t-1}] . W^T + b,  (i, f, g, o) = act(z_t),  c_t = i g + f c_{t-1},
//             h_t = o * A tanh(B c_t)                         (/root/reference/lstm.py:75-143)
//   backward  dh_t = err_t + dz_{t+1} . W_h,  cell derivative -> dz_t,  dc_{t-1} = dc_t f
//
// The per-time-step path is 2-3 launches per step (gemm + cell kernel, ~4 us each: the recurrence
// is latency bound). Here a CLUSTER of H / 32 CTAs owns R batch rows (R = 32 / 64 / 128, chosen so
// that the clusters spread over the SMs) for all T steps:
//
// forward
// * CTA c owns hidden units [32 c, 32 c + 32): the 4 x 32 rows of W of their gates stay RESIDENT
//   in shared memory for the whole sequence (96 KB at I = 128, H = 256), loaded once by TMA;
// * per step one wgmma accumulation D[R x 128] in registers (two MMA warpgroups of 64 rows): the
//   x part (K = I, no recurrence) is issued first and runs while the h part (K = H) waits for
//   h_{t-1};
// * the cell math runs straight on the accumulator fragment: the 4 gate columns of a unit sit in
//   the same thread (thread = 2 batch rows x 8 units), c_t lives in registers across the steps;
// * the cluster exchanges h_t through L2: bf16 stores into the [x | h] operand of step t + 1 ->
//   fence.proxy.async -> barrier.cluster (release / acquire) -> TMA loads.
// * critical path first: h is stored and announced BEFORE the state for the backward pass is
//   written; that state (gates as bf16, c as fp32) uses a lane-major private layout in which every
//   warp-wide store is one contiguous 512-byte piece.
// backward
// * dz_t of the CTA's own units goes from the epilogue straight into its own A operand (swizzled
//   smem) and is multiplied by the resident W_h rows of those gates: P_c[R x H] = dz_t[:, own] .
//   W_h[own, :] (K = 128, N = H, one accumulation per step);
// * the partial sums are reduce-scattered through L2 as bf16 (the owner of a unit has the same
//   fragment rows as every producer of it: 32 contiguous bytes per thread and owner) under
//   barrier.cluster; CTA d adds the H / 32 pieces of its units in fp32 -> dh_{t-1}; dc lives in
//   registers.
// Launch-count: 2 (+ the W_h^T permutation) instead of ~5 T.
#include "common.cuh"
#include "umma.cuh"

namespace zn {

using namespace umma;

namespace lp {

constexpr int BM = 128;
constexpr int U = 32;                   // hidden units per CTA
constexpr int NG = 4 * U;               // gate columns per CTA
constexpr int THREADS = 384;            // warpgroup 0 TMA, warpgroups 1, 2 MMA + cell math
constexpr int SVEC = 12;                // 16-byte vectors per thread and step in the private state layout

__device__ __forceinline__ uint32_t cl_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cl_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cl_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
// generic-proxy global stores of this thread become visible to later async-proxy (TMA) reads
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigm_fast(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
__device__ __forceinline__ uint4 pack8(const float* v) {
  return make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}
__device__ __forceinline__ void unpack8(uint4 u, float* v) {
  v[0] = bf_lo(u.x); v[1] = bf_hi(u.x); v[2] = bf_lo(u.y); v[3] = bf_hi(u.y);
  v[4] = bf_lo(u.z); v[5] = bf_hi(u.z); v[6] = bf_lo(u.w); v[7] = bf_hi(u.w);
}
// byte offset of 16-byte chunk `ch` of row `r` in a [128 rows][128 B] SWIZZLE_128B K-major block
__device__ __forceinline__ uint32_t sw128(int r, int ch) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((ch ^ (r & 7)) << 4));
}

// Consumer-thread geometry shared by both kernels and the state unpacker: consumer thread
// tid = threadIdx.x - 128 (warp ew = tid / 32 of warpgroup wgc = ew / 4) owns batch rows
// rA = 64 wgc + 16 (ew % 4) + lane / 4 and rA + 8 and, of the CTA's 32 units, 8 ii + 2 (lane % 4) + e
// (ii < 4, e < 2): the wgmma accumulator fragment. Its 16 (row, unit) "slots" are numbered
// s = 4 ii + 2 h + e (h: row rA + 8 h), so gate g of slot s is accumulator register 16 g + s.
__device__ __forceinline__ int slot_row(int ew, int lane, int s) {
  return (ew >> 2) * 64 + 16 * (ew & 3) + (lane >> 2) + 8 * ((s >> 1) & 1);
}
__device__ __forceinline__ int slot_unit(int lane, int s) { return 8 * (s >> 2) + 2 * (lane & 3) + (s & 1); }

// Private state layout (forward -> backward), 16-byte vectors:
//   ((t * n_ctas + cta) * 8 + consumer warp) * SVEC + v) * 32 + lane
// v = 2 g + j: gate g (input, forget, memory maker, output) of slots 8 j .. 8 j + 7 as bf16;
// v = 8 + j: cell state of slots 4 j .. 4 j + 3 as fp32. Every warp-wide access is one contiguous
// 512-byte piece.
__device__ __forceinline__ size_t state_idx(int t, int n_ctas, int cta, int ew, int v, int lane) {
  return ((((size_t)t * n_ctas + cta) * 8 + ew) * SVEC + v) * 32 + lane;
}

struct FwdP {
  int T, B, I, H, R;          // R: batch rows per cluster
  const float* bias;          // [4H] or null
  uint4* state;               // private layout, see state_idx
  __nv_bfloat16* xh;          // [T + 1][B][I + H]
  long long* dbg;             // optional clock64 stamps [T][8] of CTA 0 (tools/lstm_probe.py)
};

__global__ void __launch_bounds__(THREADS, 1)
lstm_fwd_k(const __grid_constant__ CUtensorMap t_xh, const __grid_constant__ CUtensorMap t_w, FwdP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int KX = p.I / 64, KH = p.H / 64;
  uint8_t* sW = sm;                                   // (KX + KH) blocks x [NG rows][128 B]
  uint8_t* sX = sW + (size_t)(KX + KH) * NG * 128;    // 2 stages x KX blocks x [128 rows][128 B]
  uint8_t* sH = sX + (size_t)2 * KX * BM * 128;       // KH blocks x [128 rows][128 B]: h_{t-1}
  __shared__ __align__(8) uint64_t w_full, x_full[2], x_empty[2], h_full;
  __shared__ float s_bias[NG];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = (int)cl_rank();
  const int T = p.T, B = p.B, I = p.I, H = p.H, R = p.R;
  const int csize = H / U;
  const int row0 = (blockIdx.x / csize) * R;           // first batch row of this cluster
  const uint32_t tile_bytes = (uint32_t)(R * 128);     // one k-block of R rows
  const int nwg = R > 64 ? 2 : 1;                      // MMA warpgroups with batch rows

  if (threadIdx.x == 0) {
    mbar_init(&w_full, 1);
    mbar_init(&h_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&x_full[s], 1); mbar_init(&x_empty[s], (uint32_t)nwg); }
    fence_barrier_init();
    tma_prefetch_desc(&t_xh);
    tma_prefetch_desc(&t_w);
  }
  if (threadIdx.x < NG) {
    const int g = threadIdx.x / U, j = threadIdx.x % U;
    s_bias[threadIdx.x] = p.bias ? p.bias[g * H + c * U + j] : 0.f;
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------------------------------------------------------- producer warpgroup
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&w_full, (uint32_t)((KX + KH) * NG * 128));
      for (int kb = 0; kb < KX + KH; ++kb)
        for (int g = 0; g < 4; ++g)
          tma_load_2d(sW + (size_t)kb * NG * 128 + g * U * 128, &t_w, &w_full, kb * 64, g * H + c * U);
      for (int t0 = 0; t0 < 2 && t0 < T; ++t0) {
        mbar_arrive_expect_tx(&x_full[t0], KX * tile_bytes);
        for (int kb = 0; kb < KX; ++kb)
          tma_load_2d(sX + (size_t)(t0 * KX + kb) * BM * 128, &t_xh, &x_full[t0], kb * 64, t0 * B + row0);
      }
    }
    for (int t = 1; t < T; ++t) {
      cl_arrive(); cl_wait();                         // every CTA's slice of h_{t-1} is in xh[t]
      if (threadIdx.x == 0) {
        fence_proxy_async_all();
        mbar_arrive_expect_tx(&h_full, KH * tile_bytes);
        for (int kb = 0; kb < KH; ++kb)
          tma_load_2d(sH + (size_t)kb * BM * 128, &t_xh, &h_full, I + kb * 64, t * B + row0);
        if (t + 1 < T) {
          const int s = (t + 1) & 1;                  // stage of x_{t+1}; its previous user was x_{t-1}
          mbar_wait(&x_empty[s], (((t + 1) >> 1) - 1) & 1);
          mbar_arrive_expect_tx(&x_full[s], KX * tile_bytes);
          for (int kb = 0; kb < KX; ++kb)
            tma_load_2d(sX + (size_t)(s * KX + kb) * BM * 128, &t_xh, &x_full[s], kb * 64, (t + 1) * B + row0);
        }
      }
      __syncwarp();
    }
  } else {
    // ------------------------------------------- MMA warpgroups: z_t = [x_t | h_{t-1}] . W^T, cell math
    reg_alloc<232>();
    const int tid = threadIdx.x - 128, ew = tid >> 5, wgc = ew >> 2;
    const bool mma = wgc < nwg;                        // warpgroup-uniform
    const int n_ctas = gridDim.x;
    float cst[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) cst[j] = 0.f;
    if (mma) mbar_wait(&w_full, 0);
    for (int t = 0; t < T; ++t) {
      float gi[16], gf[16], gg[16], go[16];
      if (mma) {
        float acc[NG / 2];
        const int s = t & 1;
        mbar_wait(&x_full[s], (t >> 1) & 1);
        if (p.dbg && blockIdx.x == 0 && tid == 0) p.dbg[t * 8 + 2] = clock64();
        wg_fence();
        // x part (no recurrence), then the h part once h_{t-1} has arrived
        for (int kb = 0; kb < KX; ++kb) {
          const uint32_t sa = smem_u32(sX + (size_t)(s * KX + kb) * BM * 128) + wgc * 8192;
          const uint32_t sb = smem_u32(sW + (size_t)kb * NG * 128);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_bf16<NG, 0, 0>(acc, make_smem_desc(sa + k * 32, 16, 1024), make_smem_desc(sb + k * 32, 16, 1024),
                                 (kb > 0 || k > 0) ? 1 : 0);
        }
        wg_commit();
        if (t > 0) {
          mbar_wait(&h_full, (t - 1) & 1);
          for (int kb = 0; kb < KH; ++kb) {
            const uint32_t sa = smem_u32(sH + (size_t)kb * BM * 128) + wgc * 8192;
            const uint32_t sb = smem_u32(sW + (size_t)(KX + kb) * NG * 128);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              wgmma_bf16<NG, 0, 0>(acc, make_smem_desc(sa + k * 32, 16, 1024), make_smem_desc(sb + k * 32, 16, 1024), 1);
          }
          wg_commit();
        }
        wg_wait<0>();
        wg_fence_regs(acc);
        if ((tid & 127) == 0) mbar_arrive(&x_empty[s]);
        if (p.dbg && blockIdx.x == 0 && tid == 0) p.dbg[t * 8 + 3] = clock64();
        float hv[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int n = slot_unit(lane, j);
          gi[j] = sigm_fast(acc[j] + s_bias[n]);
          gf[j] = sigm_fast(acc[16 + j] + s_bias[U + n]);
          gg[j] = 1.7159f * tanh_fast(0.6666f * (acc[32 + j] + s_bias[2 * U + n]));
          go[j] = sigm_fast(acc[48 + j] + s_bias[3 * U + n]);
          cst[j] = fmaf(gi[j], gg[j], gf[j] * cst[j]);
          hv[j] = go[j] * (1.7159f * tanh_fast(0.6666f * cst[j]));
        }
        if (p.dbg && blockIdx.x == 0 && tid == 0) p.dbg[t * 8 + 4] = clock64();
        // critical path first: h_t into the operand of step t + 1 (also the wgrad operand)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = slot_row(ew, lane, 2 * h);
          const int b = row0 + r;
          if (r < R && b < B) {
            __nv_bfloat16* hp = p.xh + ((size_t)(t + 1) * B + b) * (I + H) + I + c * U;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) {
              const int j = 4 * ii + 2 * h;
              *reinterpret_cast<__nv_bfloat162*>(hp + slot_unit(lane, j)) = __floats2bfloat162_rn(hv[j], hv[j + 1]);
            }
          }
        }
      }
      if (t < T - 1) {
        fence_proxy_async_all();
        if (t > 0) cl_wait();                         // close phase t - 1 before arriving on phase t
        cl_arrive();
      }
      if (p.dbg && blockIdx.x == 0 && tid == 0) p.dbg[t * 8 + 5] = clock64();
      if (mma) {
        // off the critical path: state for the backward pass, one 512-byte piece per warp store
        uint4* sp = p.state + state_idx(t, n_ctas, blockIdx.x, ew, 0, lane);
        sp[0 * 32] = pack8(gi); sp[1 * 32] = pack8(gi + 8);
        sp[2 * 32] = pack8(gf); sp[3 * 32] = pack8(gf + 8);
        sp[4 * 32] = pack8(gg); sp[5 * 32] = pack8(gg + 8);
        sp[6 * 32] = pack8(go); sp[7 * 32] = pack8(go + 8);
#pragma unroll
        for (int v = 0; v < 4; ++v)
          sp[(8 + v) * 32] = make_uint4(__float_as_uint(cst[4 * v]), __float_as_uint(cst[4 * v + 1]),
                                        __float_as_uint(cst[4 * v + 2]), __float_as_uint(cst[4 * v + 3]));
      }
      if (p.dbg && blockIdx.x == 0 && tid == 0) p.dbg[t * 8 + 6] = clock64();
    }
    if (T > 1) cl_wait();
  }
}

struct BwdP {
  int T, B, H, R;
  const __nv_bfloat16* err;   // dL/dh from above: [B][T][H] (seq) or [B][H] (last step only)
  long long lde;              // row pitch of err (elements)
  int seq;
  const uint4* state;         // private layout written by lstm_fwd_k
  uint4* part;                // [2][n_ctas][H / 32 owners][256 threads][2]: bf16 partial sums
  __nv_bfloat16* dz;          // [T][B][4H]
};

template <int HN>
__global__ void __launch_bounds__(THREADS, 1)
lstm_bwd_k(const __grid_constant__ CUtensorMap t_whp, BwdP p) {
  constexpr int H = HN, CS = HN / U;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int T = p.T, B = p.B, R = p.R;
  uint8_t* sB = sm;                                   // 2 k-blocks x [H rows][128 B]: W_h rows of own gates
  uint8_t* sA = sB + (size_t)2 * H * 128;             // 2 k-blocks x [128 rows][128 B]: own dz_t
  __shared__ __align__(8) uint64_t b_full;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = (int)cl_rank();
  const int row0 = (blockIdx.x / CS) * R;
  const int n_ctas = gridDim.x;
  const size_t part_buf = (size_t)n_ctas * CS * 256 * 2;
  const int nwg = R > 64 ? 2 : 1;

  if (threadIdx.x == 0) {
    mbar_init(&b_full, 1);
    fence_barrier_init();
    tma_prefetch_desc(&t_whp);
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&b_full, (uint32_t)(2 * H * 128));
      for (int kb = 0; kb < 2; ++kb) tma_load_2d(sB + (size_t)kb * H * 128, &t_whp, &b_full, c * NG + kb * 64, 0);
    }
    for (int k = 0; k < T - 1; ++k) { cl_arrive(); cl_wait(); }
  } else {
    reg_alloc<232>();
    const int tid = threadIdx.x - 128, ew = tid >> 5, wgc = ew >> 2;
    const bool mma = wgc < nwg;
    const int cta0 = (blockIdx.x / CS) * CS;          // first CTA of this cluster
    if (mma) mbar_wait(&b_full, 0);
    float dcs[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) dcs[j] = 0.f;
    for (int s = T - 1; s >= 0; --s) {
      const int k = T - 1 - s;
      if (mma) {
        // -------- dh_s -> dz_s of the own units
        float gi[16], gf[16], gg[16], go[16], cc[16], cp[16], dh[16];
        {
          const uint4* sp = p.state + state_idx(s, n_ctas, blockIdx.x, ew, 0, lane);
          const uint4* pp = p.state + state_idx(s > 0 ? s - 1 : 0, n_ctas, blockIdx.x, ew, 8, lane);
          const uint4 a0 = sp[0], a1 = sp[32], a2 = sp[64], a3 = sp[96], a4 = sp[128], a5 = sp[160];
          const uint4 a6 = sp[192], a7 = sp[224];
          unpack8(a0, gi); unpack8(a1, gi + 8); unpack8(a2, gf); unpack8(a3, gf + 8);
          unpack8(a4, gg); unpack8(a5, gg + 8); unpack8(a6, go); unpack8(a7, go + 8);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            const uint4 cv = sp[(8 + v) * 32];
            cc[4 * v] = __uint_as_float(cv.x); cc[4 * v + 1] = __uint_as_float(cv.y);
            cc[4 * v + 2] = __uint_as_float(cv.z); cc[4 * v + 3] = __uint_as_float(cv.w);
            const uint4 pv = s > 0 ? pp[v * 32] : make_uint4(0u, 0u, 0u, 0u);
            cp[4 * v] = __uint_as_float(pv.x); cp[4 * v + 1] = __uint_as_float(pv.y);
            cp[4 * v + 2] = __uint_as_float(pv.z); cp[4 * v + 3] = __uint_as_float(pv.w);
          }
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) dh[j] = 0.f;
        if (p.seq || s == T - 1) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int b = row0 + slot_row(ew, lane, 2 * h);
            if (slot_row(ew, lane, 2 * h) < R && b < B) {
              const __nv_bfloat16* e = p.err + (size_t)b * p.lde + (p.seq ? (size_t)s * H : 0) + c * U;
#pragma unroll
              for (int ii = 0; ii < 4; ++ii) {
                const int j = 4 * ii + 2 * h;
                const __nv_bfloat162 x = *reinterpret_cast<const __nv_bfloat162*>(e + slot_unit(lane, j));
                dh[j] = __low2float(x); dh[j + 1] = __high2float(x);
              }
            }
          }
        }
        if (k > 0) {
          cl_wait();                                   // phase k - 1: every CTA's partial sums are out
          const uint4* pb = p.part + (size_t)((k - 1) & 1) * part_buf;
          for (int src = 0; src < CS; ++src) {
            const uint4* pv = pb + ((size_t)((cta0 + src) * CS + c) * 256 + tid) * 2;
            float t0[8], t1[8];
            unpack8(__ldcg(pv), t0);
            unpack8(__ldcg(pv + 1), t1);
#pragma unroll
            for (int j = 0; j < 8; ++j) { dh[j] += t0[j]; dh[8 + j] += t1[j]; }
          }
        }
        float zz[4][16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float tc = 1.7159f * tanh_fast(0.6666f * cc[j]);
          const float dtc = fmaf(tc * tc, -0.388484177f, 1.14381894f);        // d(A tanh(B c)) / dc
          const float dc = fmaf(dh[j] * go[j], dtc, dcs[j]);
          zz[0][j] = dc * gg[j] * gi[j] * (1.f - gi[j]);
          zz[1][j] = dc * cp[j] * gf[j] * (1.f - gf[j]);
          zz[2][j] = dc * gi[j] * fmaf(gg[j] * gg[j], -0.388484177f, 1.14381894f);
          zz[3][j] = dh[j] * tc * go[j] * (1.f - go[j]);
          dcs[j] = dc * gf[j];
        }
        if (s > 0) {
          // own A operand: k index = gate * 32 + local unit (the order W_h^T was permuted to)
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            uint8_t* blk = sA + (size_t)(g >> 1) * BM * 128;
#pragma unroll
            for (int j = 0; j < 16; j += 2) {
              const int r = slot_row(ew, lane, j), u = (g & 1) * 32 + slot_unit(lane, j);
              *reinterpret_cast<__nv_bfloat162*>(blk + sw128(r, u >> 3) + (u & 7) * 2) =
                  __floats2bfloat162_rn(zz[g][j], zz[g][j + 1]);
            }
          }
          fence_proxy_async_smem();
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int b = row0 + slot_row(ew, lane, 2 * h);
          if (slot_row(ew, lane, 2 * h) < R && b < B) {
            __nv_bfloat16* dr = p.dz + ((size_t)s * B + b) * 4 * H + c * U;
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int ii = 0; ii < 4; ++ii) {
                const int j = 4 * ii + 2 * h;
                *reinterpret_cast<__nv_bfloat162*>(dr + (size_t)g * H + slot_unit(lane, j)) =
                    __floats2bfloat162_rn(zz[g][j], zz[g][j + 1]);
              }
          }
        }
        if (s > 0) {
          // -------- P = dz_s[:, own] . W_h[own, :] -> bf16 pieces for the owners of its columns
          named_bar_sync(1 + wgc, 128);                // the warpgroup's rows of sA are complete
          float acc[HN / 2];
          wg_fence();
#pragma unroll
          for (int kb = 0; kb < 2; ++kb) {
            const uint32_t sa = smem_u32(sA + (size_t)kb * BM * 128) + wgc * 8192;
            const uint32_t sb = smem_u32(sB + (size_t)kb * H * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
              wgmma_bf16<HN, 0, 0>(acc, make_smem_desc(sa + kk * 32, 16, 1024), make_smem_desc(sb + kk * 32, 16, 1024),
                                   (kb > 0 || kk > 0) ? 1 : 0);
          }
          wg_commit();
          wg_wait<0>();
          wg_fence_regs(acc);
          // owner d of columns [32 d, 32 d + 32) holds the same fragment rows: registers 16 d .. 16 d + 15
          uint4* pw = p.part + (size_t)(k & 1) * part_buf + ((size_t)blockIdx.x * CS * 256 + tid) * 2;
#pragma unroll
          for (int d = 0; d < CS; ++d) {
            pw[(size_t)d * 512] = pack8(acc + 16 * d);
            pw[(size_t)d * 512 + 1] = pack8(acc + 16 * d + 8);
          }
          // sA is rewritten next step only after every thread of this warpgroup passed its MMA
          named_bar_sync(1 + wgc, 128);
        }
      } else if (k > 0) {
        cl_wait();
      }
      if (s == 0) break;
      cl_arrive();                                     // phase k: this thread's partial sums are out
    }
  }
}

// W_h^T in the k order of the backward kernel: dst[n][c * 128 + g * 32 + j] = w[g * H + c * 32 + j][col0 + n]
__global__ void permute_wh_k(const __nv_bfloat16* __restrict__ w, long long ldw, int col0, int H,
                             __nv_bfloat16* __restrict__ dst) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;          // k0: permuted k index (multiple of 32)
  const int c = k0 / NG, g = (k0 % NG) / U;
  const int row = g * H + c * U;                                  // first source row of this k run
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    tile[i][threadIdx.x] = w[(size_t)(row + i) * ldw + col0 + n0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    dst[(size_t)(n0 + i) * 4 * H + k0 + threadIdx.x] = tile[threadIdx.x][i];
}

// private state layout -> the unit's public gates [T][B][4H] / cells [T][B][H] (per-step fallback)
__global__ void lstm_unpack_state_k(const uint4* __restrict__ state, float* __restrict__ gates,
                                    float* __restrict__ cells, int T, int B, int H, int R, int n_ctas) {
  const size_t total = (size_t)T * n_ctas * 8 * SVEC * 32;
  const int csize = H / U;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int lane = (int)(i % 32);
    const int v = (int)((i / 32) % SVEC);
    const int ew = (int)((i / (32 * SVEC)) % 8);
    const int cta = (int)((i / (32 * SVEC * 8)) % n_ctas);
    const int t = (int)(i / ((size_t)32 * SVEC * 8 * n_ctas));
    const uint4 val = state[i];
    const int n = v < 8 ? 8 : 4;                      // slots in this vector
    const int s0 = v < 8 ? 8 * (v & 1) : 4 * (v - 8);
    float f[8];
    if (v < 8) {
      unpack8(val, f);
    } else {
      f[0] = __uint_as_float(val.x); f[1] = __uint_as_float(val.y);
      f[2] = __uint_as_float(val.z); f[3] = __uint_as_float(val.w);
    }
    for (int k = 0; k < n; ++k) {
      const int sl = s0 + k;
      const int r = slot_row(ew, lane, sl);
      const int b = (cta / csize) * R + r;
      if (r >= R || b >= B) continue;
      const int j = (cta % csize) * U + slot_unit(lane, sl);
      if (v < 8) gates[((size_t)t * B + b) * 4 * H + (size_t)(v >> 1) * H + j] = f[k];
      else cells[((size_t)t * B + b) * H + j] = f[k];
    }
  }
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
static int make_map(CUtensorMap* m, const void* ptr, long long inner, long long outer, long long ld, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -1;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)(ld * 2)};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

template <typename... KArgs, typename... Args>
static int launch_cluster(void (*kernel)(KArgs...), int blocks, int csize, size_t smem, cudaStream_t st,
                          Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return (int)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace lp

static long long g_lstm_persist_launches = 0;
long long lstm_persist_launches() { return g_lstm_persist_launches; }

static bool lstm_shape_ok(int T, int B, int I, int H) {
  const int cs = H / lp::U;
  return I >= 64 && I % 64 == 0 && H >= 64 && H % 64 == 0 && cs <= 8 && T >= 1 && B >= 1;
}
// batch rows per cluster: the smallest of 128 / 64 / 32 that keeps the grid within ~one wave
// (fewer rows per CTA = less epilogue math, TMA bytes and state traffic per step and SM)
int lstm_persist_rows(int B, int H) {
  const int cs = H / lp::U;
  const char* e = getenv("ZNICZ_LSTM_ROWS");
  if (e && (atoi(e) == 32 || atoi(e) == 64 || atoi(e) == 128)) return atoi(e);
  for (int r = 32; r < 128; r *= 2)
    if (((B + r - 1) / r) * cs <= 128) return r;
  return 128;
}
static int lstm_ctas(int B, int H) {
  const int R = lstm_persist_rows(B, H);
  return ((B + R - 1) / R) * (H / lp::U);
}
// 16-byte elements of the private state buffer the forward kernel needs (0: shape not supported)
long long lstm_persist_state_elems(int T, int B, int I, int H) {
  if (!lstm_shape_ok(T, B, I, H)) return 0;
  return (long long)T * lstm_ctas(B, H) * 8 * lp::SVEC * 32;
}
// 16-byte elements of the backward kernel's partial-sum exchange buffer
long long lstm_persist_part_elems(int B, int H) { return 2LL * lstm_ctas(B, H) * 8 * (H / 16) * 32; }

// 0 = launched; < 0 = shape outside the kernel's range (the caller keeps the per-step path)
int launch_lstm_fwd_persist(void* xh, const void* w_lp, long long ldw, const float* bias, void* state,
                            int T, int B, int I, int H, long long* dbg, cudaStream_t st) {
  using namespace lp;
  if (!lstm_shape_ok(T, B, I, H)) return -3;
  const int KX = I / 64, KH = H / 64;
  const size_t smem = (size_t)(KX + KH) * NG * 128 + (size_t)2 * KX * BM * 128 + (size_t)KH * BM * 128 + 1024;
  if (smem > 227 * 1024 - 2048) return -4;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(lstm_fwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 2048) != cudaSuccess)
      return -5;
    attr_set = true;
  }
  CUtensorMap t_xh, t_w;
  const int R = lstm_persist_rows(B, H);
  int r = make_map(&t_xh, xh, I + H, (long long)(T + 1) * B, I + H, R);
  if (r) return -6;
  r = make_map(&t_w, w_lp, I + H, 4LL * H, ldw, U);
  if (r) return -6;
  FwdP p{T, B, I, H, R, bias, (uint4*)state, (__nv_bfloat16*)xh, dbg};
  const int csize = H / U;
  const int clusters = (B + R - 1) / R;
  r = launch_cluster(lstm_fwd_k, clusters * csize, csize, smem, st, t_xh, t_w, p);
  if (r == 0) ++g_lstm_persist_launches;
  return r == 0 ? 0 : -7;
}

int launch_lstm_bwd_persist(const void* err, long long lde, int seq, const void* state, void* part, void* dz,
                            const void* w_lp, long long ldw, void* whp, int T, int B, int I, int H,
                            cudaStream_t st) {
  using namespace lp;
  if (!lstm_shape_ok(T, B, I, H)) return -3;
  const int csize = H / U;
  const size_t smem = (size_t)2 * H * 128 + (size_t)2 * BM * 128 + 1024;
  if (smem > 227 * 1024 - 2048) return -4;
  static bool attr_set = false;
  if (!attr_set) {
    for (auto k : {lstm_bwd_k<64>, lstm_bwd_k<128>, lstm_bwd_k<192>, lstm_bwd_k<256>})
      if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 2048) != cudaSuccess)
        return -5;
    attr_set = true;
  }
  // W_h^T [H][4H], columns permuted to (CTA, gate, unit) order, from the bf16 weight shadow
  {
    dim3 grid(H / 32, 4 * H / 32), block(32, 8);
    permute_wh_k<<<grid, block, 0, st>>>((const __nv_bfloat16*)w_lp, ldw, I, H, (__nv_bfloat16*)whp);
  }
  CUtensorMap t_whp;
  int r = make_map(&t_whp, whp, 4LL * H, H, 4LL * H, H);
  if (r) return -6;
  const int R = lstm_persist_rows(B, H);
  BwdP p{T, B, H, R, (const __nv_bfloat16*)err, lde, seq, (const uint4*)state, (uint4*)part, (__nv_bfloat16*)dz};
  const int clusters = (B + R - 1) / R;
  void (*kern)(const CUtensorMap, BwdP) = H == 64 ? lstm_bwd_k<64> : H == 128 ? lstm_bwd_k<128>
                                            : H == 192 ? lstm_bwd_k<192> : lstm_bwd_k<256>;
  r = launch_cluster(kern, clusters * csize, csize, smem, st, t_whp, p);
  if (r == 0) ++g_lstm_persist_launches;
  return r == 0 ? 0 : -7;
}

void launch_lstm_unpack_state(const void* state, float* gates, float* cells, int T, int B, int H,
                              cudaStream_t st) {
  using namespace lp;
  lstm_unpack_state_k<<<2 * num_sms(), 256, 0, st>>>((const uint4*)state, gates, cells, T, B, H, lstm_persist_rows(B, H),
                                           lstm_ctas(B, H));
}

}  // namespace zn
