// Restricted Boltzmann machine kernels (ops/rbm_units.py). The batch statistics run on the GEMM
// and column-sum kernels; only the two steps no existing kernel does are here.
//
// rbm_sample_k: Bernoulli draw of the Gibbs chain. For flat index i of the first batch_size rows
//   out[i] = u < p ? 1 : 0,   u = (hash_u32(seed, counter, i) >> 8) * 2^-24,   p = in[i] as fp32
// (u takes the 2^24 values k / 2^24, so p = 0 never fires and p = 1 always does); rows past the
// batch copy the input, as Binarization.numpy_run does. (seed, counter) are read from the device
// like dropout's, so a captured graph replays with the values uploaded before each replay.
//
// rbm_apply_k: the CD-k update in one launch,
//   W[h][v] += lr * G[v][h],   hbias += lr * hbias_grad,   vbias += lr * vbias_grad,
// fp32 master weights. G is transposed through a 32 x 33 shared tile so that the read of G and
// the read-modify-write of W are both row-contiguous across a warp.
#include "common.cuh"

namespace zn {

template <typename T>
__global__ void __launch_bounds__(256) rbm_sample_k(const T* __restrict__ in, T* __restrict__ out,
                                                    long long n_sampled, long long n,
                                                    const int* __restrict__ rng) {
  pdl_entry();
  const uint32_t seed = (uint32_t)rng[0], counter = (uint32_t)rng[1];
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const float p = ldf(in + i);
    if (i < n_sampled) {
      const float u = (float)(hash_u32(seed, counter, (uint64_t)i) >> 8) * 5.9604644775390625e-8f;
      stf(out + i, u < p ? 1.f : 0.f);
    } else {
      stf(out + i, p);
    }
  }
}

constexpr int RBM_TILE = 32;

// blocks [0, tiles): one 32 x 32 tile of W each (block 32 x 8, 4 rows per thread);
// every block then takes a grid-stride share of the H + V bias elements
__global__ void __launch_bounds__(256) rbm_apply_k(float* __restrict__ w, const float* __restrict__ g,
                                                   float* __restrict__ hbias, const float* __restrict__ hgrad,
                                                   float* __restrict__ vbias, const float* __restrict__ vgrad,
                                                   int H, int V, int tiles_v, int tiles, float lr) {
  pdl_entry();
  __shared__ float tile[RBM_TILE][RBM_TILE + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;
  if ((int)blockIdx.x < tiles) {
    const int v0 = (blockIdx.x % tiles_v) * RBM_TILE, h0 = (blockIdx.x / tiles_v) * RBM_TILE;
    // G[v][h]: warp reads 32 consecutive h of one v
#pragma unroll
    for (int k = 0; k < RBM_TILE; k += 8) {
      const int v = v0 + ty + k, h = h0 + tx;
      tile[ty + k][tx] = (v < V && h < H) ? g[(size_t)v * H + h] : 0.f;
    }
    __syncthreads();
    // W[h][v]: warp updates 32 consecutive v of one h
#pragma unroll
    for (int k = 0; k < RBM_TILE; k += 8) {
      const int h = h0 + ty + k, v = v0 + tx;
      if (h < H && v < V) {
        float* p = w + (size_t)h * V + v;
        *p += lr * tile[tx][ty + k];
      }
    }
  }
  const int tid = ty * RBM_TILE + tx;
  for (int j = blockIdx.x * 256 + tid; j < H + V; j += gridDim.x * 256) {
    if (j < H) hbias[j] += lr * hgrad[j];
    else vbias[j - H] += lr * vgrad[j - H];
  }
}

void launch_rbm_sample(const void* in, void* out, long long n_sampled, long long n, const int* rng, bool bf16,
                       cudaStream_t st) {
  long long b = (n + 255) / 256;
  const long long cap = 16LL * num_sms();
  const int grid = (int)(b < 1 ? 1 : (b > cap ? cap : b));
  if (bf16)
    launch_k(rbm_sample_k<__nv_bfloat16>, grid, 256, 0, st, (const __nv_bfloat16*)in, (__nv_bfloat16*)out,
             n_sampled, n, rng);
  else
    launch_k(rbm_sample_k<float>, grid, 256, 0, st, (const float*)in, (float*)out, n_sampled, n, rng);
}

void launch_rbm_apply(float* w, const float* g, float* hbias, const float* hgrad, float* vbias,
                      const float* vgrad, int H, int V, float lr, cudaStream_t st) {
  const int tiles_v = (V + RBM_TILE - 1) / RBM_TILE;
  const int tiles = tiles_v * ((H + RBM_TILE - 1) / RBM_TILE);
  const int grid = tiles > 0 ? tiles : 1;
  launch_k(rbm_apply_k, grid, dim3(RBM_TILE, 8), 0, st, w, g, hbias, hgrad, vbias, vgrad, H, V, tiles_v,
           tiles, lr);
}

}  // namespace zn
