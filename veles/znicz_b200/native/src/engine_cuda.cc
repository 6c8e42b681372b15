// sm_90a executor of the native runtime: launches the training engine's own kernels through
// their C++ launchers - no libtorch, no cuBLAS. Weights are uploaded once and stay resident in HBM.
// FC and conv layers run on the wgmma tensor cores with fp32-class accuracy: weights are split
// ONCE at load time into bf16 hi/lo parts laid side by side along the reduction dimension, the
// activations per call (csrc/split.cu), one bf16 wgmma GEMM / implicit-GEMM conv
// (csrc/gemm_umma.cu) accumulates hi.hi + hi.lo + lo.hi (+ lo.lo) in fp32 - the scheme of
// kernels/fp32x.py. The LSTM runs one such GEMM per time step over a [B][T][3 K8] operand whose
// h columns the cell kernel (csrc/elementwise.cu lstm_cell_split_k) fills with the split h_t for
// step t + 1 - two launches per step. ZNICZ_NATIVE_TC=0 (or a shape the kernels decline) keeps the
// SIMT fp32 kernels (csrc/gemm_simt.cu); pooling / LRN / activations / softmax are the training
// kernels as well.
#include "znicz_native.h"

#include <cuda_runtime.h>
#include <cuda_bf16.h>

#include <cstdlib>

#include <stdexcept>
#include <string>

namespace zn {
void launch_gemm_simt(const void*, bool, long long, int, const void*, bool, long long, int, void*, bool,
                      long long, int, int, int, int, const float*, int, float, float, int, long long,
                      cudaStream_t);
void launch_conv_fprop_simt_raw(const void*, bool, const float*, long long, int, const float*, void*, bool,
                                const int*, int, cudaStream_t);
void launch_pool_forward(const void*, void*, int*, int, int, int, int, int, int, int, int, int, int, int,
                         const int*, bool, int, cudaStream_t);
void launch_lrn_forward(const void*, void*, long long, int, int, float, float, float, bool, cudaStream_t);
void launch_act_forward(const void*, void*, long long, int, float, bool, cudaStream_t);
void launch_softmax_rows(const void*, bool, float*, int*, int, int, cudaStream_t);
void launch_crop_nhwc(const void*, void*, int, int, int, int, int, int, int, int, int, bool, cudaStream_t);
int launch_gemm_umma(const void*, long long, int, const void*, long long, int, void*, int, long long, int, int, int,
                     int, const float*, int, float, float, int, long long, cudaStream_t);
int launch_conv_fprop_umma(const void*, const void*, long long, const float*, void*, int, int, int, int, int, int,
                           int, int, int, int, int, int, int, int, int, cudaStream_t);
void launch_split_parts(const float*, long long, int, __nv_bfloat16*, long long, long long, int, int, int,
                        __nv_bfloat16*, long long, long long, int, int, int, cudaStream_t);
void launch_lstm_cell_fwd(const float*, const float*, float*, float*, void*, long long, void*, long long, int, int,
                          bool, cudaStream_t);
void launch_lstm_cell_split(const float*, const float*, float*, float*, long long, __nv_bfloat16*, long long, int,
                            int, int, cudaStream_t);
}  // namespace zn

namespace znicz {

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw std::runtime_error(std::string("CUDA: ") + cudaGetErrorString(e_)); } while (0)

struct Engine::CudaState {
  std::vector<float*> w, b;
  std::vector<__nv_bfloat16*> wsplit;     // hi/lo parts of the weights (null: SIMT path for that unit)
  std::vector<int> part;                  // padded per-part reduction length (FC: K8, conv: channels per part)
  float* buf[2] = {nullptr, nullptr};
  int* ibuf = nullptr;
  __nv_bfloat16* xsplit = nullptr;        // hi/lo parts of the current activations
  // LSTM step state, carved from one allocation: gate pre-activations Z [B][4H], the ping-pong
  // cells 2 x [B][H], and for the SIMT form the gates [B][4H] and the fp32 operand [B][T][I + H]
  float* lstm = nullptr;
  size_t cap = 0, icap = 0, xcap = 0, lcap = 0;
  long long tc_launches = 0;
  bool use_tc = true;
  cudaStream_t st = nullptr;
  ~CudaState() {
    for (auto p : w) cudaFree(p);
    for (auto p : b) cudaFree(p);
    for (auto p : wsplit) cudaFree(p);
    cudaFree(buf[0]); cudaFree(buf[1]); cudaFree(ibuf); cudaFree(xsplit); cudaFree(lstm);
    if (st) cudaStreamDestroy(st);
  }
};

static int round_up(int v, int a) { return (v + a - 1) / a * a; }
// channels per hi/lo part of a conv operand: 4 parts per pixel must give the implicit-GEMM gather
// 32 / 64 channels per tap or a multiple of 64
static int conv_part(int c) { return c <= 8 ? 8 : round_up(c, 16); }
// time steps of an LSTM unit's input (out_shape has checked that I divides the sample size)
static int lstm_steps(const UnitSpec& u, const Shape4& s) {
  return (int)((int64_t)s.h * s.w * s.c / (u.weights.shape[1] - u.hidden));
}
// CudaState::lstm for one unit, offsets in floats, each part 256-byte aligned: [0] Z [B][4H],
// [1] [2] cells [B][H], [3] gates [B][4H], [4] SIMT operand [B][T][I + H]; [5] = total
static void lstm_carve(int B, int T, int I, int H, size_t off[6]) {
  const size_t len[5] = {(size_t)B * 4 * H, (size_t)B * H, (size_t)B * H, (size_t)B * 4 * H,
                         (size_t)B * T * (I + H)};
  off[0] = 0;
  for (int p = 0; p < 5; ++p) off[p + 1] = off[p] + (len[p] + 63) / 64 * 64;
}

long long Engine::cuda_tensor_core_launches() const { return cuda_ ? cuda_->tc_launches : 0; }

bool Engine::cuda_available() {
  int n = 0;
  return cudaGetDeviceCount(&n) == cudaSuccess && n > 0;
}

std::vector<float> Engine::run_cuda(const float* input, const Shape4& in) {
  if (!cuda_available()) throw std::runtime_error("no CUDA device available");
  if (!cuda_) {
    cuda_.reset(new CudaState());
    CK(cudaStreamCreate(&cuda_->st));
    for (auto& u : units_) {
      float *w = nullptr, *b = nullptr;
      if (!u.weights.data.empty()) { CK(cudaMalloc(&w, u.weights.data.size() * 4)); CK(cudaMemcpy(w, u.weights.data.data(), u.weights.data.size() * 4, cudaMemcpyHostToDevice)); }
      if (u.include_bias && !u.bias.data.empty()) { CK(cudaMalloc(&b, u.bias.data.size() * 4)); CK(cudaMemcpy(b, u.bias.data.data(), u.bias.data.size() * 4, cudaMemcpyHostToDevice)); }
      cuda_->w.push_back(w); cuda_->b.push_back(b);
      // split weights for the tensor-core path: FC and LSTM [N][3 K8], conv [F][taps][4 Cp], B-side pattern
      __nv_bfloat16* ws = nullptr; int part = 0;
      const char* env = std::getenv("ZNICZ_NATIVE_TC");
      cuda_->use_tc = !(env && std::atoi(env) == 0);
      if (cuda_->use_tc && w != nullptr && u.weights.shape.size() == 2) {
        const int rows = (int)u.weights.shape[0], cols = (int)u.weights.shape[1];
        if ((u.kind == "all2all" || u.kind == "lstm") && cols >= 32) {
          part = round_up(cols, 8);
          CK(cudaMalloc(&ws, (size_t)rows * 3 * part * 2));
          zn::launch_split_parts(w, rows, cols, ws, 3LL * part, part, part, 3, 1, nullptr, 0, 0, 0, 0, 0, cuda_->st);
        } else if (u.kind == "conv" && u.ky > 0 && u.kx > 0 && cols % (u.ky * u.kx) == 0) {
          const int taps = u.ky * u.kx, c = cols / taps;
          part = conv_part(c);
          CK(cudaMalloc(&ws, (size_t)rows * taps * 4 * part * 2));
          zn::launch_split_parts(w, (long long)rows * taps, c, ws, 4LL * part, part, part, 4, 1, nullptr, 0, 0, 0, 0, 0,
                                 cuda_->st);
        }
        CK(cudaGetLastError());
      }
      cuda_->wsplit.push_back(ws); cuda_->part.push_back(part);
    }
    CK(cudaStreamSynchronize(cuda_->st));
  }
  // size the ping-pong activation buffers
  size_t need = (size_t)in.size(); Shape4 s = in; size_t ineed = 0;
  for (auto& u : units_) { s = out_shape(u, s); need = std::max(need, (size_t)s.size()); if (u.kind == "pool" && u.pool_mode != 2) ineed = std::max(ineed, (size_t)s.size()); if (u.softmax) ineed = std::max(ineed, (size_t)s.n); }
  if (need > cuda_->cap) { cudaFree(cuda_->buf[0]); cudaFree(cuda_->buf[1]); CK(cudaMalloc(&cuda_->buf[0], need * 4)); CK(cudaMalloc(&cuda_->buf[1], need * 4)); cuda_->cap = need; }
  if (ineed > cuda_->icap) { cudaFree(cuda_->ibuf); CK(cudaMalloc(&cuda_->ibuf, ineed * 4)); cuda_->icap = ineed; }
  {   // scratch for the split activations of the widest tensor-core layer, and the LSTM step state
    size_t xneed = 0, lneed = 0; Shape4 t = in;
    for (size_t i = 0; i < units_.size(); ++i) {
      auto& u = units_[i];
      if (u.kind == "lstm") {
        size_t off[6];
        lstm_carve(t.n, lstm_steps(u, t), (int)u.weights.shape[1] - u.hidden, u.hidden, off);
        lneed = std::max(lneed, off[5]);
      }
      if (cuda_->wsplit[i]) {
        if (u.kind == "all2all") xneed = std::max(xneed, (size_t)t.n * 3 * cuda_->part[i]);
        else if (u.kind == "lstm") xneed = std::max(xneed, (size_t)t.n * lstm_steps(u, t) * 3 * cuda_->part[i]);
        else xneed = std::max(xneed, (size_t)t.n * t.h * t.w * 4 * cuda_->part[i]);
      }
      t = out_shape(u, t);
    }
    if (xneed > cuda_->xcap) { cudaFree(cuda_->xsplit); CK(cudaMalloc(&cuda_->xsplit, xneed * 2)); cuda_->xcap = xneed; }
    if (lneed > cuda_->lcap) { cudaFree(cuda_->lstm); CK(cudaMalloc(&cuda_->lstm, lneed * 4)); cuda_->lcap = lneed; }
  }
  cudaStream_t st = cuda_->st;
  CK(cudaMemcpyAsync(cuda_->buf[0], input, (size_t)in.size() * 4, cudaMemcpyHostToDevice, st));
  int cur = 0; s = in;
  for (size_t i = 0; i < units_.size(); ++i) {
    auto& u = units_[i];
    Shape4 o = out_shape(u, s);
    float* x = cuda_->buf[cur]; float* y = cuda_->buf[cur ^ 1];
    if (u.kind == "all2all") {
      int K = (int)u.weights.shape[1], N = o.c;
      int r = -1;
      if (cuda_->wsplit[i]) {
        const int k8 = cuda_->part[i];
        zn::launch_split_parts(x, s.n, K, cuda_->xsplit, 3LL * k8, k8, k8, 3, 0, nullptr, 0, 0, 0, 0, 0, st);
        r = zn::launch_gemm_umma(cuda_->xsplit, 3LL * k8, 0, cuda_->wsplit[i], 3LL * k8, 0, y, 0, N, 0, s.n, N,
                                 3 * k8, cuda_->b[i], u.softmax ? 0 : (int)u.act, 1.f, 0.f, 1, 0, st);
        if (r == 0) ++cuda_->tc_launches;
      }
      if (r != 0)
        zn::launch_gemm_simt(x, false, K, 0, cuda_->w[i], false, K, 1, y, false, N, 0, s.n, N, K, cuda_->b[i],
                             u.softmax ? 0 : (int)u.act, 1.f, 0.f, 1, 0, st);
      if (u.softmax) { zn::launch_softmax_rows(y, false, x, cuda_->ibuf, s.n, N, st); std::swap(x, y); cur ^= 1; }
    } else if (u.kind == "conv") {
      int g[13] = {s.n, s.h, s.w, s.c, o.h, o.w, o.c, u.ky, u.kx, u.sy, u.sx, u.pad[1], u.pad[0]};
      int r = -1;
      if (cuda_->wsplit[i]) {
        const int cp = cuda_->part[i];
        zn::launch_split_parts(x, (long long)s.n * s.h * s.w, s.c, cuda_->xsplit, 4LL * cp, cp, cp, 4, 0, nullptr, 0, 0,
                               0, 0, 0, st);
        r = zn::launch_conv_fprop_umma(cuda_->xsplit, cuda_->wsplit[i], (long long)u.ky * u.kx * 4 * cp, cuda_->b[i], y,
                                       0, s.n, s.h, s.w, 4 * cp, o.h, o.w, o.c, u.ky, u.kx, u.sy, u.sx, u.pad[1],
                                       u.pad[0], (int)u.act, st);
        if (r == 0) ++cuda_->tc_launches;
      }
      if (r != 0)
        zn::launch_conv_fprop_simt_raw(x, false, cuda_->w[i], u.weights.shape[1], 0, cuda_->b[i], y, false, g, (int)u.act, st);
    } else if (u.kind == "pool") {
      zn::launch_pool_forward(x, y, cuda_->ibuf, s.n, s.h, s.w, s.c, o.h, o.w, u.ky, u.kx, u.sy, u.sx, u.pool_mode, nullptr, false, 0, st);
    } else if (u.kind == "lrn") {
      zn::launch_lrn_forward(x, y, s.size() / s.c, s.c, u.n, u.alpha, u.beta, u.k, false, st);
    } else if (u.kind == "act") {
      zn::launch_act_forward(x, y, s.size(), u.act_code, u.factor, false, st);
    } else if (u.kind == "lstm") {
      const int H = u.hidden, K = (int)u.weights.shape[1], I = K - H, B = s.n, T = lstm_steps(u, s);
      const bool seq = u.return_sequences;
      size_t off[6];
      lstm_carve(B, T, I, H, off);
      float* z = cuda_->lstm + off[0];
      float* cell[2] = {cuda_->lstm + off[1], cuda_->lstm + off[2]};
      // h_t goes to y[b][t] with return_sequences, otherwise to y[b] at the last step
      auto h_out = [&](int t) -> float* { return seq ? y + (size_t)t * H : (t == T - 1 ? y : nullptr); };
      const long long ldh = seq ? (long long)T * H : H;
      int r = -1;
      if (cuda_->wsplit[i]) {
        // [B][T][3 K8] operand [x_t | h_{t-1}] in the A-side parts [hi | hi | lo]; zero: h_{-1} and the padding
        const int k8 = cuda_->part[i];
        const long long ld = (long long)T * 3 * k8;
        __nv_bfloat16* xh = cuda_->xsplit;
        CK(cudaMemsetAsync(xh, 0, (size_t)B * ld * 2, st));
        zn::launch_split_parts(x, (long long)B * T, I, xh, 3LL * k8, k8, I, 3, 0, nullptr, 0, 0, 0, 0, 0, st);
        for (int t = 0; t < T; ++t) {
          r = zn::launch_gemm_umma(xh + (size_t)t * 3 * k8, ld, 0, cuda_->wsplit[i], 3LL * k8, 0, z, 0, 4 * H, 0, B,
                                   4 * H, 3 * k8, cuda_->b[i], 0, 1.f, 0.f, 1, 0, st);
          if (r != 0 && t == 0) break;     // declined shape: the whole sequence takes the SIMT form
          if (r != 0) throw std::runtime_error(u.cls + ": tensor-core GEMM failed at step " + std::to_string(t));
          ++cuda_->tc_launches;
          zn::launch_lstm_cell_split(z, t ? cell[(t - 1) & 1] : nullptr, cell[t & 1], h_out(t), ldh,
                                     t + 1 < T ? xh + (size_t)(t + 1) * 3 * k8 + I : nullptr, ld, k8, B, H, st);
        }
      }
      if (r != 0) {
        float* gates = cuda_->lstm + off[3];
        float* xhf = cuda_->lstm + off[4];
        const long long ld = (long long)T * K;
        CK(cudaMemsetAsync(xhf, 0, (size_t)B * ld * 4, st));
        CK(cudaMemcpy2DAsync(xhf, (size_t)K * 4, x, (size_t)I * 4, (size_t)I * 4, (size_t)B * T,
                             cudaMemcpyDeviceToDevice, st));
        for (int t = 0; t < T; ++t) {
          zn::launch_gemm_simt(xhf + (size_t)t * K, false, ld, 0, cuda_->w[i], false, K, 1, z, false, 4 * H, 0, B, 4 * H,
                               K, cuda_->b[i], 0, 1.f, 0.f, 1, 0, st);
          zn::launch_lstm_cell_fwd(z, t ? cell[(t - 1) & 1] : nullptr, cell[t & 1], gates, seq ? y + (size_t)t * H : y,
                                   ldh, t + 1 < T ? xhf + (size_t)(t + 1) * K + I : nullptr, ld, B, H, false, st);
        }
      }
    } else if (u.kind == "cutter") {
      zn::launch_crop_nhwc(x, y, s.n, s.h, s.w, s.c, o.h, o.w, u.pad[1], u.pad[0], 0, false, st);
    } else {
      CK(cudaMemcpyAsync(y, x, (size_t)s.size() * 4, cudaMemcpyDeviceToDevice, st));
    }
    CK(cudaGetLastError());
    cur ^= 1; s = o;
  }
  std::vector<float> out((size_t)s.size());
  CK(cudaMemcpyAsync(out.data(), cuda_->buf[cur], out.size() * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return out;
}

}  // namespace znicz
