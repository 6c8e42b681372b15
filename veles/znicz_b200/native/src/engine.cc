// Unit list construction + CPU executor (+ C ABI).
#include "znicz_native.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>

namespace znicz {

static const std::map<std::string, std::string>& fc_uuids() {
  // uuids of the reference's FC units (/root/reference/all2all.py:88,274,301,323,346,385)
  static const std::map<std::string, std::string> m = {
      {"58a5eadf-ae1e-498f-bf35-7d93939c4c86", "All2All"},
      {"b3a2bd5c-3c01-46ef-978a-fef22e008f31", "All2AllTanh"},
      {"5b7f36d8-f8c8-4eb7-8af3-75eb3cfca3fe", "All2AllRELU"},
      {"fe63baf0-4fe4-4cf3-bafb-ef1215bf27a8", "All2AllStrictRELU"},
      {"a27974ec-1764-4944-925d-4862de237881", "All2AllSigmoid"},
      {"420219fc-3e1a-45b1-87f8-aaa0c1540de4", "All2AllSoftmax"}};
  return m;
}

static Act act_from_mode(const std::string& m) {
  if (m == "ACTIVATION_TANH") return Act::Tanh;
  if (m == "ACTIVATION_RELU") return Act::Relu;
  if (m == "ACTIVATION_STRICT_RELU") return Act::StrictRelu;
  if (m == "ACTIVATION_SIGMOID") return Act::Sigmoid;
  return Act::Linear;
}

static std::vector<int> int_list(const Json& j) {
  std::vector<int> v;
  for (auto& e : j.arr) v.push_back((int)e.num);
  return v;
}

Engine::Engine(const std::string& path) {
  auto files = read_package_files(path);
  auto it = files.find("contents.json");
  if (it == files.end()) throw std::runtime_error("package has no contents.json");
  Json c = Json::parse(it->second);
  workflow_ = c.has("workflow") ? c.at("workflow").str : "";
  auto load_array = [&](const Json& v) -> NpyArray {
    if (v.type != Json::String || v.str.empty() || v.str[0] != '@') throw std::runtime_error("expected array reference");
    auto f = files.find(v.str.substr(1) + ".npy");
    if (f == files.end()) throw std::runtime_error("missing array file " + v.str.substr(1) + ".npy");
    return parse_npy(f->second);
  };
  for (auto& ju : c.at("units").arr) {
    UnitSpec u;
    u.cls = ju.at("class").at("name").str;
    u.uuid = ju.at("class").at("uuid").str;
    auto byuuid = fc_uuids().find(u.uuid);
    std::string cls = byuuid != fc_uuids().end() ? byuuid->second : u.cls;
    const Json& d = ju.at("data");
    if (ju.has("links")) u.links = int_list(ju.at("links"));
    if (d.has("include_bias")) u.include_bias = d.at("include_bias").b;
    bool wt = d.has("weights_transposed") && d.at("weights_transposed").b;
    if (d.has("activation_mode")) u.act = act_from_mode(d.at("activation_mode").str);
    auto take_weights = [&]() {
      u.weights = load_array(d.at("weights"));
      if (u.weights.shape.size() != 2) throw std::runtime_error(u.cls + ": weights must be 2-D");
      if (wt) {  // stored [in][out] -> [out][in]
        int64_t r = u.weights.shape[0], cc = u.weights.shape[1];
        std::vector<float> t((size_t)r * cc);
        for (int64_t i = 0; i < r; ++i) for (int64_t j = 0; j < cc; ++j) t[(size_t)j * r + i] = u.weights.data[(size_t)i * cc + j];
        u.weights.data.swap(t); std::swap(u.weights.shape[0], u.weights.shape[1]);
      }
      if (u.include_bias && d.has("bias")) {
        u.bias = load_array(d.at("bias"));
        if (u.bias.size() != u.weights.shape[0]) throw std::runtime_error(u.cls + ": bias size mismatch");
      } else u.include_bias = false;
    };
    if (cls.rfind("All2All", 0) == 0 || cls == "ResizableAll2All") {
      u.kind = "all2all"; take_weights();
      if (cls == "All2AllSoftmax") u.softmax = true;
      if (cls == "All2AllTanh") u.act = Act::Tanh;
      if (cls == "All2AllRELU") u.act = Act::Relu;
      if (cls == "All2AllStrictRELU") u.act = Act::StrictRelu;
      if (cls == "All2AllSigmoid") u.act = Act::Sigmoid;
    } else if (cls.rfind("Conv", 0) == 0) {
      u.kind = "conv"; take_weights();
      u.kx = (int)d.at("kx").num; u.ky = (int)d.at("ky").num; u.n_kernels = (int)d.at("n_kernels").num;
      auto pd = int_list(d.at("padding")); auto sl = int_list(d.at("sliding"));
      for (int i = 0; i < 4; ++i) u.pad[i] = pd.at(i);
      u.sx = sl.at(0); u.sy = sl.at(1);
      if (cls == "ConvTanh") u.act = Act::Tanh;
      if (cls == "ConvRELU") u.act = Act::Relu;
      if (cls == "ConvStrictRELU") u.act = Act::StrictRelu;
      if (cls == "ConvSigmoid") u.act = Act::Sigmoid;
    } else if (cls.find("Pooling") != std::string::npos) {
      u.kind = "pool";
      u.kx = (int)d.at("kx").num; u.ky = (int)d.at("ky").num;
      auto sl = int_list(d.at("sliding")); u.sx = sl.at(0); u.sy = sl.at(1);
      u.pool_mode = cls == "AvgPooling" ? 2 : (cls == "MaxAbsPooling" ? 1 : 0);
      if (cls.find("Stochastic") != std::string::npos)
        u.pool_mode = cls.find("Abs") != std::string::npos ? 1 : 0;   // inference: deterministic max
    } else if (cls == "LRNormalizerForward") {
      u.kind = "lrn";
      u.alpha = (float)d.at("alpha").num; u.beta = (float)d.at("beta").num;
      u.k = (float)d.at("k").num; u.n = (int)d.at("n").num;
    } else if (cls.rfind("Forward", 0) == 0) {
      u.kind = "act";
      static const std::map<std::string, int> codes = {
          {"ForwardTanh", 1}, {"ForwardRELU", 2}, {"ForwardStrictRELU", 3}, {"ForwardSigmoid", 4},
          {"ForwardMul", 5}, {"ForwardLog", 6}, {"ForwardTanhLog", 7}, {"ForwardSinCos", 8}};
      auto ci = codes.find(cls);
      if (ci == codes.end()) throw std::runtime_error("unknown activation unit " + cls);
      u.act_code = ci->second;
      if (d.has("factor") && d.at("factor").type == Json::Number) u.factor = (float)d.at("factor").num;
    } else if (cls == "Cutter") {
      u.kind = "cutter";
      auto pd = int_list(d.at("padding")); for (int i = 0; i < 4; ++i) u.pad[i] = pd.at(i);
    } else if (cls == "DropoutForward" || cls == "ZeroFiller") {
      u.kind = "identity";
    } else if (cls == "LSTMSequence") {
      u.kind = "lstm";
      if (wt) throw std::runtime_error(u.cls + ": weights_transposed is not supported (weights must be [4H][I + H])");
      take_weights();
      u.hidden = (int)d.at("hidden_size").num;
      u.return_sequences = d.has("return_sequences") && d.at("return_sequences").b;
      const int64_t rows = u.weights.shape[0], cols = u.weights.shape[1];
      if (u.hidden <= 0 || u.hidden >= cols)
        throw std::runtime_error(u.cls + ": hidden_size " + std::to_string(u.hidden) + " does not fit weights of " +
                                 std::to_string(cols) + " columns (I + H)");
      if (rows != 4LL * u.hidden)
        throw std::runtime_error(u.cls + ": weights have " + std::to_string(rows) + " rows, expected 4 * hidden_size = " +
                                 std::to_string(4LL * u.hidden));
    } else {
      throw std::runtime_error("unit class " + cls + " is not supported by the native runtime");
    }
    units_.push_back(std::move(u));
  }
  if (units_.empty()) throw std::runtime_error("package has no units");
}

Engine::~Engine() = default;

static int conv_out(int s, int k, int pa, int pb, int st) { return 1 + (s - k + pa + pb) / st; }
static int pool_out(int s, int k, int st) { int last = std::max(s - k, 0); return last / st + 1 + (last % st ? 1 : 0); }

Shape4 Engine::out_shape(const UnitSpec& u, const Shape4& in) const {
  Shape4 o = in;
  if (u.kind == "all2all") {
    if ((int64_t)in.h * in.w * in.c != u.weights.shape[1]) throw std::runtime_error(u.cls + ": input size != weights columns");
    o.h = o.w = 1; o.c = (int)u.weights.shape[0];
  } else if (u.kind == "conv") {
    if ((int64_t)u.kx * u.ky * in.c != u.weights.shape[1]) throw std::runtime_error(u.cls + ": channels mismatch");
    o.h = conv_out(in.h, u.ky, u.pad[1], u.pad[3], u.sy); o.w = conv_out(in.w, u.kx, u.pad[0], u.pad[2], u.sx);
    o.c = u.n_kernels;
  } else if (u.kind == "pool") {
    o.h = pool_out(in.h, u.ky, u.sy); o.w = pool_out(in.w, u.kx, u.sx);
  } else if (u.kind == "cutter") {
    o.h = in.h - u.pad[1] - u.pad[3]; o.w = in.w - u.pad[0] - u.pad[2];
    if (o.h <= 0 || o.w <= 0) throw std::runtime_error("cutter: empty output");
  } else if (u.kind == "lstm") {
    // a sample is [T][I]: [n, T, I] from python, [n, T * I], or the [T][H] output of an LSTM below
    const int64_t feat = u.weights.shape[1] - u.hidden, sz = (int64_t)in.h * in.w * in.c;
    if (sz <= 0 || sz % feat)
      throw std::runtime_error(u.cls + ": sample size " + std::to_string(sz) + " is not a multiple of " +
                               std::to_string(feat) + " input features");
    o.h = u.return_sequences ? (int)(sz / feat) : 1; o.w = 1; o.c = u.hidden;
  }
  return o;
}

Shape4 Engine::infer(const Shape4& in) {
  Shape4 s = in;
  for (auto& u : units_) s = out_shape(u, s);
  return s;
}

static inline float act5(Act a, float s) {
  switch (a) {
    case Act::Tanh: return 1.7159f * std::tanh(0.6666f * s);
    case Act::Relu: return s > 15.f ? s : std::log1p(std::exp(s));
    case Act::StrictRelu: return std::max(s, 0.f);
    case Act::Sigmoid: return 1.f / (1.f + std::exp(-s));
    default: return s;
  }
}
static inline float act_code(int code, float s, float factor, int idx) {
  switch (code) {
    case 1: return 1.7159f * std::tanh(0.6666f * s);
    case 2: return s > 15.f ? s : std::log1p(std::exp(s));
    case 3: return std::max(s, 0.f);
    case 4: return 1.f / (1.f + std::exp(-s));
    case 5: return s * factor;
    case 6: return std::log(s + std::sqrt(s * s + 1.f));
    case 7: { float a = std::fabs(s); if (a > 3.f) return std::copysign(std::log(a * 305.459953195f) * 0.242528761112f, s);
              return 1.7159f * std::tanh(0.6666f * s); }
    case 8: return (idx & 1) ? std::sin(s) : std::cos(s);
    default: return s;
  }
}
static void softmax_rows(float* y, int rows, int cols) {
  for (int r = 0; r < rows; ++r) {
    float* p = y + (size_t)r * cols;
    float m = *std::max_element(p, p + cols), s = 0.f;
    for (int c = 0; c < cols; ++c) { p[c] = std::exp(p[c] - m); s += p[c]; }
    for (int c = 0; c < cols; ++c) p[c] /= s;
  }
}

std::vector<float> Engine::run_cpu(const float* input, const Shape4& in) {
  std::vector<float> cur(input, input + in.size()), nxt;
  Shape4 s = in;
  for (auto& u : units_) {
    Shape4 o = out_shape(u, s);
    nxt.assign((size_t)o.size(), 0.f);
    if (u.kind == "all2all") {
      const int K = (int)u.weights.shape[1], N = o.c;
      // (pragmas are inert unless the build enables OpenMP: -DZNICZ_OPENMP=ON)
#pragma omp parallel for collapse(2) schedule(static)
      for (int b = 0; b < s.n; ++b) {
        for (int n = 0; n < N; ++n) {
          const float* x = cur.data() + (size_t)b * K;
          const float* w = u.weights.data.data() + (size_t)n * K;
          double acc = u.include_bias ? u.bias.data[n] : 0.0;
          for (int k = 0; k < K; ++k) acc += (double)x[k] * w[k];
          nxt[(size_t)b * N + n] = u.softmax ? (float)acc : act5(u.act, (float)acc);
        }
      }
      if (u.softmax) softmax_rows(nxt.data(), s.n, N);
    } else if (u.kind == "conv") {
      const int K = u.kx * u.ky * s.c;
#pragma omp parallel for collapse(3) schedule(static)
      for (int b = 0; b < s.n; ++b) for (int oy = 0; oy < o.h; ++oy) for (int ox = 0; ox < o.w; ++ox)
        for (int f = 0; f < o.c; ++f) {
          const float* w = u.weights.data.data() + (size_t)f * K;
          double acc = u.include_bias ? u.bias.data[f] : 0.0;
          for (int ky = 0; ky < u.ky; ++ky) {
            int iy = oy * u.sy - u.pad[1] + ky; if (iy < 0 || iy >= s.h) continue;
            for (int kx = 0; kx < u.kx; ++kx) {
              int ix = ox * u.sx - u.pad[0] + kx; if (ix < 0 || ix >= s.w) continue;
              const float* x = cur.data() + (((size_t)b * s.h + iy) * s.w + ix) * s.c;
              const float* ww = w + (size_t)(ky * u.kx + kx) * s.c;
              for (int c = 0; c < s.c; ++c) acc += (double)x[c] * ww[c];
            }
          }
          nxt[(((size_t)b * o.h + oy) * o.w + ox) * o.c + f] = act5(u.act, (float)acc);
        }
    } else if (u.kind == "pool") {
      for (int b = 0; b < s.n; ++b) for (int oy = 0; oy < o.h; ++oy) for (int ox = 0; ox < o.w; ++ox)
        for (int c = 0; c < s.c; ++c) {
          int y1 = oy * u.sy, x1 = ox * u.sx, y2 = std::min(y1 + u.ky, s.h), x2 = std::min(x1 + u.kx, s.w);
          float best = 0.f, key = -3.0e38f, sum = 0.f;
          for (int y = y1; y < y2; ++y) for (int x = x1; x < x2; ++x) {
            float v = cur[(((size_t)b * s.h + y) * s.w + x) * s.c + c];
            sum += v; float kk = u.pool_mode == 1 ? std::fabs(v) : v;
            if (kk > key) { key = kk; best = v; }
          }
          nxt[(((size_t)b * o.h + oy) * o.w + ox) * o.c + c] = u.pool_mode == 2 ? sum / ((y2 - y1) * (x2 - x1)) : best;
        }
    } else if (u.kind == "lrn") {
      const int C = s.c, half = u.n / 2; const int64_t px = s.size() / C;
      for (int64_t p = 0; p < px; ++p) for (int c = 0; c < C; ++c) {
        float sum = 0.f;
        for (int j = std::max(0, c - half); j <= std::min(C - 1, c + half); ++j) { float v = cur[p * C + j]; sum += v * v; }
        nxt[p * C + c] = cur[p * C + c] * std::pow(u.k + u.alpha * sum, -u.beta);
      }
    } else if (u.kind == "act") {
      for (int64_t i = 0; i < s.size(); ++i) nxt[i] = act_code(u.act_code, cur[i], u.factor, (int)(i & 1));
    } else if (u.kind == "lstm") {
      // ops/lstm_seq.py numpy_run: z = [x_t | h_{t-1}] W^T + b; i, f, o = sigma, g = A tanh(B z);
      // c = i g + f c_prev; h = o A tanh(B c); h_{-1} = c_{-1} = 0
      const int H = u.hidden, K = (int)u.weights.shape[1], I = K - H, T = (int)(s.size() / s.n / I);
      const float* W = u.weights.data.data();
      auto sigm = [](double v) { return 1.0 / (1.0 + std::exp(-v)); };
      auto stanh = [](double v) { return 1.7159 * std::tanh(0.6666 * v); };
#pragma omp parallel for schedule(static)
      for (int b = 0; b < s.n; ++b) {
        std::vector<float> xh(K, 0.f);
        std::vector<double> z(4 * H), c(H, 0.0);
        for (int t = 0; t < T; ++t) {
          std::memcpy(xh.data(), cur.data() + ((size_t)b * T + t) * I, sizeof(float) * I);
          for (int n = 0; n < 4 * H; ++n) {
            const float* w = W + (size_t)n * K;
            double acc = u.include_bias ? u.bias.data[n] : 0.0;
            for (int k = 0; k < K; ++k) acc += (double)xh[k] * w[k];
            z[n] = acc;
          }
          float* h = u.return_sequences ? &nxt[((size_t)b * T + t) * H] : (t == T - 1 ? &nxt[(size_t)b * H] : nullptr);
          for (int j = 0; j < H; ++j) {
            c[j] = sigm(z[j]) * stanh(z[2 * H + j]) + sigm(z[H + j]) * c[j];
            xh[I + j] = (float)(sigm(z[3 * H + j]) * stanh(c[j]));
            if (h) h[j] = xh[I + j];
          }
        }
      }
    } else if (u.kind == "cutter") {
      for (int b = 0; b < o.n; ++b) for (int y = 0; y < o.h; ++y) for (int x = 0; x < o.w; ++x)
        std::memcpy(&nxt[(((size_t)b * o.h + y) * o.w + x) * o.c],
                    &cur[(((size_t)b * s.h + y + u.pad[1]) * s.w + x + u.pad[0]) * s.c], sizeof(float) * o.c);
    } else {  // identity
      nxt = cur;
    }
    cur.swap(nxt); s = o;
  }
  return cur;
}

}  // namespace znicz

// ----------------------------------------------------------------------------------- C ABI
using znicz::Engine; using znicz::Shape4;
static void set_err(char* err, int n, const std::string& m) { if (err && n > 0) { std::strncpy(err, m.c_str(), n - 1); err[n - 1] = 0; } }
extern "C" {
void* znicz_engine_create(const char* path, char* err, int errlen) {
  try { return new Engine(path); } catch (const std::exception& e) { set_err(err, errlen, e.what()); return nullptr; }
}
void znicz_engine_destroy(void* e) { delete static_cast<Engine*>(e); }
int znicz_engine_num_units(void* e) { return (int)static_cast<Engine*>(e)->num_units(); }
int znicz_engine_infer(void* e, const int* s, int* o) {
  try { Shape4 in{s[0], s[1], s[2], s[3]}; Shape4 r = static_cast<Engine*>(e)->infer(in); o[0] = r.n; o[1] = r.h; o[2] = r.w; o[3] = r.c; return 0; }
  catch (...) { return 1; }
}
int znicz_engine_run(void* e, int backend, const float* input, const int* s, float* output, long long cap,
                     char* err, int errlen) {
  try {
    Shape4 in{s[0], s[1], s[2], s[3]};
    auto r = backend == 1 ? static_cast<Engine*>(e)->run_cuda(input, in) : static_cast<Engine*>(e)->run_cpu(input, in);
    if ((long long)r.size() > cap) { set_err(err, errlen, "output buffer too small"); return 2; }
    std::memcpy(output, r.data(), r.size() * sizeof(float));
    return 0;
  } catch (const std::exception& ex) { set_err(err, errlen, ex.what()); return 1; }
}
int znicz_cuda_available() { return Engine::cuda_available() ? 1 : 0; }
long long znicz_engine_tc_launches(void* e) { return static_cast<Engine*>(e)->cuda_tensor_core_launches(); }
}
