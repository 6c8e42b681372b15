// znicz_native — forward-only inference runtime for packages written by
// veles.znicz_b200.export.package (contents.json + NNNN_shape.npy in a zip).
//
// H100-native equivalent of the reference's libZnicz (All2All,
// All2AllLinear/Tanh/Softmax on libVeles+libSimd, single sample, CPU/NEON), extended to every
// exportable forward unit (conv, pooling, LRN, activations, cutter, dropout, the whole-sequence
// LSTM) and to batches.
// Two executors over one unit list: a portable CPU executor (the oracle of the C++ tests) and
// an sm_90a executor that launches the same hand-written kernels as the training engine
// (no libtorch, no cuBLAS/cuDNN).
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace znicz {

// ----------------------------------------------------------------------------- JSON (minimal)
struct Json {
  enum Type { Null, Bool, Number, String, Array, Object } type = Null;
  bool b = false;
  double num = 0;
  std::string str;
  std::vector<Json> arr;
  std::map<std::string, Json> obj;
  bool has(const std::string& k) const { return type == Object && obj.count(k); }
  const Json& at(const std::string& k) const;
  static Json parse(const std::string& text);
};

// ----------------------------------------------------------------------------- arrays
struct NpyArray {
  std::vector<int64_t> shape;
  std::vector<float> data;       // always widened to fp32 on load (f2 / f4 / f8 / i4 / i8 accepted)
  int64_t size() const;
};
NpyArray parse_npy(const std::string& bytes);

// zip archive (stored + deflate) -> name -> bytes; also accepts a directory path
std::map<std::string, std::string> read_package_files(const std::string& path);

// ----------------------------------------------------------------------------- units
enum class Act { Linear = 0, Tanh = 1, Relu = 2 /*softplus*/, StrictRelu = 3, Sigmoid = 4 };

struct Shape4 { int n = 1, h = 1, w = 1, c = 1; int64_t size() const { return (int64_t)n * h * w * c; } };

struct UnitSpec {
  std::string cls, uuid;
  std::string kind;              // all2all | conv | pool | lrn | act | cutter | identity | softmax | lstm
  Act act = Act::Linear;
  int act_code = 0;              // stand-alone activation kernel code (1..8)
  float factor = 1.f;
  bool softmax = false;
  NpyArray weights, bias;        // weights always [out][in] / [F][ky*kx*C] after load
  bool include_bias = true;
  int kx = 0, ky = 0, n_kernels = 0, sx = 1, sy = 1;
  int pad[4] = {0, 0, 0, 0};     // left, top, right, bottom
  int pool_mode = 0;             // 0 max, 1 maxabs, 2 avg
  float alpha = 1e-4f, beta = 0.75f, k = 2.f; int n = 5;
  // lstm: weights [4H][I + H] (gates input, forget, memory, output), bias [4H]; a sample of
  // h*w*c floats is T = h*w*c / I steps of I features; output [T][H] or the last step's [H]
  int hidden = 0;
  bool return_sequences = false;
  std::vector<int> links;
};

class Engine {
 public:
  // Loads and validates a package (.zip or extracted directory).
  explicit Engine(const std::string& package_path);
  ~Engine();
  const std::string& workflow_name() const { return workflow_; }
  size_t num_units() const { return units_.size(); }
  const UnitSpec& unit(size_t i) const { return units_[i]; }

  // Infers output shape for an input of `in` (NHWC; FC nets: h = w = 1, c = features).
  Shape4 infer(const Shape4& in);
  // CPU executor. input: n*h*w*c floats. Returns the last unit's output.
  std::vector<float> run_cpu(const float* input, const Shape4& in);
  // sm_90a executor (throws std::runtime_error when no CUDA device is usable).
  std::vector<float> run_cuda(const float* input, const Shape4& in);
  static bool cuda_available();
  // wgmma GEMM / conv launches issued by run_cuda() so far (0: every layer took the SIMT path)
  long long cuda_tensor_core_launches() const;

 private:
  struct CudaState;
  std::string workflow_;
  std::vector<UnitSpec> units_;
  std::shared_ptr<CudaState> cuda_;   // type-erased deleter: CudaState is private to engine_cuda.cc
  Shape4 out_shape(const UnitSpec& u, const Shape4& in) const;
};

}  // namespace znicz

// ----------------------------------------------------------------------------- C ABI (ctypes)
extern "C" {
void* znicz_engine_create(const char* path, char* err, int errlen);
void znicz_engine_destroy(void* e);
int znicz_engine_num_units(void* e);
int znicz_engine_infer(void* e, const int* in_shape4, int* out_shape4);
// backend: 0 = cpu, 1 = cuda. Returns 0 on success.
int znicz_engine_run(void* e, int backend, const float* input, const int* in_shape4, float* output,
                     long long out_capacity, char* err, int errlen);
int znicz_cuda_available();
long long znicz_engine_tc_launches(void* e);
}
