// C++ tests of the native runtime (mirrors /root/reference/libZnicz/tests/all2all*.cc:
// typed fixtures with hand-computed expectations to 1e-6 relative), plus package parsing,
// conv/pool/LRN/cutter units and (when a GPU is present) CPU-vs-sm_90a agreement.
#include "../src/znicz_native.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <sys/stat.h>
#include <unistd.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_NEAR(a, b, tol) do { ++g_checks; double a_ = (a), b_ = (b); if (!(std::fabs(a_ - b_) <= (tol))) { ++g_fail; std::printf("FAIL %s:%d %s=%g vs %s=%g\n", __FILE__, __LINE__, #a, a_, #b, b_); } } while (0)
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); } } while (0)

static void write_npy(const std::string& path, const std::vector<int>& shape, const std::vector<float>& data) {
  std::string sh = "(";
  for (size_t i = 0; i < shape.size(); ++i) sh += std::to_string(shape[i]) + (shape.size() == 1 || i + 1 < shape.size() ? "," : "");
  sh += ")";
  std::string hdr = "{'descr': '<f4', 'fortran_order': False, 'shape': " + sh + ", }";
  while ((10 + hdr.size() + 1) % 64) hdr += ' ';
  hdr += '\n';
  std::ofstream f(path, std::ios::binary);
  f.write("\x93NUMPY\x01\x00", 8);
  uint16_t l = (uint16_t)hdr.size(); f.write(reinterpret_cast<char*>(&l), 2);
  f.write(hdr.data(), hdr.size());
  f.write(reinterpret_cast<const char*>(data.data()), data.size() * 4);
}

struct TmpDir {
  std::string path;
  TmpDir() { char t[] = "/tmp/znicz_native_XXXXXX"; path = mkdtemp(t); }
  ~TmpDir() { std::string c = "rm -rf " + path; if (std::system(c.c_str())) {} }
};

static void write_contents(const std::string& dir, const std::string& units_json) {
  std::ofstream f(dir + "/contents.json");
  f << "{\"checksum\": \"x_1\", \"workflow\": \"TestWorkflow\", \"units\": [" << units_json << "]}";
}

// 3x5 weights / 5 inputs as in the reference FC fixtures
static const std::vector<float> W = {1, 2, 3, 2, 1,  0, 1, 2, 1, 0,  0, 1, 0, 1, 0};
static const std::vector<float> B = {10, -10, 5};
static const std::vector<float> X = {1, 2, 3, 2, 1};

static void test_fc(const char* cls, const char* uuid, const char* mode, const double* expect) {
  TmpDir d;
  write_npy(d.path + "/0000_3.npy", {3}, B);
  write_npy(d.path + "/0001_3x5.npy", {3, 5}, W);
  std::ostringstream u;
  u << "{\"class\": {\"name\": \"" << cls << "\", \"uuid\": \"" << uuid << "\"}, \"data\": {\"activation_mode\": \"" << mode
    << "\", \"bias\": \"@0000_3\", \"include_bias\": true, \"weights\": \"@0001_3x5\", \"weights_transposed\": false}, \"links\": []}";
  write_contents(d.path, u.str());
  znicz::Engine e(d.path);
  EXPECT_TRUE(e.num_units() == 1);
  znicz::Shape4 in{1, 1, 1, 5};
  auto y = e.run_cpu(X.data(), in);
  EXPECT_TRUE(y.size() == 3);
  for (int i = 0; i < 3; ++i) EXPECT_NEAR(y[i], expect[i], std::fabs(expect[i]) / 1e6 + 1e-9);
  if (znicz::Engine::cuda_available()) {
    auto g = e.run_cuda(X.data(), in);
    for (int i = 0; i < 3; ++i) EXPECT_NEAR(g[i], y[i], 1e-5 + std::fabs(y[i]) * 1e-5);
  }
}

static void test_conv_chain() {
  TmpDir d;
  // conv 2 kernels 2x2 on 1x3x3x1, padding 0, stride 1 -> 2x2x2; maxpool 2x2 -> 1x1x2; softmax FC 2->2
  write_npy(d.path + "/0000_2.npy", {2}, {0.5f, -0.5f});
  write_npy(d.path + "/0001_2x4.npy", {2, 4}, {1, 0, 0, 1,  -1, 1, 1, -1});
  write_npy(d.path + "/0002_2.npy", {2}, {0.f, 0.f});
  write_npy(d.path + "/0003_2x2.npy", {2, 2}, {1, 0, 0, 1});
  std::string u =
      "{\"class\": {\"name\": \"ConvStrictRELU\", \"uuid\": \"c1\"}, \"data\": {\"activation_mode\": \"ACTIVATION_STRICT_RELU\","
      " \"bias\": \"@0000_2\", \"include_bias\": true, \"weights\": \"@0001_2x4\", \"weights_transposed\": false, \"kx\": 2, \"ky\": 2,"
      " \"n_kernels\": 2, \"padding\": [0, 0, 0, 0], \"sliding\": [1, 1]}, \"links\": [1]},"
      "{\"class\": {\"name\": \"MaxPooling\", \"uuid\": \"p1\"}, \"data\": {\"kx\": 2, \"ky\": 2, \"sliding\": [2, 2]}, \"links\": [2]},"
      "{\"class\": {\"name\": \"All2AllSoftmax\", \"uuid\": \"420219fc-3e1a-45b1-87f8-aaa0c1540de4\"}, \"data\": {\"activation_mode\":"
      " \"ACTIVATION_LINEAR\", \"bias\": \"@0002_2\", \"include_bias\": true, \"weights\": \"@0003_2x2\", \"weights_transposed\": false}, \"links\": []}";
  write_contents(d.path, u);
  znicz::Engine e(d.path);
  std::vector<float> x = {1, 2, 3, 4, 5, 6, 7, 8, 9};
  znicz::Shape4 in{1, 3, 3, 1};
  znicz::Shape4 o = e.infer(in);
  EXPECT_TRUE(o.n == 1 && o.h == 1 && o.w == 1 && o.c == 2);
  auto y = e.run_cpu(x.data(), in);
  // conv k0 = x[y,x] + x[y+1,x+1] + 0.5: {6.5, 8.5, 12.5, 14.5}; k1 = -a+b+c-d-0.5 = -0.5 -> relu 0
  // maxpool -> {14.5, 0}; softmax -> {1/(1+e^-14.5), ...}
  double e0 = 1.0 / (1.0 + std::exp(-14.5));
  EXPECT_NEAR(y[0], e0, 1e-6);
  EXPECT_NEAR(y[1], 1.0 - e0, 1e-6);
  if (znicz::Engine::cuda_available()) {
    auto g = e.run_cuda(x.data(), in);
    EXPECT_NEAR(g[0], y[0], 1e-5);
    EXPECT_NEAR(g[1], y[1], 1e-5);
  }
}

static void test_errors() {
  bool thrown = false;
  try { znicz::Engine e("/nonexistent/package.zip"); } catch (const std::exception&) { thrown = true; }
  EXPECT_TRUE(thrown);
  znicz::Json j = znicz::Json::parse("{\"a\": [1, 2.5, true, null, \"s\\n\"], \"b\": {\"c\": -3e2}}");
  EXPECT_TRUE(j.at("a").arr.size() == 5);
  EXPECT_NEAR(j.at("b").at("c").num, -300.0, 0);
}

static std::string slurp(const char* path) {
  std::FILE* f = std::fopen(path, "rb");
  if (!f) throw std::runtime_error(std::string("cannot open ") + path);
  std::string data; char buf[65536]; size_t n;
  while ((n = std::fread(buf, 1, sizeof buf, f)) > 0) data.append(buf, n);
  std::fclose(f);
  return data;
}

// End-to-end check of an exported network (the body the reference's functional_mnist.cc never
// got, /root/reference/libZnicz/tests/functional_mnist.cc): run the packaged workflow on a batch
// saved by python and compare with python's own forward pass, on every available executor.
static void test_functional(const char* pkg, const char* in_npy, const char* ref_npy) {
  try {
    znicz::Engine e(pkg);
    znicz::NpyArray x = znicz::parse_npy(slurp(in_npy)), ref = znicz::parse_npy(slurp(ref_npy));
    znicz::Shape4 in;
    in.n = (int)x.shape.at(0);
    if (x.shape.size() == 4) { in.h = (int)x.shape[1]; in.w = (int)x.shape[2]; in.c = (int)x.shape[3]; }
    else { int64_t k = 1; for (size_t i = 1; i < x.shape.size(); ++i) k *= x.shape[i]; in.c = (int)k; }
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 1 && !znicz::Engine::cuda_available()) break;
      std::vector<float> y = pass ? e.run_cuda(x.data.data(), in) : e.run_cpu(x.data.data(), in);
      EXPECT_TRUE(y.size() == ref.data.size());
      double worst = 0;
      for (size_t i = 0; i < y.size() && i < ref.data.size(); ++i)
        worst = std::max(worst, std::fabs((double)y[i] - ref.data[i]));
      std::printf("functional %s: %zu outputs, max |diff| %.3g\n", pass ? "cuda" : "cpu", y.size(), worst);
      EXPECT_TRUE(worst < 2e-3);    // fp16-packed weights vs python fp32
    }
  } catch (const std::exception& ex) { ++g_fail; std::printf("FAIL functional: %s\n", ex.what()); }
}

int main(int argc, char** argv) {
  // expectations: s = W x + b = {29, 0, 9}
  const double lin[3] = {29, 0, 9};
  const double tnh[3] = {1.7159 * std::tanh(0.6666 * 29), 1.7159 * std::tanh(0.6666 * 0), 1.7159 * std::tanh(0.6666 * 9)};
  double m = 29, s = std::exp(29 - m) + std::exp(0 - m) + std::exp(9 - m);
  const double smx[3] = {std::exp(29 - m) / s, std::exp(0 - m) / s, std::exp(9 - m) / s};
  const double sig[3] = {1 / (1 + std::exp(-29.0)), 1 / (1 + std::exp(-0.0)), 1 / (1 + std::exp(-9.0))};
  test_fc("All2All", "58a5eadf-ae1e-498f-bf35-7d93939c4c86", "ACTIVATION_LINEAR", lin);
  test_fc("All2AllTanh", "b3a2bd5c-3c01-46ef-978a-fef22e008f31", "ACTIVATION_TANH", tnh);
  test_fc("All2AllSoftmax", "420219fc-3e1a-45b1-87f8-aaa0c1540de4", "ACTIVATION_LINEAR", smx);
  test_fc("All2AllSigmoid", "a27974ec-1764-4944-925d-4862de237881", "ACTIVATION_SIGMOID", sig);
  test_conv_chain();
  test_errors();
  if (argc > 1) {   // extra: load a package produced by the python exporter
    try { znicz::Engine e(argv[1]); EXPECT_TRUE(e.num_units() > 0); std::printf("loaded %s: %zu units\n", argv[1], e.num_units()); }
    catch (const std::exception& ex) { ++g_fail; std::printf("FAIL load %s: %s\n", argv[1], ex.what()); }
  }
  if (argc > 3) {   // functional: package + input.npy + expected.npy (python forward of the same net)
    test_functional(argv[1], argv[2], argv[3]);
  }
  std::printf("%d checks, %d failures, cuda=%d\n", g_checks, g_fail, (int)znicz::Engine::cuda_available());
  return g_fail ? 1 : 0;
}
