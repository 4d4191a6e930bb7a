// Host-side harness: runs the SAME __host__ __device__ token parser and "%f" formatter (csrc/bvh_text.cuh) the BVH text kernels
// use, so that tests/test_bvh_text_cpu.py checks them against Python's float() and '%f' without a GPU.  Test tooling only.
#include "../../ubisoft-laforge-zeroeggs_b200/csrc/bvh_text.cuh"
using namespace zeggs;

// tokens [n] as offsets into text (start, end pairs) -> out[i] and ok[i] (1: fast path, 0: flagged)
extern "C" void parse_tokens_host(const unsigned char* text, const long long* bounds, int n, double* out, int* ok) {
  for (int i = 0; i < n; ++i) {
    double v = 0.0;
    ok[i] = bvh_parse_token(text + bounds[2 * i], text + bounds[2 * i + 1], &v);
    out[i] = v;
  }
}

// values [n] -> "%f" texts, each in a slot of `stride` bytes; len[i] = length or -1 (flagged)
extern "C" void format_values_host(const double* v, int n, char* out, int stride, int* len) {
  for (int i = 0; i < n; ++i) {
    const int k = bvh_format_f(v[i], nullptr);
    len[i] = k;
    if (k >= 0 && k <= stride && bvh_format_f(v[i], out + (long long)i * stride) != k) len[i] = -2;
  }
}
