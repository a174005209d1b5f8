// The library's own runtime: the last-error string, the launch counter, the partial-sum buffer of the deterministic
// cross-block reductions, and the host-side entries that launch no kernel.
#include <stdarg.h>
#include <string.h>

#include "twg_common.cuh"

namespace twg {

thread_local char g_err[512] = {0};
std::atomic<int64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TWG_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return TWG_OK;
}

constexpr int64_t kPartialFloats = 8 << 20;        // 32 MB: the largest user is the tensor-core weight gradient (<= ~5 M)
__device__ float g_partials[kPartialFloats];

float* partials(int64_t n, bool zero, cudaStream_t st) {
  if (n > kPartialFloats) return nullptr;
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, g_partials) != cudaSuccess) return nullptr;
  if (zero) cudaMemsetAsync(p, 0, sizeof(float) * n, st);
  return static_cast<float*>(p);
}

__global__ void __launch_bounds__(256) k_add_partials(float* __restrict__ out, const float* __restrict__ parts, int nb,
                                                      int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < nb; ++b) s += parts[(int64_t)b * n + i];
    out[i] += s;
  }
}

int add_partials(float* out, const float* parts, int nb, int64_t n, cudaStream_t st) {
  int64_t blocks = cdiv(n, 256);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  k_add_partials<<<(unsigned)blocks, 256, 0, st>>>(out, parts, nb, n);
  return check_launch("add_partials");
}

// slicing-by-8 tables of CRC-32C (reflected polynomial 0x82F63B78)
struct Crc32cTable {
  uint32_t t[8][256];
  Crc32cTable() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int s = 1; s < 8; ++s) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 0xFF];
  }
};

}  // namespace twg

using namespace twg;

extern "C" {

int twg_version(void) { return 101; }
const char* twg_last_error(void) { return g_err; }
int64_t twg_launch_count(void) { return g_launches.load(); }

int64_t twg_crc32c(const void* data, int64_t n, int64_t crc) {
  static const Crc32cTable tables;        // built once, on first use; the initialisation is thread-safe
  const auto& table = tables.t;
  const uint8_t* p = static_cast<const uint8_t*>(data);
  uint32_t c = (uint32_t)crc ^ 0xFFFFFFFFu;
  while (n >= 8) {                       // slicing-by-8
    uint32_t lo, hi;
    memcpy(&lo, p, 4); memcpy(&hi, p + 4, 4);
    lo ^= c;
    c = table[7][lo & 0xFF] ^ table[6][(lo >> 8) & 0xFF] ^ table[5][(lo >> 16) & 0xFF] ^ table[4][lo >> 24] ^
        table[3][hi & 0xFF] ^ table[2][(hi >> 8) & 0xFF] ^ table[1][(hi >> 16) & 0xFF] ^ table[0][hi >> 24];
    p += 8; n -= 8;
  }
  while (n-- > 0) c = table[0][(c ^ *p++) & 0xFF] ^ (c >> 8);
  return (int64_t)(c ^ 0xFFFFFFFFu);
}

}  // extern "C"
