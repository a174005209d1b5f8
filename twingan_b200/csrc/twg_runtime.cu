// The library's own runtime: the last-error string, the launch counter, the partial-sum buffer of the deterministic
// cross-block reductions, and the host-side entries that launch no kernel.
#include <stdarg.h>
#include <string.h>

#include <mutex>

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
// One region per stream that may run library work concurrently with another: region 0 serves every stream not bound
// to a region of its own, regions 1.. are bound one stream each per device (twg_partials_bind; the table is keyed on the
// current device, which is the device of the stream a launch goes to).  Fixed and preallocated, so a launch captured into
// a CUDA graph never allocates.
constexpr int kPartialRegions = 2;
constexpr int kMaxDevices = 64;
__device__ float g_partials[kPartialRegions * kPartialFloats];

std::mutex g_region_mu;
cudaStream_t g_region_stream[kMaxDevices][kPartialRegions] = {};   // [d][0] unused: region 0 has no owner
bool g_region_bound[kMaxDevices][kPartialRegions] = {};
std::atomic<int64_t> g_region_uses[kPartialRegions] = {};           // partials() calls served, all devices

int current_device() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess) {     // no device (host-only use of the table): keep slot 0
    cudaGetLastError();
    d = 0;
  }
  return d;
}

int partials_region(int dev, cudaStream_t st) {
  if (dev < 0 || dev >= kMaxDevices) return 0;
  std::lock_guard<std::mutex> lock(g_region_mu);
  for (int r = 1; r < kPartialRegions; ++r)
    if (g_region_bound[dev][r] && g_region_stream[dev][r] == st) return r;
  return 0;
}

float* partials(int64_t n, bool zero, cudaStream_t st) {
  if (n > kPartialFloats) return nullptr;
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, g_partials) != cudaSuccess) return nullptr;
  int r = partials_region(current_device(), st);
  g_region_uses[r].fetch_add(1, std::memory_order_relaxed);
  float* region = static_cast<float*>(p) + r * kPartialFloats;
  if (zero) cudaMemsetAsync(region, 0, sizeof(float) * n, st);
  return region;
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

int twg_partials_regions(void) { return kPartialRegions; }
int64_t twg_partials_region_floats(void) { return kPartialFloats; }
int twg_partials_region(const void* stream_key) { return partials_region(current_device(), (cudaStream_t)stream_key); }

int64_t twg_partials_region_uses(int region) {
  return (region >= 0 && region < kPartialRegions) ? g_region_uses[region].load() : -1;
}

int twg_partials_bind(const void* stream_key, int region) {
  cudaStream_t st = (cudaStream_t)stream_key;
  if (region < 0 || region >= kPartialRegions)
    return fail(TWG_ERR_INVALID, "partials_bind: region %d is not one of 0..%d", region, kPartialRegions - 1);
  if (st == nullptr) return fail(TWG_ERR_INVALID, "partials_bind: the default stream keeps region 0");
  int dev = current_device();
  if (dev >= kMaxDevices) return fail(TWG_ERR_INVALID, "partials_bind: device %d is beyond %d", dev, kMaxDevices);
  std::lock_guard<std::mutex> lock(g_region_mu);
  cudaStream_t* owner = g_region_stream[dev];
  bool* bound = g_region_bound[dev];
  for (int r = 1; r < kPartialRegions; ++r)
    if (bound[r] && owner[r] == st && r != region) {
      if (region != 0) return fail(TWG_ERR_INVALID, "partials_bind: the stream already owns region %d", r);
      bound[r] = false;                               // region 0: the stream gives its region back
      owner[r] = nullptr;
    }
  if (region == 0) return TWG_OK;
  if (bound[region] && owner[region] != st)
    return fail(TWG_ERR_INVALID, "partials_bind: region %d belongs to another stream", region);
  owner[region] = st;
  bound[region] = true;
  return TWG_OK;
}

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
