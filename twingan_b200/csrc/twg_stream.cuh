// A shared-memory ring that one 256-thread block fills with 1-D bulk copies (cp.async.bulk, completion on an mbarrier).
// The blocks that use it are each the only writer of a sum (one per sample, or one per batch), so the grid cannot be
// widened without changing the order of the additions; with direct loads such a block has the few float4 its threads hold
// in registers in flight, with the ring it has STAGES * NOPS * 16 KB.  The ring changes how the bytes reach a thread and
// nothing else: a thread reads from shared memory the elements it would have loaded, in the same order.
#pragma once
#include <mutex>

#include "twg_common.cuh"

namespace twg {

constexpr int kStreamStage = 16384;       // bytes of one operand in one stage: 1024 float4, four per thread

// An array is streamed when it fills at least two stages; below that the launch latency dominates and the direct-load
// kernels stay.
static inline bool stream_fills(int64_t bytes) { return bytes >= 2 * (int64_t)kStreamStage; }

// NOPS contiguous arrays of the same length advance together, chunk k of each in stage k % STAGES.  Every thread of the
// block calls start() once and then, for k = 0 .. chunks - 1: wait(k), its reads of at(k, op), release(k).
template <int NOPS, int STAGES>
struct StreamRing {
  static constexpr int kBytes = NOPS * STAGES * kStreamStage + 2 * STAGES * (int)sizeof(uint64_t);

  unsigned char* buf;
  uint64_t* full;
  uint64_t* empty;
  const unsigned char* src[NOPS];       // a null operand is not copied
  int64_t total;                        // bytes of each array (a multiple of 16)
  int chunks;

  // thread 0 only: the bulk copies of chunk k; the last chunk of an array is short and the barrier expects what is copied
  __device__ __forceinline__ void fill(int k) {
    const int s = k % STAGES;
    const int64_t off = (int64_t)k * kStreamStage;
    const uint32_t n = (uint32_t)(total - off < kStreamStage ? total - off : kStreamStage);
    uint32_t ops = 0;
#pragma unroll
    for (int op = 0; op < NOPS; ++op) ops += src[op] ? 1u : 0u;
    mbar_expect_tx(&full[s], n * ops);
#pragma unroll
    for (int op = 0; op < NOPS; ++op)
      if (src[op]) bulk_load_1d(buf + (size_t)(op * STAGES + s) * kStreamStage, src[op] + off, n, &full[s]);
  }

  __device__ __forceinline__ void start(unsigned char* smem, const void* const (&arrays)[NOPS], int64_t bytes) {
    buf = smem;
    full = reinterpret_cast<uint64_t*>(smem + (size_t)NOPS * STAGES * kStreamStage);
    empty = full + STAGES;
#pragma unroll
    for (int op = 0; op < NOPS; ++op) src[op] = static_cast<const unsigned char*>(arrays[op]);
    total = bytes;
    chunks = (int)((bytes + kStreamStage - 1) / kStreamStage);
    if (threadIdx.x == 0) {
      for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // empty: one arrive per warp
      fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int k = 0; k < STAGES && k < chunks; ++k) fill(k);
  }

  __device__ __forceinline__ void wait(int k) { mbar_wait(&full[k % STAGES], (uint32_t)(k / STAGES) & 1u); }

  __device__ __forceinline__ const float4* at(int k, int op) const {
    return reinterpret_cast<const float4*>(buf + (size_t)(op * STAGES + k % STAGES) * kStreamStage);
  }

  // The caller has its elements of chunk k in registers.  Thread 0 refills the stage of chunk k - 1, not of chunk k: by now
  // the other warps have most likely left that chunk, so the wait does not hold warp 0 back, and STAGES - 2 chunks stay in
  // flight.
  __device__ __forceinline__ void release(int k) {
    __syncwarp();
    mbar_arrive_lane0(&empty[k % STAGES], threadIdx.x & 31);
    if (threadIdx.x == 0 && k >= 1 && k - 1 + STAGES < chunks) {
      mbar_wait(&empty[(k - 1) % STAGES], (uint32_t)((k - 1) / STAGES) & 1u);
      fill(k - 1 + STAGES);
    }
  }
};

// one-time opt-in of a streamed kernel to its ring's dynamic shared memory, safe from several host threads
template <typename Kernel>
static cudaError_t allow_ring(Kernel kern, int bytes, std::once_flag& once, cudaError_t& err) {
  std::call_once(once, [&] { err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); });
  return err;
}

}  // namespace twg
