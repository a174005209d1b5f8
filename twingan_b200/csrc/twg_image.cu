// Image translation front and back end (inference/image_translation_infer.py:54-58, util_io.imsave): decoded uint8 RGB
// images of any size -> the model's [B, hw, hw, 3] fp32 input, and the model's output -> uint8 images.  Not part of the
// step.
//
// The front end restates TF 1.8's tf.image.convert_image_dtype (multiply by the fp32 constant 1/255) followed by
// tf.image.resize_images(method=BILINEAR, align_corners=False): resize_bilinear_op.cc without half-pixel centres, scale =
// in / out in fp32, source coordinate = dst * scale in fp32, the upper neighbour clamped to the last row / column.  Every
// operation is a separately rounded fp32 operation (no FMA contraction), in TF's order, so an image already at hw x hw
// comes out as exactly u8 * fl32(1/255).
#include "twg_common.cuh"

namespace twg {

constexpr float kInv255 = 1.0f / 255.0f;      // fl32(1/255), as convert_image_dtype's scale tensor

struct Taps {
  int i0, i1;
  float l;
};

// compute_interpolation_weights of resize_bilinear_op.cc for one output coordinate
__device__ __forceinline__ Taps taps_of(int o, float scale, int in_size) {
  const float in = __fmul_rn((float)o, scale);
  Taps t;
  t.i0 = min((int)in, in_size - 1);
  t.i1 = min(t.i0 + 1, in_size - 1);
  t.l = __fsub_rn(in, (float)t.i0);
  return t;
}

__device__ __forceinline__ float lerp_tf(float a, float b, float l) { return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), l)); }

// the three channels of output pixel P (flat over the batch: P = (b * hw + y) * hw + x)
__device__ __forceinline__ void resize_pixel(const uint8_t* __restrict__ payload, const int64_t* __restrict__ table,
                                             int64_t P, int hw, float* v) {
  const int64_t per = (int64_t)hw * hw;
  const int64_t b = P / per;
  const int r = (int)(P - b * per);
  const int y = r / hw, x = r - y * hw;
  const int64_t off = __ldg(table + 3 * b);
  const int H = (int)__ldg(table + 3 * b + 1), W = (int)__ldg(table + 3 * b + 2);
  const Taps ty = taps_of(y, __fdiv_rn((float)H, (float)hw), H);
  const Taps tx = taps_of(x, __fdiv_rn((float)W, (float)hw), W);
  const uint8_t* img = payload + off;
  const uint8_t* r0 = img + (int64_t)ty.i0 * W * 3;
  const uint8_t* r1 = img + (int64_t)ty.i1 * W * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float p00 = __fmul_rn((float)__ldg(r0 + tx.i0 * 3 + c), kInv255);
    const float p01 = __fmul_rn((float)__ldg(r0 + tx.i1 * 3 + c), kInv255);
    const float p10 = __fmul_rn((float)__ldg(r1 + tx.i0 * 3 + c), kInv255);
    const float p11 = __fmul_rn((float)__ldg(r1 + tx.i1 * 3 + c), kInv255);
    v[c] = lerp_tf(lerp_tf(p00, p01, tx.l), lerp_tf(p10, p11, tx.l), ty.l);
  }
}

// One thread per 4 consecutive output pixels of the flat batch: 12 floats, stored as 3 float4 (full 32-byte sectors
// across a warp).  The last group of a pixel count that is not a multiple of 4 is stored element by element.
__global__ void __launch_bounds__(256) k_images_u8_to_batch(const uint8_t* __restrict__ payload,
                                                            const int64_t* __restrict__ table, float* __restrict__ out,
                                                            int64_t npix, int hw) {
  const int64_t groups = (npix + 3) / 4;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t P0 = 4 * g;
    float v[12];
    if (P0 + 4 <= npix) {
#pragma unroll
      for (int j = 0; j < 4; ++j) resize_pixel(payload, table, P0 + j, hw, v + 3 * j);
      st4(out, 3 * g, make_float4(v[0], v[1], v[2], v[3]));
      st4(out, 3 * g + 1, make_float4(v[4], v[5], v[6], v[7]));
      st4(out, 3 * g + 2, make_float4(v[8], v[9], v[10], v[11]));
    } else {
      for (int64_t P = P0; P < npix; ++P) {
        resize_pixel(payload, table, P, hw, v);
        out[3 * P] = v[0];
        out[3 * P + 1] = v[1];
        out[3 * P + 2] = v[2];
      }
    }
  }
}

// util_io.imsave of the reference: clip(x * 255, 0, 255).astype(uint8) with the product rounded in fp32 and the
// conversion truncating.  fmaxf returns the other operand for a NaN, so NaN maps to 0.
__device__ __forceinline__ uint32_t to_u8(float x) {
  return (uint32_t)fminf(fmaxf(__fmul_rn(x, 255.f), 0.f), 255.f);
}

// One thread per 16 elements: four float4 loads, one 16-byte store (`vec`: both pointers 16-byte aligned).
__global__ void __launch_bounds__(256) k_batch_to_u8(const float* __restrict__ x, uint8_t* __restrict__ out, int64_t n,
                                                     int vec) {
  const int64_t groups = (n + 15) / 16;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e0 = 16 * g;
    if (vec && e0 + 16 <= n) {
      uint32_t w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 f = ld4(x, 4 * g + q);
        w[q] = to_u8(f.x) | (to_u8(f.y) << 8) | (to_u8(f.z) << 16) | (to_u8(f.w) << 24);
      }
      reinterpret_cast<uint4*>(out)[g] = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
      for (int64_t e = e0; e < n && e < e0 + 16; ++e) out[e] = (uint8_t)to_u8(x[e]);
    }
  }
}

}  // namespace twg

using namespace twg;

extern "C" {

int twg_images_u8_to_batch(const void* payload, const int64_t* table, float* out, int B, int hw, twg_stream_t stream) {
  if (!payload || !table || !out) return fail(TWG_ERR_INVALID, "twg_images_u8_to_batch: null");
  if (B < 1 || hw < 1 || hw > 32768)
    return fail(TWG_ERR_INVALID, "twg_images_u8_to_batch: B=%d hw=%d (B >= 1, 1 <= hw <= 32768)", B, hw);
  if (reinterpret_cast<uintptr_t>(out) & 15) return fail(TWG_ERR_INVALID, "twg_images_u8_to_batch: out not 16-byte aligned");
  const int64_t npix = (int64_t)B * hw * hw;
  k_images_u8_to_batch<<<grid_for(cdiv(npix, 4), 1), 256, 0, S(stream)>>>(static_cast<const uint8_t*>(payload), table,
                                                                         out, npix, hw);
  return check_launch("twg_images_u8_to_batch");
}

int twg_batch_to_u8(const float* x, void* out_u8, int64_t n, twg_stream_t stream) {
  if (!x || !out_u8) return fail(TWG_ERR_INVALID, "twg_batch_to_u8: null");
  if (n < 1) return fail(TWG_ERR_INVALID, "twg_batch_to_u8: n=%lld", (long long)n);
  const int vec = !(reinterpret_cast<uintptr_t>(x) & 15) && !(reinterpret_cast<uintptr_t>(out_u8) & 15);
  k_batch_to_u8<<<grid_for(cdiv(n, 16), 1), 256, 0, S(stream)>>>(x, static_cast<uint8_t*>(out_u8), n, vec);
  return check_launch("twg_batch_to_u8");
}

}  // extern "C"
