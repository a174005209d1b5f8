// C-ABI entry points of the convolution family: dispatch between the exact-fp32 CUDA-core path
// (prec=0, twg_conv_simt.cu) and the wgmma tensor-core path (prec=1, twg_conv_tc.cu).
#include <string.h>
#include "twg_common.cuh"

namespace twg {
int conv_fwd_simt(const float*, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int conv_dgrad_simt(const float*, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int conv_wgrad_simt(const float*, const float*, float*, int, int, int, int, int, int, int, int, cudaStream_t);
// tensor-core path; return TWG_ERR_UNSUPPORTED for shapes they do not cover
int conv_fwd_tc(const float*, const float*, float*, int, int, int, int, int, int, int, bool dgrad, void*, int64_t, cudaStream_t);
int conv_wgrad_tc(const float*, const float*, float*, int, int, int, int, int, int, int, int, void*, int64_t, cudaStream_t);
int64_t conv_tc_workspace(int, int, int, int, int, int, int);
bool conv_tc_supported(int, int, int, int, int, int, int);
int split_act_planes(const float*, void*, int64_t, cudaStream_t);
int split_weight_planes(const float*, void*, int, int, int, int, cudaStream_t);
int conv_fwd_tc_planes(const void*, const void*, float*, int, int, int, int, int, int, int, bool, cudaStream_t,
                       const float* bias = nullptr, int act = 0, void* z_planes = nullptr, float4* stats = nullptr,
                       uint8_t* act_mask = nullptr, const float* aff_a = nullptr);
bool conv_fwd_has_act_mask(int, int, int, int, int, int, int);
int conv_fwd_stats_slots(int, int, int, int, int, int, int);
int conv_wgrad_tc_planes(const void*, const void*, float*, int, int, int, int, int, int, int, int, cudaStream_t);
// thin 1x1 convs (fromRGB / toRGB), exact fp32
bool pw_supported(int Cin, int Cout, int k, int pad);
int pw_fwd(const float*, const float*, float*, int64_t, int, int, cudaStream_t);
int pw_dgrad(const float*, const float*, float*, int64_t, int, int, cudaStream_t);
int pw_wgrad(const float*, const float*, float*, int64_t, int, int, int, cudaStream_t);
}  // namespace twg

using namespace twg;

static int check_geom(const char* who, const void* a, const void* b, const void* c, int N, int H, int W, int Cin, int Cout,
                      int k, int pad) {
  if (!a || !b || !c) return fail(TWG_ERR_INVALID, "%s: null pointer", who);
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || k <= 0 || pad < 0 || pad >= k)
    return fail(TWG_ERR_INVALID, "%s: bad geometry N=%d H=%d W=%d Cin=%d Cout=%d k=%d pad=%d", who, N, H, W, Cin, Cout, k, pad);
  if (H + 2 * pad - k + 1 <= 0 || W + 2 * pad - k + 1 <= 0) return fail(TWG_ERR_INVALID, "%s: empty output", who);
  return TWG_OK;
}

extern "C" {

int64_t twg_conv_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int pad, int prec) {
  if (prec == 0 || pw_supported(Cin, Cout, k, pad)) return 0;
  return conv_tc_workspace(N, H, W, Cin, Cout, k, pad);
}

int twg_conv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, int k, int pad,
                 int prec, void* workspace, int64_t workspace_bytes, twg_stream_t stream) {
  int rc = check_geom("twg_conv_fwd", x, w, y, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_fwd(x, w, y, (int64_t)N * H * W, Cin, Cout, S(stream));
  if (prec == 1) return conv_fwd_tc(x, w, y, N, H, W, Cin, Cout, k, pad, false, workspace, workspace_bytes, S(stream));
  return conv_fwd_simt(x, w, y, N, H, W, Cin, Cout, k, pad, S(stream));
}

int twg_conv_dgrad(const float* gy, const float* w, float* gx, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   int prec, void* workspace, int64_t workspace_bytes, twg_stream_t stream) {
  int rc = check_geom("twg_conv_dgrad", gy, w, gx, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_dgrad(gy, w, gx, (int64_t)N * H * W, Cin, Cout, S(stream));
  if (prec == 1) return conv_fwd_tc(gy, w, gx, N, H, W, Cin, Cout, k, pad, true, workspace, workspace_bytes, S(stream));
  return conv_dgrad_simt(gy, w, gx, N, H, W, Cin, Cout, k, pad, S(stream));
}

int twg_conv_wgrad(const float* x, const float* gy, float* gw, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   int accumulate, int prec, void* workspace, int64_t workspace_bytes, twg_stream_t stream) {
  int rc = check_geom("twg_conv_wgrad", x, gy, gw, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_wgrad(x, gy, gw, (int64_t)N * H * W, Cin, Cout, accumulate, S(stream));
  if (prec == 1) return conv_wgrad_tc(x, gy, gw, N, H, W, Cin, Cout, k, pad, accumulate, workspace, workspace_bytes, S(stream));
  return conv_wgrad_simt(x, gy, gw, N, H, W, Cin, Cout, k, pad, accumulate, S(stream));
}

int twg_conv_tc_supported(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (pw_supported(Cin, Cout, k, pad)) return 0;
  return conv_tc_supported(N, H, W, Cin, Cout, k, pad) ? 1 : 0;
}

int twg_split_act(const float* x, void* planes, int64_t n, twg_stream_t stream) {
  if (!x || !planes || n <= 0) return fail(TWG_ERR_INVALID, "twg_split_act: bad args");
  return split_act_planes(x, planes, n, S(stream));
}

int twg_split_weights(const float* w, void* planes, int k, int Cin, int Cout, int dgrad, twg_stream_t stream) {
  if (!w || !planes || k <= 0 || Cin <= 0 || Cout <= 0) return fail(TWG_ERR_INVALID, "twg_split_weights: bad args");
  return split_weight_planes(w, planes, k, Cin, Cout, dgrad, S(stream));
}

int twg_conv_fwd_planes(const void* x_planes, const void* w_planes, float* y, int N, int H, int W, int Cin, int Cout,
                        int k, int pad, twg_stream_t stream) {
  int rc = check_geom("twg_conv_fwd_planes", x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  return conv_fwd_tc_planes(x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad, false, S(stream));
}

int twg_conv_stats_slots(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return 0;
  return conv_fwd_stats_slots(N, H, W, Cin, Cout, k, pad);
}

int twg_conv_fwd_planes_stats(const void* x_planes, const void* w_planes, float* y, float* stats, int N, int H, int W,
                              int Cin, int Cout, int k, int pad, twg_stream_t stream) {
  int rc = check_geom("twg_conv_fwd_planes_stats", x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (!stats) return fail(TWG_ERR_INVALID, "twg_conv_fwd_planes_stats: null stats");
  return conv_fwd_tc_planes(x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad, false, S(stream), nullptr, 0, nullptr,
                            reinterpret_cast<float4*>(stats));
}

int twg_conv_bias_act_fwd_planes(const void* x_planes, const void* w_planes, const float* bias, int lrelu_on, float* z,
                                 void* z_planes, int N, int H, int W, int Cin, int Cout, int k, int pad,
                                 twg_stream_t stream) {
  int rc = check_geom("twg_conv_bias_act_fwd_planes", x_planes, w_planes, z, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (!bias) return fail(TWG_ERR_INVALID, "twg_conv_bias_act_fwd_planes: null bias");
  return conv_fwd_tc_planes(x_planes, w_planes, z, N, H, W, Cin, Cout, k, pad, false, S(stream), bias, lrelu_on, z_planes);
}

int twg_conv_has_act_mask(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return 0;
  return conv_fwd_has_act_mask(N, H, W, Cin, Cout, k, pad) ? 1 : 0;
}

int twg_conv_bias_act_fwd_planes_mask(const void* x_planes, const void* w_planes, const float* bias, float* z, void* z_planes,
                                      void* act_mask, int N, int H, int W, int Cin, int Cout, int k, int pad,
                                      twg_stream_t stream) {
  int rc = check_geom("twg_conv_bias_act_fwd_planes_mask", x_planes, w_planes, z, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (!bias || !act_mask) return fail(TWG_ERR_INVALID, "twg_conv_bias_act_fwd_planes_mask: null bias / mask");
  return conv_fwd_tc_planes(x_planes, w_planes, z, N, H, W, Cin, Cout, k, pad, false, S(stream), bias, 1, z_planes, nullptr,
                            reinterpret_cast<uint8_t*>(act_mask));
}

int twg_conv_affine_act_fwd_planes(const void* x_planes, const void* w_planes, const float* a, const float* b, int flags,
                                   float* z, void* z_planes, int N, int H, int W, int Cin, int Cout, int k, int pad,
                                   twg_stream_t stream) {
  if (!z && !z_planes) return fail(TWG_ERR_INVALID, "twg_conv_affine_act_fwd_planes: no output");
  int rc = check_geom("twg_conv_affine_act_fwd_planes", x_planes, w_planes, a, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (!b) return fail(TWG_ERR_INVALID, "twg_conv_affine_act_fwd_planes: null affine");
  const int act = ((flags & TWG_FLAG_LRELU) ? 1 : 0) | ((flags & TWG_FLAG_PIXNORM) ? 2 : 0);
  return conv_fwd_tc_planes(x_planes, w_planes, z, N, H, W, Cin, Cout, k, pad, false, S(stream), b, act, z_planes, nullptr,
                            nullptr, a);
}

int twg_conv_dgrad_planes(const void* gy_planes, const void* w_planes, float* gx, int N, int H, int W, int Cin,
                          int Cout, int k, int pad, twg_stream_t stream) {
  int rc = check_geom("twg_conv_dgrad_planes", gy_planes, w_planes, gx, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  return conv_fwd_tc_planes(gy_planes, w_planes, gx, N, H, W, Cin, Cout, k, pad, true, S(stream));
}

int twg_conv_wgrad_planes(const void* x_planes, const void* gy_planes, float* gw, int N, int H, int W, int Cin,
                          int Cout, int k, int pad, int accumulate, twg_stream_t stream) {
  int rc = check_geom("twg_conv_wgrad_planes", x_planes, gy_planes, gw, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  return conv_wgrad_tc_planes(x_planes, gy_planes, gw, N, H, W, Cin, Cout, k, pad, accumulate, S(stream));
}

int64_t twg_crc32c(const void* data, int64_t n, int64_t crc) {
  static uint32_t table[8][256];
  static bool init = false;
  if (!init) {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      table[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int t = 1; t < 8; ++t) table[t][i] = (table[t - 1][i] >> 8) ^ table[0][table[t - 1][i] & 0xFF];
    init = true;
  }
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
