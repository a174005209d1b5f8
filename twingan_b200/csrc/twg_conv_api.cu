// C-ABI entry points of the convolution family: the exact-fp32 kernels on fp32 operands (pointwise for the thin 1x1
// layers, twg_conv_pw.cu; SIMT otherwise, twg_conv_simt.cu) and the wgmma tensor-core kernels on split-bf16 planes
// (twg_conv_tc.cu).
#include "twg_common.cuh"

namespace twg {
int conv_fwd_simt(const float*, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int conv_dgrad_simt(const float*, const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int conv_wgrad_simt(const float*, const float*, float*, int, int, int, int, int, int, int, int, cudaStream_t);
bool conv_tc_supported(int, int, int, int, int, int, int);
int split_act_planes(const float*, void*, int64_t, cudaStream_t);
int split_weight_planes(const float*, void*, int, int, int, int, cudaStream_t);
int split_weight_table(const float*, void*, const void*, int, int64_t, cudaStream_t);
int conv_fwd_tc_planes(const void*, const void*, float*, int, int, int, int, int, int, int, bool, cudaStream_t,
                       const float* bias = nullptr, int act = 0, void* z_planes = nullptr, float4* stats = nullptr,
                       uint8_t* act_mask = nullptr, const float* aff_a = nullptr);
int conv_fwd_epilogue_slots(int, int, int, int, int, int, int);
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

int twg_conv_path(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (pw_supported(Cin, Cout, k, pad)) return TWG_CONV_PW;
  return conv_tc_supported(N, H, W, Cin, Cout, k, pad) ? TWG_CONV_TC : TWG_CONV_SIMT;
}

int twg_conv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, int k, int pad,
                 twg_stream_t stream) {
  int rc = check_geom("twg_conv_fwd", x, w, y, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_fwd(x, w, y, (int64_t)N * H * W, Cin, Cout, S(stream));
  return conv_fwd_simt(x, w, y, N, H, W, Cin, Cout, k, pad, S(stream));
}

int twg_conv_dgrad(const float* gy, const float* w, float* gx, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   twg_stream_t stream) {
  int rc = check_geom("twg_conv_dgrad", gy, w, gx, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_dgrad(gy, w, gx, (int64_t)N * H * W, Cin, Cout, S(stream));
  return conv_dgrad_simt(gy, w, gx, N, H, W, Cin, Cout, k, pad, S(stream));
}

int twg_conv_wgrad(const float* x, const float* gy, float* gw, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   int accumulate, twg_stream_t stream) {
  int rc = check_geom("twg_conv_wgrad", x, gy, gw, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (pw_supported(Cin, Cout, k, pad)) return pw_wgrad(x, gy, gw, (int64_t)N * H * W, Cin, Cout, accumulate, S(stream));
  return conv_wgrad_simt(x, gy, gw, N, H, W, Cin, Cout, k, pad, accumulate, S(stream));
}

int twg_split_act(const float* x, void* planes, int64_t n, twg_stream_t stream) {
  if (!x || !planes || n <= 0) return fail(TWG_ERR_INVALID, "twg_split_act: bad args");
  return split_act_planes(x, planes, n, S(stream));
}

int twg_split_weights(const float* w, void* planes, int k, int Cin, int Cout, int dgrad, twg_stream_t stream) {
  if (!w || !planes || k <= 0 || Cin <= 0 || Cout <= 0) return fail(TWG_ERR_INVALID, "twg_split_weights: bad args");
  return split_weight_planes(w, planes, k, Cin, Cout, dgrad, S(stream));
}

int twg_split_weights_table(const float* flat, void* planes, const void* table, int rows, int64_t max_elems,
                            twg_stream_t stream) {
  if (!flat || !planes || !table || rows <= 0) return fail(TWG_ERR_INVALID, "twg_split_weights_table: bad args");
  return split_weight_table(flat, planes, table, rows, max_elems, S(stream));
}

int twg_conv_epilogue_slots(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return 0;
  return conv_fwd_epilogue_slots(N, H, W, Cin, Cout, k, pad);
}

int twg_conv_fwd_planes(const void* x_planes, const void* w_planes, const float* bias, int act, float* y, void* z_planes,
                        void* act_mask, float* stats, int N, int H, int W, int Cin, int Cout, int k, int pad,
                        twg_stream_t stream) {
  int rc = check_geom("twg_conv_fwd_planes", x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad);
  if (rc) return rc;
  if (act && !bias) return fail(TWG_ERR_INVALID, "twg_conv_fwd_planes: the activation needs a bias");
  return conv_fwd_tc_planes(x_planes, w_planes, y, N, H, W, Cin, Cout, k, pad, false, S(stream), bias, act, z_planes,
                            reinterpret_cast<float4*>(stats), reinterpret_cast<uint8_t*>(act_mask));
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

}  // extern "C"
