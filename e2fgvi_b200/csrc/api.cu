// extern "C" boundary of libe2fgvi_b200.so (declared in include/e2fgvi_b200.h): argument validation, error
// strings, launch accounting, TMA tensor-map encoding.  No torch types, no allocation; the only process-wide state is per-device-ordinal caches
// of immutable facts (SM count, "function attributes already set on device d", cluster occupancy; launch.h DeviceOnce).
#include <atomic>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "e2fgvi_b200.h"
#include "launch.h"

namespace e2f {

static thread_local char g_err[512] = {0};
static std::atomic<long long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static std::atomic<int> cache[64];
  const int dev = current_device();
  int v = (dev >= 0 && dev < 64) ? cache[dev].load(std::memory_order_relaxed) : 0;
  if (!v) {
    v = 132;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (dev >= 0 && dev < 64) cache[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int encode_tmap(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                const cuuint32_t* box, const cuuint32_t* estr, const char* what, CUtensorMapDataType type) {
  using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeTiledFn encode = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  if (!encode) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the driver", what);
    return -4;
  }
  const CUresult r = encode(map, type, static_cast<cuuint32_t>(rank), const_cast<void*>(base), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char shape[128] = "";
    for (int i = 0, len = 0; i < rank; ++i)
      len += snprintf(shape + len, sizeof(shape) - len, "%s%llu", i ? " x " : "", static_cast<unsigned long long>(dims[i]));
    set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (dims %s)", what, static_cast<int>(r), shape);
    return -4;
  }
  return 0;
}

static int finish(int status, const char* what) {
  if (status > 0) set_error("%s: CUDA error %d (%s)", what, status, cudaGetErrorString(static_cast<cudaError_t>(status)));
  return status;
}

static bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace e2f

using namespace e2f;

extern "C" {

const char* e2f_version(void) { return "e2fgvi_b200 0.1.0 sm_90a"; }

const char* e2f_last_error(void) { return g_err; }

int64_t e2f_launch_count(void) { return static_cast<int64_t>(g_launches.load(std::memory_order_relaxed)); }

int e2f_flow_warp(const void* x, const float* flow, void* out, int n, int h, int w, int c, int dtype, int pad_mode,
                  void* stream) {
  if (!x || !flow || !out) { set_error("e2f_flow_warp: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c <= 0) { set_error("e2f_flow_warp: bad shape n=%d h=%d w=%d c=%d", n, h, w, c); return E2F_ERR_BAD_ARG; }
  if (dtype != E2F_F32 && dtype != E2F_F16) { set_error("e2f_flow_warp: dtype %d", dtype); return E2F_ERR_BAD_ARG; }
  if (pad_mode != E2F_PAD_ZEROS && pad_mode != E2F_PAD_BORDER) { set_error("e2f_flow_warp: pad_mode %d", pad_mode); return E2F_ERR_BAD_ARG; }
  const int vec = dtype == E2F_F16 ? 8 : 4;
  if (c % vec) { set_error("e2f_flow_warp: C=%d must be a multiple of %d for the NHWC kernel (use e2f_flow_warp_nchw)", c, vec); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(x, 16) || !aligned(out, 16) || !aligned(flow, 8)) { set_error("e2f_flow_warp: x/out need 16-byte, flow 8-byte alignment"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_flow_warp_nhwc(x, flow, out, n, h, w, c, dtype, pad_mode, static_cast<cudaStream_t>(stream)), "e2f_flow_warp");
}

int e2f_flow_warp_nchw(const float* x, const float* flow, float* out, int n, int c, int h, int w, int pad_mode,
                       void* stream) {
  if (!x || !flow || !out) { set_error("e2f_flow_warp_nchw: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c <= 0) { set_error("e2f_flow_warp_nchw: bad shape"); return E2F_ERR_BAD_ARG; }
  if (pad_mode != E2F_PAD_ZEROS && pad_mode != E2F_PAD_BORDER) { set_error("e2f_flow_warp_nchw: pad_mode %d", pad_mode); return E2F_ERR_BAD_ARG; }
  if (!aligned(flow, 8)) { set_error("e2f_flow_warp_nchw: flow needs 8-byte alignment"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_flow_warp_nchw(x, flow, out, n, c, h, w, pad_mode, static_cast<cudaStream_t>(stream)), "e2f_flow_warp_nchw");
}

static int flow_warp_backward_checks(const char* who, const float* x, const float* flow, const float* dout,
                                     const float* dflow_res, const float* dflow, const float* dx_res, const float* dx,
                                     const void* work, int n, int h, int w, int c) {
  if (!flow || !dout) { set_error("%s: null flow / dout", who); return E2F_ERR_BAD_ARG; }
  if (!dflow && !dx) { set_error("%s: nothing to compute (need dflow or dx)", who); return E2F_ERR_BAD_ARG; }
  if (dflow && !x) { set_error("%s: dflow needs x", who); return E2F_ERR_BAD_ARG; }
  if (dx && !work) { set_error("%s: dx needs the scatter workspace", who); return E2F_ERR_BAD_ARG; }
  if ((dflow_res && !dflow) || (dx_res && !dx)) { set_error("%s: a residual goes with its output", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c <= 0) { set_error("%s: bad shape n=%d h=%d w=%d c=%d", who, n, h, w, c); return E2F_ERR_BAD_ARG; }
  if (static_cast<long long>(n) * h * w * 4 > INT_MAX) { set_error("%s: N*H*W=%lld too large (N*H*W*4 must fit in int)", who, static_cast<long long>(n) * h * w); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(flow, 8) || (dflow && !aligned(dflow, 8)) || (dflow_res && !aligned(dflow_res, 8)) || (work && !aligned(work, 256))) { set_error("%s: flow / dflow need 8-byte, work 256-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return 0;
}

int64_t e2f_flow_warp_backward_work_elems(int n, int h, int w) {
  const char* who = "e2f_flow_warp_backward_work_elems";
  if (n < 0 || h <= 0 || w <= 0) { set_error("%s: bad shape n=%d h=%d w=%d", who, n, h, w); return E2F_ERR_BAD_ARG; }
  if (static_cast<long long>(n) * h * w * 4 > INT_MAX) { set_error("%s: N*H*W=%lld too large (N*H*W*4 must fit in int)", who, static_cast<long long>(n) * h * w); return E2F_ERR_UNSUPPORTED; }
  return static_cast<int64_t>(flow_warp_backward_work_elems(n, h, w));
}

int e2f_flow_warp_backward_nhwc(const float* x, const float* flow, const float* dout, const float* dflow_residual,
                                float* dflow, const float* dx_residual, float* dx, void* work, int n, int h, int w,
                                int c, void* stream) {
  const char* who = "e2f_flow_warp_backward_nhwc";
  if (const int st = flow_warp_backward_checks(who, x, flow, dout, dflow_residual, dflow, dx_residual, dx, work, n, h, w, c)) return st;
  if (c % 4) { set_error("%s: C=%d must be a multiple of 4 (use e2f_flow_warp_backward_nchw)", who, c); return E2F_ERR_UNSUPPORTED; }
  if ((x && !aligned(x, 16)) || !aligned(dout, 16) || (dx && !aligned(dx, 16)) || (dx_residual && !aligned(dx_residual, 16))) { set_error("%s: x / dout / dx / dx_residual need 16-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_flow_warp_backward(x, 0, 0, flow, dout, dflow_residual, dflow, dx_residual, dx, work, n, h, w, c,
                                          static_cast<cudaStream_t>(stream)), who);
}

int e2f_flow_warp_backward_nchw(const float* x, int64_t x_bstride, const float* flow, const float* dout,
                                const float* dflow_residual, float* dflow, const float* dx_residual, float* dx,
                                void* work, int n, int c, int h, int w, void* stream) {
  const char* who = "e2f_flow_warp_backward_nchw";
  if (const int st = flow_warp_backward_checks(who, x, flow, dout, dflow_residual, dflow, dx_residual, dx, work, n, h, w, c)) return st;
  if (x && x_bstride < static_cast<int64_t>(c) * h * w) { set_error("%s: x batch stride %lld < C*H*W", who, static_cast<long long>(x_bstride)); return E2F_ERR_BAD_ARG; }
  return finish(launch_flow_warp_backward(x, static_cast<long long>(x_bstride), 1, flow, dout, dflow_residual, dflow,
                                          dx_residual, dx, work, n, h, w, c, static_cast<cudaStream_t>(stream)), who);
}

int e2f_dcn_pack_weight(const float* w, void* w_packed_f16, int cout, int cin, int deform_groups, void* stream) {
  if (!w || !w_packed_f16) { set_error("e2f_dcn_pack_weight: null pointer"); return E2F_ERR_BAD_ARG; }
  if (cout <= 0 || cin <= 0 || deform_groups <= 0 || cin % deform_groups) { set_error("e2f_dcn_pack_weight: bad shape"); return E2F_ERR_BAD_ARG; }
  return finish(launch_dcn_pack_weight(w, w_packed_f16, cout, cin, deform_groups, static_cast<cudaStream_t>(stream)), "e2f_dcn_pack_weight");
}

static int dcn_common_checks(const char* who, const void* x, const void* w_packed, const void* out, int n, int h, int w,
                             int out_dtype) {
  if (!x || !w_packed || !out) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0) { set_error("%s: bad shape n=%d h=%d w=%d", who, n, h, w); return E2F_ERR_BAD_ARG; }
  if (out_dtype != E2F_F32 && out_dtype != E2F_F16) { set_error("%s: out_dtype %d", who, out_dtype); return E2F_ERR_BAD_ARG; }
  if (!aligned(x, 32) || !aligned(w_packed, 128) || !aligned(out, 16)) { set_error("%s: x needs 32-byte, w_packed 128-byte, out 16-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return 0;
}

int e2f_modulated_deform_conv2d(const void* x, const float* offset, const float* mask, const void* w_packed,
                                const float* bias, void* out, int n, int h, int w, int cin, int cout,
                                int deform_groups, int out_dtype, int x_layout, void* stream) {
  int st = dcn_common_checks("e2f_modulated_deform_conv2d", x, w_packed, out, n, h, w, out_dtype);
  if (st) return st;
  if (!offset || !mask) { set_error("e2f_modulated_deform_conv2d: null offset/mask"); return E2F_ERR_BAD_ARG; }
  if (!aligned(offset, 16) || !aligned(mask, 16)) { set_error("e2f_modulated_deform_conv2d: offset / mask need 16-byte alignment"); return E2F_ERR_ALIGNMENT; }
  if (x_layout != E2F_X_NHWC && x_layout != E2F_X_GROUPED) { set_error("e2f_modulated_deform_conv2d: x_layout %d", x_layout); return E2F_ERR_BAD_ARG; }
  return finish(launch_dcn(x, offset, mask, nullptr, nullptr, nullptr, w_packed, bias, out, n, h, w, cin, cout,
                           deform_groups, 0.f, out_dtype, x_layout, static_cast<cudaStream_t>(stream)),
                "e2f_modulated_deform_conv2d");
}

int e2f_deform_align_fused(const void* x, const float* head, const float* flow1, const float* flow2,
                           const void* w_packed, const float* bias, void* out, int n, int h, int w, int cin, int cout,
                           int deform_groups, float max_residue, int out_dtype, int x_layout, void* stream) {
  int st = dcn_common_checks("e2f_deform_align_fused", x, w_packed, out, n, h, w, out_dtype);
  if (st) return st;
  if (!head || !flow1 || !flow2) { set_error("e2f_deform_align_fused: null head/flow"); return E2F_ERR_BAD_ARG; }
  if (!aligned(head, 16) || !aligned(flow1, 8) || !aligned(flow2, 8)) { set_error("e2f_deform_align_fused: head needs 16-byte, flow 8-byte alignment"); return E2F_ERR_ALIGNMENT; }
  if (x_layout != E2F_X_NHWC && x_layout != E2F_X_GROUPED) { set_error("e2f_deform_align_fused: x_layout %d", x_layout); return E2F_ERR_BAD_ARG; }
  return finish(launch_dcn(x, nullptr, nullptr, head, flow1, flow2, w_packed, bias, out, n, h, w, cin, cout,
                           deform_groups, max_residue, out_dtype, x_layout, static_cast<cudaStream_t>(stream)),
                "e2f_deform_align_fused");
}

int e2f_deform_align_fused_split(const void* x, const float* head, const float* flow1, const float* flow2,
                                 const void* w_packed, const float* bias, float* out, void* out_hi, void* out_lo, int n,
                                 int h, int w, int cin, int cout, int deform_groups, float max_residue, int x_layout,
                                 void* stream) {
  const char* who = "e2f_deform_align_fused_split";
  int st = dcn_common_checks(who, x, w_packed, out, n, h, w, E2F_F32);
  if (st) return st;
  if (!head || !flow1 || !flow2 || !out_hi || !out_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(head, 16) || !aligned(flow1, 8) || !aligned(flow2, 8) || !aligned(out_hi, 16) || !aligned(out_lo, 16)) { set_error("%s: head / out_hi / out_lo need 16-byte, flow 8-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  if (x_layout != E2F_X_NHWC && x_layout != E2F_X_GROUPED) { set_error("%s: x_layout %d", who, x_layout); return E2F_ERR_BAD_ARG; }
  return finish(launch_dcn(x, nullptr, nullptr, head, flow1, flow2, w_packed, bias, out, n, h, w, cin, cout,
                           deform_groups, max_residue, E2F_F32, x_layout, static_cast<cudaStream_t>(stream), out_hi, out_lo), who);
}

static int dcn_backward_shape_checks(const char* who, int n, int h, int w, int cin, int deform_groups) {
  if (n < 0 || h <= 0 || w <= 0) { set_error("%s: bad shape n=%d h=%d w=%d", who, n, h, w); return E2F_ERR_BAD_ARG; }
  if (cin != 256 || deform_groups != 16) { set_error("%s: specialised for Cin=256, deform_groups=16 (got %d, %d)", who, cin, deform_groups); return E2F_ERR_UNSUPPORTED; }
  if (static_cast<long long>(n) * h * w * 576 > INT_MAX) { set_error("%s: N*H*W=%lld too large (N*H*W*576 must fit in int)", who, static_cast<long long>(n) * h * w); return E2F_ERR_UNSUPPORTED; }
  return 0;
}

int64_t e2f_deform_align_backward_work_elems(int n, int h, int w, int cin, int deform_groups) {
  if (const int st = dcn_backward_shape_checks("e2f_deform_align_backward_work_elems", n, h, w, cin, deform_groups)) return st;
  return static_cast<int64_t>(dcn_backward_work_elems(n, h, w));
}

int e2f_deform_align_backward_sample(const void* x, const float* head, const float* flow1, const float* flow2,
                                     const float* da, float* dhead, float* dflow, void* a_hi, void* a_lo, void* work,
                                     int n, int h, int w, int cin, int deform_groups, float max_residue, void* stream) {
  const char* who = "e2f_deform_align_backward_sample";
  if (!x || !head || !flow1 || !flow2) { set_error("%s: null x/head/flow", who); return E2F_ERR_BAD_ARG; }
  if ((!a_hi) != (!a_lo)) { set_error("%s: a_hi and a_lo go together", who); return E2F_ERR_BAD_ARG; }
  if (!dhead && !a_hi && !work) { set_error("%s: nothing to compute (need dhead, a_hi/a_lo or the scatter workspace)", who); return E2F_ERR_BAD_ARG; }
  if (dhead && !da) { set_error("%s: dhead needs da", who); return E2F_ERR_BAD_ARG; }
  if (dflow && !dhead) { set_error("%s: dflow goes with dhead", who); return E2F_ERR_BAD_ARG; }
  if (const int st = dcn_backward_shape_checks(who, n, h, w, cin, deform_groups)) return st;
  if (!aligned(x, 32) || !aligned(head, 16) || !aligned(flow1, 8) || !aligned(flow2, 8) || (da && !aligned(da, 16)) ||
      (dhead && !aligned(dhead, 16)) || (dflow && !aligned(dflow, 16)) || (a_hi && (!aligned(a_hi, 16) || !aligned(a_lo, 16))) ||
      (work && !aligned(work, 256))) { set_error("%s: x needs 32-byte, head / da / dhead / dflow / a 16-byte, flow 8-byte, work 256-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dcn_sample_backward(x, head, flow1, flow2, da, dhead, dflow, a_hi, a_lo, work, n, h, w, max_residue,
                                           static_cast<cudaStream_t>(stream)), who);
}

int e2f_deform_align_backward_scatter(const float* da, void* work, float* dx, int n, int h, int w, int cin,
                                      int deform_groups, void* stream) {
  const char* who = "e2f_deform_align_backward_scatter";
  if (!da || !work || !dx) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (const int st = dcn_backward_shape_checks(who, n, h, w, cin, deform_groups)) return st;
  if (!aligned(da, 16) || !aligned(dx, 16) || !aligned(work, 256)) { set_error("%s: da / dx need 16-byte, work 256-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dcn_scatter_backward(da, work, dx, n, h, w, static_cast<cudaStream_t>(stream)), who);
}

int e2f_focal_window_attention(const void* qkv, const void* qkv_pooled, void* out, int b, int t, int h, int w,
                               int heads, int head_dim, int wh, int ww, int eh, int ew, int fh, int fw,
                               int use_pooled, float scale, int out_dtype, void* stream) {
  if (!qkv || !out || (use_pooled && !qkv_pooled)) { set_error("e2f_focal_window_attention: null pointer"); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || heads <= 0 || wh <= 0 || ww <= 0 || eh < 0 || ew < 0) { set_error("e2f_focal_window_attention: bad shape"); return E2F_ERR_BAD_ARG; }
  if (h % wh || w % ww) { set_error("e2f_focal_window_attention: token grid %dx%d is not a multiple of the window %dx%d", h, w, wh, ww); return E2F_ERR_BAD_ARG; }
  if (use_pooled && (fh <= 0 || fw <= 0 || !(fh & 1) || !(fw & 1))) { set_error("e2f_focal_window_attention: pooled neighbourhood %dx%d must be odd", fh, fw); return E2F_ERR_BAD_ARG; }
  if (out_dtype != E2F_F32 && out_dtype != E2F_F16 && out_dtype != E2F_SPLIT_BF16) { set_error("e2f_focal_window_attention: out_dtype %d", out_dtype); return E2F_ERR_BAD_ARG; }
  if (head_dim != 128) { set_error("e2f_focal_window_attention: head_dim %d unsupported (128 only)", head_dim); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(qkv, 16) || !aligned(out, 16) || (use_pooled && !aligned(qkv_pooled, 16))) { set_error("e2f_focal_window_attention: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_focal_attention(qkv, qkv_pooled, out, b, t, h, w, heads, head_dim, wh, ww, eh, ew, fh, fw,
                                       use_pooled, scale, out_dtype, static_cast<cudaStream_t>(stream)),
                "e2f_focal_window_attention");
}

static int focal_grad_geometry_checks(const char* who, int b, int t, int h, int w, int heads, int head_dim, int wh,
                                      int ww, int eh, int ew, int fh, int fw, int use_pooled) {
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || heads <= 0 || wh <= 0 || ww <= 0 || eh < 0 || ew < 0) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if (h % wh || w % ww) { set_error("%s: token grid %dx%d is not a multiple of the window %dx%d", who, h, w, wh, ww); return E2F_ERR_BAD_ARG; }
  if (use_pooled != 0 && use_pooled != 1) { set_error("%s: use_pooled %d", who, use_pooled); return E2F_ERR_BAD_ARG; }
  if (use_pooled && (fh <= 0 || fw <= 0 || !(fh & 1) || !(fw & 1))) { set_error("%s: pooled neighbourhood %dx%d must be odd", who, fh, fw); return E2F_ERR_BAD_ARG; }
  if (head_dim != 128) { set_error("%s: head_dim %d unsupported (128 only)", who, head_dim); return E2F_ERR_UNSUPPORTED; }
  return 0;
}

int64_t e2f_focal_window_attention_backward_work_elems(int b, int t, int h, int w, int heads, int head_dim, int wh,
                                                       int ww, int eh, int ew, int fh, int fw, int use_pooled) {
  const char* who = "e2f_focal_window_attention_backward_work_elems";
  if (const int st = focal_grad_geometry_checks(who, b, t, h, w, heads, head_dim, wh, ww, eh, ew, fh, fw, use_pooled)) return st;
  return static_cast<int64_t>(focal_attention_backward_work_elems(b, t, h, w, heads, wh, ww, eh, ew, fh, fw, use_pooled));
}

int e2f_focal_window_attention_key_sources(int t_count, int h, int w, int wh, int ww, int eh, int ew, int fh, int fw,
                                           int use_pooled, int t, int pooled, int y, int x, int* win, int* slot,
                                           int* mult, int cap) {
  const char* who = "e2f_focal_window_attention_key_sources";
  if (const int st = focal_grad_geometry_checks(who, 1, t_count, h, w, 1, 128, wh, ww, eh, ew, fh, fw, use_pooled)) return st;
  if (!win || !slot || !mult || cap <= 0) { set_error("%s: null pointer or cap %d", who, cap); return E2F_ERR_BAD_ARG; }
  if (t < 0 || t >= t_count || (pooled && !use_pooled) || y < 0 || x < 0 || y >= (pooled ? h / wh : h) || x >= (pooled ? w / ww : w)) { set_error("%s: key token (%d, %d, %d) outside the grid", who, t, y, x); return E2F_ERR_BAD_ARG; }
  return focal_attention_key_sources(t_count, h, w, wh, ww, eh, ew, fh, fw, use_pooled, t, pooled, y, x, win, slot, mult, cap);
}

int e2f_focal_window_attention_backward(const void* qkv, const void* qkv_pooled, const float* dout, float* dqkv,
                                        float* dqkv_pooled, float* work, int b, int t, int h, int w, int heads,
                                        int head_dim, int wh, int ww, int eh, int ew, int fh, int fw, int use_pooled,
                                        float scale, void* stream) {
  const char* who = "e2f_focal_window_attention_backward";
  if (!qkv || !dout || !dqkv || !work || (use_pooled && (!qkv_pooled || !dqkv_pooled))) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (const int st = focal_grad_geometry_checks(who, b, t, h, w, heads, head_dim, wh, ww, eh, ew, fh, fw, use_pooled)) return st;
  if (!(scale > 0.f)) { set_error("%s: scale must be positive", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(qkv, 16) || !aligned(dout, 16) || !aligned(dqkv, 16) || !aligned(work, 16) || (use_pooled && (!aligned(qkv_pooled, 16) || !aligned(dqkv_pooled, 16)))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_focal_attention_backward(qkv, qkv_pooled, dout, dqkv, dqkv_pooled, work, b, t, h, w, heads, wh, ww,
                                                eh, ew, fh, fw, use_pooled, scale, static_cast<cudaStream_t>(stream)), who);
}

int e2f_dcn_pack_input(const float* a, const float* b, void* xg, int n, int h, int w, int ca, int cb, void* stream) {
  if (!a || !b || !xg) { set_error("e2f_dcn_pack_input: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || ca <= 0 || cb <= 0 || ca % 16 || cb % 16) { set_error("e2f_dcn_pack_input: bad shape (channels must be multiples of 16)"); return E2F_ERR_BAD_ARG; }
  if (!aligned(a, 16) || !aligned(b, 16) || !aligned(xg, 16)) { set_error("e2f_dcn_pack_input: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dcn_pack_input(a, b, xg, n, h, w, ca, cb, static_cast<cudaStream_t>(stream)), "e2f_dcn_pack_input");
}

static int t2t_checks(const char* who, const void* a, const void* b, int bt, int c, int h, int w, int k, int s, int p) {
  if (!a || !b) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (bt < 0 || c <= 0 || h <= 0 || w <= 0 || k <= 0 || s <= 0 || p < 0 || h + 2 * p < k || w + 2 * p < k) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if ((c * k * k) % 4) { set_error("%s: C*k*k=%d must be a multiple of 4", who, c * k * k); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(a, 16) || !aligned(b, 16)) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  return 0;
}

int e2f_t2t_unfold(const float* img, float* tokens, void* tokens_hi, void* tokens_lo, int bt, int c, int h, int w, int k,
                   int stride, int pad, int gelu, void* stream) {
  if ((!tokens && !tokens_hi) || (!tokens_hi) != (!tokens_lo)) { set_error("e2f_t2t_unfold: need tokens and/or both of tokens_hi/tokens_lo"); return E2F_ERR_BAD_ARG; }
  int st = t2t_checks("e2f_t2t_unfold", img, tokens ? static_cast<const void*>(tokens) : tokens_hi, bt, c, h, w, k, stride, pad);
  if (st) return st;
  if (tokens_hi && (!aligned(tokens_hi, 16) || !aligned(tokens_lo, 16))) { set_error("e2f_t2t_unfold: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_t2t_unfold(img, tokens, tokens_hi, tokens_lo, bt, c, h, w, k, stride, pad, gelu, 0, static_cast<cudaStream_t>(stream)), "e2f_t2t_unfold");
}

int e2f_t2t_unfold_nhwc(const float* img_nhwc, float* tokens, void* tokens_hi, void* tokens_lo, int bt, int c, int h, int w,
                        int k, int stride, int pad, int gelu, void* stream) {
  if ((!tokens && !tokens_hi) || (!tokens_hi) != (!tokens_lo)) { set_error("e2f_t2t_unfold_nhwc: need tokens and/or both of tokens_hi/tokens_lo"); return E2F_ERR_BAD_ARG; }
  int st = t2t_checks("e2f_t2t_unfold_nhwc", img_nhwc, tokens ? static_cast<const void*>(tokens) : tokens_hi, bt, c, h, w, k, stride, pad);
  if (st) return st;
  if (tokens_hi && (!aligned(tokens_hi, 16) || !aligned(tokens_lo, 16))) { set_error("e2f_t2t_unfold_nhwc: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  st = launch_t2t_unfold(img_nhwc, tokens, tokens_hi, tokens_lo, bt, c, h, w, k, stride, pad, gelu, 1, static_cast<cudaStream_t>(stream));
  if (st == E2F_ERR_UNSUPPORTED) { set_error("e2f_t2t_unfold_nhwc: channels_last input needs k=7 stride=3 pad=3 and C %% 8 == 0 (k=%d s=%d p=%d c=%d)", k, stride, pad, c); return st; }
  return finish(st, "e2f_t2t_unfold_nhwc");
}

int e2f_t2t_fold_unfold(const float* tokens_in, float* tokens, void* tokens_hi, void* tokens_lo, int bt, int c, int h,
                        int w, int k, int stride, int pad, int gelu, int out_pitch, void* stream) {
  if ((!tokens && !tokens_hi) || (!tokens_hi) != (!tokens_lo)) { set_error("e2f_t2t_fold_unfold: need tokens and/or both of tokens_hi/tokens_lo"); return E2F_ERR_BAD_ARG; }
  int st = t2t_checks("e2f_t2t_fold_unfold", tokens_in, tokens ? static_cast<const void*>(tokens) : tokens_hi, bt, c, h, w, k, stride, pad);
  if (st) return st;
  if (tokens_hi && (!aligned(tokens_hi, 16) || !aligned(tokens_lo, 16))) { set_error("e2f_t2t_fold_unfold: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  if (out_pitch == 0) out_pitch = c * k * k;
  if (out_pitch < c * k * k || out_pitch % 4) { set_error("e2f_t2t_fold_unfold: out_pitch=%d must be 0 or a multiple of 4 >= C*k*k=%d", out_pitch, c * k * k); return E2F_ERR_BAD_ARG; }
  st = launch_t2t_fold_unfold(tokens_in, tokens, tokens_hi, tokens_lo, bt, c, h, w, k, stride, pad, gelu, out_pitch, static_cast<cudaStream_t>(stream));
  if (st == E2F_ERR_UNSUPPORTED) { set_error("e2f_t2t_fold_unfold: only k=7 stride=3 pad=3, C %% 4 == 0, bt <= 65535 and W <= 1800 are fused (k=%d s=%d p=%d c=%d w=%d); compose e2f_t2t_fold + e2f_t2t_unfold", k, stride, pad, c, w); return st; }
  return finish(st, "e2f_t2t_fold_unfold");
}

int e2f_t2t_fold_unfold_train(const float* tokens_in, float* u, float* tokens, void* tokens_hi, void* tokens_lo, int bt, int c,
                              int h, int w, int k, int stride, int pad, int backward, int out_pitch, void* stream) {
  const char* who = "e2f_t2t_fold_unfold_train";
  if ((!tokens && !tokens_hi) || (!tokens_hi) != (!tokens_lo)) { set_error("%s: need tokens and/or both of tokens_hi/tokens_lo", who); return E2F_ERR_BAD_ARG; }
  if (!u) { set_error("%s: null u", who); return E2F_ERR_BAD_ARG; }
  if (backward != 0 && backward != 1) { set_error("%s: backward=%d (0 or 1)", who, backward); return E2F_ERR_BAD_ARG; }
  int st = t2t_checks(who, tokens_in, tokens ? static_cast<const void*>(tokens) : tokens_hi, bt, c, h, w, k, stride, pad);
  if (st) return st;
  if (!aligned(u, 16) || (tokens_hi && (!aligned(tokens_hi, 16) || !aligned(tokens_lo, 16)))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  if (out_pitch == 0) out_pitch = c * k * k;
  if (out_pitch < c * k * k || out_pitch % 4) { set_error("%s: out_pitch=%d must be 0 or a multiple of 4 >= C*k*k=%d", who, out_pitch, c * k * k); return E2F_ERR_BAD_ARG; }
  if (k != 7 || stride != 3 || pad != 3 || c % 4 || bt > 65535) { set_error("%s: only k=7 stride=3 pad=3 with C %% 4 == 0 and bt <= 65535 (k=%d s=%d p=%d c=%d)", who, k, stride, pad, c); return E2F_ERR_UNSUPPORTED; }
  st = launch_t2t_fold_unfold(tokens_in, tokens, tokens_hi, tokens_lo, bt, c, h, w, k, stride, pad, 1, out_pitch,
                              static_cast<cudaStream_t>(stream), backward ? u : nullptr, backward ? nullptr : u);
  if (st == E2F_ERR_UNSUPPORTED) { set_error("%s: the image (w=%d) does not fit the fused kernel's shared memory", who, w); return st; }
  return finish(st, who);
}

int e2f_layernorm_pool_split(const float* x, const float* gamma, const float* beta, const float* pool_w,
                             const float* pool_b, void* out_hi, void* out_lo, int bt, int h, int w, int c, int wh, int ww,
                             float eps, void* stream) {
  const char* who = "e2f_layernorm_pool_split";
  if (!x || !gamma || !beta || !pool_w || !out_hi || !out_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (bt < 0 || h <= 0 || w <= 0 || c <= 0 || wh <= 0 || ww <= 0 || h % wh || w % ww) { set_error("%s: bad shape bt=%d h=%d w=%d c=%d window=%dx%d", who, bt, h, w, c, wh, ww); return E2F_ERR_BAD_ARG; }
  if (!aligned(x, 16) || !aligned(out_hi, 16) || !aligned(out_lo, 16) || !aligned(gamma, 4) || !aligned(beta, 4)) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_layernorm_pool_split(x, gamma, beta, pool_w, pool_b, out_hi, out_lo, bt, h, w, c, wh, ww, eps, static_cast<cudaStream_t>(stream)), who);
}

int e2f_window_pool(const void* x_hi, const void* x_lo, const float* weight, const float* bias, float* out, void* out_hi,
                    void* out_lo, int bt, int h, int w, int c, int wh, int ww, void* stream) {
  if (!x_hi || !x_lo || !weight) { set_error("e2f_window_pool: null pointer"); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("e2f_window_pool: need out and/or both of out_hi/out_lo"); return E2F_ERR_BAD_ARG; }
  if (bt < 0 || h <= 0 || w <= 0 || c <= 0 || wh <= 0 || ww <= 0) { set_error("e2f_window_pool: bad shape"); return E2F_ERR_BAD_ARG; }
  if (h % wh || w % ww) { set_error("e2f_window_pool: token grid %dx%d is not a multiple of the window %dx%d", h, w, wh, ww); return E2F_ERR_BAD_ARG; }
  if (c % 8 || wh > 8 || static_cast<size_t>(wh) * c * 4 > 48 * 1024 || bt > 65535) { set_error("e2f_window_pool: needs C %% 8 == 0, wh <= 8, wh*C <= 12288, bt <= 65535 (c=%d wh=%d bt=%d)", c, wh, bt); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(x_hi, 16) || !aligned(x_lo, 16) || (out && !aligned(out, 16)) || (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16)))) { set_error("e2f_window_pool: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_window_pool(x_hi, x_lo, weight, bias, out, out_hi, out_lo, bt, h, w, c, wh, ww, static_cast<cudaStream_t>(stream)), "e2f_window_pool");
}

int e2f_upsample2x_split(const float* x, void* out_hi, void* out_lo, int n, int h, int w, int c, void* stream) {
  if (!x || !out_hi || !out_lo) { set_error("e2f_upsample2x_split: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c <= 0) { set_error("e2f_upsample2x_split: bad shape"); return E2F_ERR_BAD_ARG; }
  if (c % 8) { set_error("e2f_upsample2x_split: C=%d must be a multiple of 8", c); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(x, 32) || !aligned(out_hi, 16) || !aligned(out_lo, 16)) { set_error("e2f_upsample2x_split: x needs 32-byte, out_hi / out_lo 16-byte alignment"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_upsample2x_split(x, out_hi, out_lo, n, h, w, c, static_cast<cudaStream_t>(stream)), "e2f_upsample2x_split");
}

int e2f_layernorm_split(const float* x, const float* gamma, const float* beta, float* out, void* out_hi, void* out_lo,
                        int64_t rows, int c, float eps, void* stream) {
  if (!x || !gamma || !beta) { set_error("e2f_layernorm_split: null pointer"); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("e2f_layernorm_split: need out and/or both of out_hi/out_lo"); return E2F_ERR_BAD_ARG; }
  if (rows < 0 || c <= 0) { set_error("e2f_layernorm_split: bad shape"); return E2F_ERR_BAD_ARG; }
  if (!aligned(x, 16) || (out && !aligned(out, 16)) || (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16)))) { set_error("e2f_layernorm_split: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_layernorm_split(x, gamma, beta, out, out_hi, out_lo, rows, c, eps, static_cast<cudaStream_t>(stream)), "e2f_layernorm_split");
}

int64_t e2f_layernorm_backward_work_elems(int64_t rows, int c) {
  if (rows < 0 || c != 512) { set_error("e2f_layernorm_backward_work_elems: rows=%lld c=%d (512 channels only)", static_cast<long long>(rows), c); return c != 512 && rows >= 0 ? E2F_ERR_UNSUPPORTED : E2F_ERR_BAD_ARG; }
  return static_cast<int64_t>(layernorm_backward_work_elems(rows));
}

int e2f_layernorm_backward(const float* x, const float* dy, const float* gamma, const float* residual, float* dx,
                           void* dx_hi, void* dx_lo, float* dgamma, float* dbeta, float* work, int64_t rows, int c,
                           float eps, void* stream) {
  const char* who = "e2f_layernorm_backward";
  const bool params = dgamma || dbeta;
  if (!x || !dy || !gamma) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!dx && !dx_hi && !params) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dx, both of dx_hi/dx_lo, or a parameter gradient", who); return E2F_ERR_BAD_ARG; }
  if (params && !work && rows > 0) { set_error("%s: null workspace (e2f_layernorm_backward_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (rows < 0 || c <= 0) { set_error("%s: bad shape rows=%lld c=%d", who, static_cast<long long>(rows), c); return E2F_ERR_BAD_ARG; }
  if (c != 512) { set_error("%s: specialised for 512 channels (got %d)", who, c); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(x, 16) || !aligned(dy, 16) || (residual && !aligned(residual, 16)) || (dx && !aligned(dx, 16)) || (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16))) || !aligned(gamma, 4) || (dgamma && !aligned(dgamma, 4)) || (dbeta && !aligned(dbeta, 4)) || (work && !aligned(work, 16))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_layernorm_backward(x, dy, gamma, residual, dx, dx_hi, dx_lo, dgamma, dbeta, params ? work : nullptr, rows, c, eps, static_cast<cudaStream_t>(stream)), who);
}

static int layernorm_pool_geometry_checks(const char* who, int bt, int h, int w, int c, int wh, int ww) {
  if (bt < 0 || h <= 0 || w <= 0 || c <= 0 || wh <= 0 || ww <= 0) { set_error("%s: bad shape bt=%d h=%d w=%d c=%d window=%dx%d", who, bt, h, w, c, wh, ww); return E2F_ERR_BAD_ARG; }
  if (h % wh || w % ww) { set_error("%s: token grid %dx%d is not a multiple of the window %dx%d", who, h, w, wh, ww); return E2F_ERR_BAD_ARG; }
  if (c != 512) { set_error("%s: specialised for 512 channels (got %d)", who, c); return E2F_ERR_UNSUPPORTED; }
  if (bt > 65535) { set_error("%s: at most 65535 frames per launch (got %d)", who, bt); return E2F_ERR_UNSUPPORTED; }
  return 0;
}

int64_t e2f_layernorm_pool_backward_work_elems(int bt, int h, int w, int c, int wh, int ww) {
  if (const int st = layernorm_pool_geometry_checks("e2f_layernorm_pool_backward_work_elems", bt, h, w, c, wh, ww)) return st;
  return static_cast<int64_t>(layernorm_pool_backward_work_elems(bt, h, w, wh, ww));
}

int e2f_layernorm_pool_backward(const float* x, const float* gamma, const float* beta, const float* pool_w,
                                const float* drows, const float* dx1, float* dx, float* dgamma, float* dbeta,
                                float* dpool_w, float* dpool_b, float* work, int bt, int h, int w, int c, int wh, int ww,
                                float eps, void* stream) {
  const char* who = "e2f_layernorm_pool_backward";
  const bool params = dgamma || dbeta || dpool_w || dpool_b;
  if (!x || !gamma || !beta || !pool_w || !drows) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (!dx && !params) { set_error("%s: need dx or a parameter gradient", who); return E2F_ERR_BAD_ARG; }
  if (dx && !dx1) { set_error("%s: dx needs dx1", who); return E2F_ERR_BAD_ARG; }
  if (params && !work && bt > 0) { set_error("%s: null workspace (e2f_layernorm_pool_backward_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (const int st = layernorm_pool_geometry_checks(who, bt, h, w, c, wh, ww)) return st;
  if (!aligned(x, 16) || !aligned(drows, 16) || (dx && (!aligned(dx, 16) || !aligned(dx1, 16))) || !aligned(gamma, 4) || !aligned(beta, 4) || !aligned(pool_w, 4) || (work && !aligned(work, 16))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_layernorm_pool_backward(x, gamma, beta, pool_w, drows, dx1, dx, dgamma, dbeta, dpool_w, dpool_b, params ? work : nullptr, bt, h, w, c, wh, ww, eps, static_cast<cudaStream_t>(stream)), who);
}

int e2f_t2t_fold(const float* tokens, const float* bias, float* img, int bt, int c, int h, int w, int k, int stride,
                 int pad, int normalize, void* stream) {
  int st = t2t_checks("e2f_t2t_fold", tokens, img, bt, c, h, w, k, stride, pad);
  if (st) return st;
  return finish(launch_t2t_fold(tokens, bias, img, bt, c, h, w, k, stride, pad, normalize, static_cast<cudaStream_t>(stream)), "e2f_t2t_fold");
}

int e2f_t2t_fold_nhwc(const float* tokens, const float* bias, const float* residual_nhwc, float* img_nhwc, int bt, int c,
                      int h, int w, int k, int stride, int pad, int normalize, void* stream) {
  int st = t2t_checks("e2f_t2t_fold_nhwc", tokens, img_nhwc, bt, c, h, w, k, stride, pad);
  if (st) return st;
  if (residual_nhwc && !aligned(residual_nhwc, 16)) { set_error("e2f_t2t_fold_nhwc: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  st = launch_t2t_fold_nhwc(tokens, bias, residual_nhwc, img_nhwc, bt, c, h, w, k, stride, pad, normalize, static_cast<cudaStream_t>(stream));
  if (st == E2F_ERR_UNSUPPORTED) { set_error("e2f_t2t_fold_nhwc: needs k=7 stride=3 pad=3, C %% 8 == 0, bt <= 65535 (k=%d s=%d p=%d c=%d)", k, stride, pad, c); return st; }
  return finish(st, "e2f_t2t_fold_nhwc");
}

int e2f_split_bf16(const float* x, void* hi_bf16, void* lo_bf16, int64_t n, void* stream) {
  if (!x || !hi_bf16 || !lo_bf16) { set_error("e2f_split_bf16: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || n % 8) { set_error("e2f_split_bf16: n=%lld must be a non-negative multiple of 8", static_cast<long long>(n)); return E2F_ERR_BAD_ARG; }
  if (!aligned(x, 16) || !aligned(hi_bf16, 16) || !aligned(lo_bf16, 16)) { set_error("e2f_split_bf16: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_split_bf16(x, hi_bf16, lo_bf16, n, static_cast<cudaStream_t>(stream)), "e2f_split_bf16");
}

int e2f_linear_bf16x3(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                      const float* residual, void* out, int m, int n, int k, int out_dtype, int tile_hint,
                      void* stream) {
  if (!a_hi || !a_lo || !w_hi || !w_lo || !out) { set_error("e2f_linear_bf16x3: null pointer"); return E2F_ERR_BAD_ARG; }
  if (m < 0 || n <= 0 || k <= 0) { set_error("e2f_linear_bf16x3: bad shape m=%d n=%d k=%d", m, n, k); return E2F_ERR_BAD_ARG; }
  if (out_dtype != E2F_F32 && out_dtype != E2F_F16) { set_error("e2f_linear_bf16x3: out_dtype %d", out_dtype); return E2F_ERR_BAD_ARG; }
  if (tile_hint != 0 && tile_hint != 128 && tile_hint != 256) { set_error("e2f_linear_bf16x3: tile_hint %d", tile_hint); return E2F_ERR_BAD_ARG; }
  if (k % 8 || n % (out_dtype == E2F_F16 ? 8 : 4)) { set_error("e2f_linear_bf16x3: K %% 8 and N %% %d must be 0 (k=%d n=%d)", out_dtype == E2F_F16 ? 8 : 4, k, n); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(a_hi, 16) || !aligned(a_lo, 16) || !aligned(w_hi, 16) || !aligned(w_lo, 16) || !aligned(out, 16) || (residual && !aligned(residual, 16))) { set_error("e2f_linear_bf16x3: 16-byte alignment required"); return E2F_ERR_ALIGNMENT; }
  // every tile_hint runs the ping-pong kernel's 128 x 128 tiles
  return finish(launch_linear_bf16x3(a_hi, a_lo, w_hi, w_lo, bias, residual, out, m, n, k, out_dtype, static_cast<cudaStream_t>(stream)), "e2f_linear_bf16x3");
}

int e2f_conv2d_rows_bf16x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                           int in_rows, const void* w_hi, const void* w_lo, const float* bias, const float* residual,
                           float* out, void* out_hi, void* out_lo, int out_lead, int n, int h, int w, int cout, int groups,
                           float leaky_slope, int ksize, int stride, int pad, void* stream) {
  const char* who = "e2f_conv2d_bf16x3";
  if (!src_hi || !src_lo || !src_channels || !w_hi || !w_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (out_hi && cout % 8) { set_error("%s: split output needs Cout %% 8 == 0", who); return E2F_ERR_UNSUPPORTED; }
  if (nsrc < 1 || nsrc > 4) { set_error("%s: nsrc=%d (1..4 supported)", who, nsrc); return E2F_ERR_UNSUPPORTED; }
  if (n < 0 || h <= 0 || w <= 0 || cout <= 0 || groups <= 0 || cout % groups) { set_error("%s: bad shape n=%d h=%d w=%d cout=%d groups=%d", who, n, h, w, cout, groups); return E2F_ERR_BAD_ARG; }
  if (ksize < 1 || ksize > 7 || (stride != 1 && stride != 2) || pad < 0 || h + 2 * pad < ksize || w + 2 * pad < ksize) { set_error("%s: unsupported geometry k=%d stride=%d pad=%d", who, ksize, stride, pad); return E2F_ERR_UNSUPPORTED; }
  if (out_lead < 0 || out_lead > 8 || (out_lead && !out_hi)) { set_error("%s: out_lead=%d needs a split output and 0..8", who, out_lead); return E2F_ERR_BAD_ARG; }
  if (out_lead && groups != 1) { set_error("%s: row-gapped output needs groups == 1", who); return E2F_ERR_UNSUPPORTED; }
  if (in_rows) {
    const int cin = src_channels[0];
    const bool pow2 = cin == 4 || cin == 8 || cin == 16 || cin == 32;
    if (nsrc != 1 || groups != 1 || !pow2 || (stride * cin * 2) % 16 || (ksize > 64 / cin && (64 / cin) % stride)) {
      set_error("%s: window-packed input needs one source, groups == 1, cin in {4,8,16,32} with stride*cin*2 %% 16 == 0 (nsrc=%d groups=%d cin=%d stride=%d)", who, nsrc, groups, cin, stride);
      return E2F_ERR_UNSUPPORTED;
    }
  }
  for (int i = 0; i < nsrc; ++i) {
    if (!src_hi[i] || !src_lo[i]) { set_error("%s: null source %d", who, i); return E2F_ERR_BAD_ARG; }
    if (!in_rows && (src_channels[i] <= 0 || src_channels[i] % 8 || src_channels[i] % groups)) { set_error("%s: source %d has %d channels (needs a multiple of 8 and of groups)", who, i, src_channels[i]); return E2F_ERR_UNSUPPORTED; }
    if (!aligned(src_hi[i], 16) || !aligned(src_lo[i], 16)) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  }
  if (!aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) || (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (residual && !aligned(residual, 16))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  return finish(launch_conv3x3(nsrc, src_hi, src_lo, src_channels, w_hi, w_lo, bias, residual, out, out_hi, out_lo, n, h, w, cout, groups, leaky_slope, ksize, stride, pad, in_rows ? 1 : 0, out_lead, static_cast<cudaStream_t>(stream)), who);
}

int e2f_conv_gather_bf16x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                           const void* w_hi, const void* w_lo, const float* bias, const float* bias_map,
                           const float* residual, float* out, void* out_hi, void* out_lo, int n, int h_in, int w_in,
                           int cout, float leaky_slope, int stride, int grid_h, int grid_w, int tile_w, int tile_h,
                           int ntaps, const int8_t* tap_dy, const int8_t* tap_dx, int nphase, const uint8_t* ph_tap0,
                           const uint8_t* ph_oy, const uint8_t* ph_ox, int ostep, int out_h, int out_w,
                           const int64_t* src_nstride, int64_t out_nstride, void* stream) {
  const char* who = "e2f_conv_gather_bf16x3";
  if (out_nstride < 0) { set_error("%s: negative out_nstride", who); return E2F_ERR_BAD_ARG; }
  if (!src_hi || !src_lo || !src_channels || !w_hi || !w_lo || !tap_dy || !tap_dx || !ph_tap0 || !ph_oy || !ph_ox) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (out_hi && cout % 8) { set_error("%s: split output needs Cout %% 8 == 0", who); return E2F_ERR_UNSUPPORTED; }
  if (nsrc < 1 || nsrc > 4) { set_error("%s: nsrc=%d (1..4 supported)", who, nsrc); return E2F_ERR_UNSUPPORTED; }
  if (n < 0 || h_in <= 0 || w_in <= 0 || cout <= 0 || grid_h <= 0 || grid_w <= 0 || out_h <= 0 || out_w <= 0) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if (stride < 1 || stride > 8 || ntaps < 1 || ntaps > 64 || nphase < 1 || nphase > 9 || ostep < 1 || ostep > 8 || tile_w < 1 || tile_h < 1 || tile_w * tile_h > 128) { set_error("%s: unsupported geometry stride=%d taps=%d phases=%d ostep=%d tile=%dx%d", who, stride, ntaps, nphase, ostep, tile_w, tile_h); return E2F_ERR_UNSUPPORTED; }
  if (ph_tap0[0] != 0 || ph_tap0[nphase] != ntaps) { set_error("%s: ph_tap0 must start at 0 and end at ntaps", who); return E2F_ERR_BAD_ARG; }
  for (int i = 0; i < nphase; ++i) {
    if (ph_tap0[i] >= ph_tap0[i + 1] || ph_oy[i] >= ostep || ph_ox[i] >= ostep) { set_error("%s: phase %d is empty or its offset exceeds ostep", who, i); return E2F_ERR_BAD_ARG; }
  }
  for (int i = 0; i < nsrc; ++i) {
    if (!src_hi[i] || !src_lo[i]) { set_error("%s: null source %d", who, i); return E2F_ERR_BAD_ARG; }
    if (src_channels[i] <= 0 || src_channels[i] % 8) { set_error("%s: source %d has %d channels (needs a multiple of 8)", who, i, src_channels[i]); return E2F_ERR_UNSUPPORTED; }
    if (!aligned(src_hi[i], 16) || !aligned(src_lo[i], 16)) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  }
  if (!aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) || (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (residual && !aligned(residual, 16)) || (bias_map && !aligned(bias_map, 16))) { set_error("%s: 16-byte alignment required", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  ConvGeom g;
  g.grid_h = grid_h; g.grid_w = grid_w; g.out_h = out_h; g.out_w = out_w; g.tile_w = tile_w; g.tile_h = tile_h;
  g.ntaps = ntaps; g.nphase = nphase; g.ostep = ostep; g.tap_dy = tap_dy; g.tap_dx = tap_dx; g.ph_tap0 = ph_tap0;
  g.ph_oy = ph_oy; g.ph_ox = ph_ox; g.bias_map = bias_map;
  long long sn[4] = {0, 0, 0, 0};
  for (int i = 0; src_nstride && i < nsrc; ++i) sn[i] = static_cast<long long>(src_nstride[i]);
  g.src_nstride = src_nstride ? sn : nullptr;
  g.out_nstride = static_cast<long long>(out_nstride);
  return finish(launch_conv3x3(nsrc, src_hi, src_lo, src_channels, w_hi, w_lo, bias, residual, out, out_hi, out_lo, n, h_in, w_in, cout, 1, leaky_slope, 0, stride, 0, 0, 0, static_cast<cudaStream_t>(stream), &g), who);
}

int e2f_conv3x3_tanh_nchw(const void* src_hi, const void* src_lo, int cin, const void* w_hi, const void* w_lo,
                          const float* bias, float* out, int n, int h, int w, int cout, void* stream) {
  const char* who = "e2f_conv3x3_tanh_nchw";
  if (!src_hi || !src_lo || !w_hi || !w_lo || !out) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || cin <= 0 || cin % 8 || cout <= 0 || cout > 32 || (cout & 3) == 0) { set_error("%s: bad shape n=%d h=%d w=%d cin=%d cout=%d (cin %% 8 == 0, cout <= 32 and not a multiple of 4)", who, n, h, w, cin, cout); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(src_hi, 16) || !aligned(src_lo, 16) || !aligned(w_hi, 16) || !aligned(w_lo, 16) || !aligned(out, 4)) { set_error("%s: alignment", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  const void* hi[1] = {src_hi};
  const void* lo[1] = {src_lo};
  const int ch[1] = {cin};
  return finish(launch_conv3x3(1, hi, lo, ch, w_hi, w_lo, bias, nullptr, out, nullptr, nullptr, n, h, w, cout, 1, 1.0f, 3, 1, 1, 0, 0, static_cast<cudaStream_t>(stream), nullptr, 3), who);
}

int e2f_conv_kxn_bf16x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                        const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* out, void* out_hi,
                        void* out_lo, int n, int h, int w, int cout, int groups, int co_pad, int ksize, float leaky_slope,
                        int flags, void* stream) {
  const char* who = "e2f_conv_kxn_bf16x3";
  if (!src_hi || !src_lo || !src_channels || !w_hi || !w_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (nsrc < 1 || nsrc > 2) { set_error("%s: nsrc=%d (1..2 supported)", who, nsrc); return E2F_ERR_UNSUPPORTED; }
  if (n < 0 || h <= 0 || w <= 0 || cout <= 0 || groups <= 0) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if (flags & ~3) { set_error("%s: flags %d", who, flags); return E2F_ERR_BAD_ARG; }
  if ((flags & 2) && (!out || out_hi)) { set_error("%s: the NCHW store goes with an fp32-only output", who); return E2F_ERR_BAD_ARG; }
  for (int i = 0; i < nsrc; ++i) {
    if (!src_hi[i] || !src_lo[i]) { set_error("%s: null source %d", who, i); return E2F_ERR_BAD_ARG; }
    if (!aligned(src_hi[i], 16) || !aligned(src_lo[i], 16)) { set_error("%s: alignment", who); return E2F_ERR_ALIGNMENT; }
  }
  if (!aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) ||
      (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (residual && !aligned(residual, 8))) { set_error("%s: alignment", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  return finish(launch_conv_kxn(nsrc, src_hi, src_lo, src_channels, w_hi, w_lo, bias, residual, out, out_hi, out_lo, n, h, w, cout,
                                groups, co_pad, ksize, leaky_slope, flags, static_cast<cudaStream_t>(stream)), who);
}

int e2f_conv2d_bf16x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                      const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* out,
                      void* out_hi, void* out_lo, int n, int h, int w, int cout, int groups, float leaky_slope, int ksize,
                      int stride, int pad, void* stream) {
  return e2f_conv2d_rows_bf16x3(nsrc, src_hi, src_lo, src_channels, 0, w_hi, w_lo, bias, residual, out, out_hi, out_lo, 0, n,
                                h, w, cout, groups, leaky_slope, ksize, stride, pad, stream);
}

int e2f_conv_rows_pitch(int w, int lead, int channels) { return (w <= 0 || lead < 0 || channels <= 0) ? E2F_ERR_BAD_ARG : conv_rows_pitch(w, lead, channels); }

int e2f_conv_rows_tail(int lead, int channels) { return (lead < 0 || channels <= 0) ? E2F_ERR_BAD_ARG : conv_rows_tail(lead, channels); }

int e2f_pack_rows_bf16(const float* x, void* out_hi, void* out_lo, int n, int c, int h, int w, int cin, int lead,
                       void* stream) {
  if (!x || !out_hi || !out_lo) { set_error("e2f_pack_rows_bf16: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || c <= 0 || h <= 0 || w <= 0 || lead < 0 || lead > 8) { set_error("e2f_pack_rows_bf16: bad shape"); return E2F_ERR_BAD_ARG; }
  if ((cin != 4 && cin != 8 && cin != 16 && cin != 32) || c > cin) { set_error("e2f_pack_rows_bf16: cin=%d must be 4, 8, 16 or 32 and >= C=%d", cin, c); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(x, 4) || !aligned(out_hi, 16) || !aligned(out_lo, 16)) { set_error("e2f_pack_rows_bf16: alignment"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_pack_rows(x, out_hi, out_lo, n, c, h, w, cin, lead, static_cast<cudaStream_t>(stream)), "e2f_pack_rows_bf16");
}

int e2f_conv3x3_bf16x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                       const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* out,
                       void* out_hi, void* out_lo, int n, int h, int w, int cout, int groups, float leaky_slope,
                       void* stream) {
  return e2f_conv2d_bf16x3(nsrc, src_hi, src_lo, src_channels, w_hi, w_lo, bias, residual, out, out_hi, out_lo, n, h, w,
                           cout, groups, leaky_slope, 3, 1, 1, stream);
}

int e2f_prop_prologue(const float* prop, const float* feat_n2, const float* flow_n1, int64_t flow_n1_bstride,
                      const float* flow_prev, int64_t flow_prev_bstride, void* cond1_hi, void* cond1_lo, void* cond2_hi,
                      void* cond2_lo, float* flow1_out, float* flow2_out, void* flows_hi, void* flows_lo, void* x_grouped,
                      int n, int h, int w, int c, void* stream) {
  if (!prop || !flow_n1 || !cond1_hi || !cond1_lo || !cond2_hi || !cond2_lo || !flow1_out || !flow2_out || !flows_hi ||
      !flows_lo || !x_grouped) { set_error("e2f_prop_prologue: null pointer"); return E2F_ERR_BAD_ARG; }
  if ((feat_n2 == nullptr) != (flow_prev == nullptr)) { set_error("e2f_prop_prologue: feat_n2 and flow_prev must both be given or both be NULL"); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c <= 0 || c % 16) { set_error("e2f_prop_prologue: bad shape n=%d h=%d w=%d c=%d (C must be a multiple of 16)", n, h, w, c); return E2F_ERR_BAD_ARG; }
  if (!aligned(prop, 16) || (feat_n2 && !aligned(feat_n2, 16)) || !aligned(cond1_hi, 8) || !aligned(cond1_lo, 8) || !aligned(cond2_hi, 8) ||
      !aligned(cond2_lo, 8) || !aligned(flow1_out, 8) || !aligned(flow2_out, 8) || !aligned(flows_hi, 16) || !aligned(flows_lo, 16) ||
      !aligned(x_grouped, 16)) { set_error("e2f_prop_prologue: alignment"); return E2F_ERR_ALIGNMENT; }
  return finish(launch_prop_prologue(prop, feat_n2, flow_n1, static_cast<long long>(flow_n1_bstride), flow_prev,
                                     static_cast<long long>(flow_prev_bstride), cond1_hi, cond1_lo, cond2_hi, cond2_lo, flow1_out,
                                     flow2_out, flows_hi, flows_lo, x_grouped, n, h, w, c, static_cast<cudaStream_t>(stream)),
                "e2f_prop_prologue");
}

int e2f_spynet_pyramid(const float* frames, float* pyramid, int b, int t, int l_t, int H, int W, int h, int w, int h_up,
                       int w_up, const float* mean3, const float* std3, void* stream) {
  const char* who = "e2f_spynet_pyramid";
  if (!frames || !pyramid || !mean3 || !std3) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || l_t <= 0 || l_t > t || H <= 0 || W <= 0 || h <= 1 || w <= 1 || h > H || w > W) { set_error("%s: bad shape b=%d t=%d l_t=%d %dx%d -> %dx%d", who, b, t, l_t, H, W, h, w); return E2F_ERR_BAD_ARG; }
  if (h_up < h || w_up < w || h_up % 32 || w_up % 32) { set_error("%s: the working size %dx%d must be multiples of 32 >= %dx%d", who, h_up, w_up, h, w); return E2F_ERR_BAD_ARG; }
  return finish(launch_spynet_pyramid(frames, pyramid, b, t, l_t, H, W, h, w, h_up, w_up, mean3, std3, static_cast<cudaStream_t>(stream)), who);
}

int e2f_spynet_level_input(const float* level_img, const float* prev_flow, void* rows_hi, void* rows_lo, float* flow_up,
                           int b, int l_t, int hk, int wk, int lead, void* stream) {
  const char* who = "e2f_spynet_level_input";
  if (!level_img || !rows_hi || !rows_lo || !flow_up) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || l_t < 2 || hk <= 0 || wk <= 0 || lead < 0 || lead > 8 || (prev_flow && ((hk | wk) & 1))) { set_error("%s: bad shape b=%d l_t=%d %dx%d lead=%d", who, b, l_t, hk, wk, lead); return E2F_ERR_BAD_ARG; }
  if (!aligned(rows_hi, 16) || !aligned(rows_lo, 16) || !aligned(flow_up, 8) || (prev_flow && !aligned(prev_flow, 8))) { set_error("%s: alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_spynet_level_input(level_img, prev_flow, rows_hi, rows_lo, flow_up, b, l_t, hk, wk, lead, static_cast<cudaStream_t>(stream)), who);
}

int e2f_spynet_final(const float* flow, float* flows_forward, float* flows_backward, int b, int l_t, int h, int w, int h_up,
                     int w_up, void* stream) {
  const char* who = "e2f_spynet_final";
  if (!flow || !flows_forward || !flows_backward) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || l_t < 2 || h <= 0 || w <= 0 || h_up < h || w_up < w) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(flow, 8)) { set_error("%s: flow needs 8-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_spynet_final(flow, flows_forward, flows_backward, b, l_t, h, w, h_up, w_up, static_cast<cudaStream_t>(stream)), who);
}

int e2f_spynet_pyramid_unit(const float* frames, float* pyramid, int b, int t, int l_t, int H, int W, int h, int w, int h_up,
                            int w_up, const float* mean3, const float* std3, void* stream) {
  const char* who = "e2f_spynet_pyramid_unit";
  if (!frames || !pyramid || !mean3 || !std3) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || l_t <= 0 || l_t > t || H <= 0 || W <= 0 || h <= 1 || w <= 1 || h > H || w > W) { set_error("%s: bad shape b=%d t=%d l_t=%d %dx%d -> %dx%d", who, b, t, l_t, H, W, h, w); return E2F_ERR_BAD_ARG; }
  if (h_up < h || w_up < w || h_up % 32 || w_up % 32) { set_error("%s: the working size %dx%d must be multiples of 32 >= %dx%d", who, h_up, w_up, h, w); return E2F_ERR_BAD_ARG; }
  return finish(launch_spynet_pyramid_unit(frames, pyramid, b, t, l_t, H, W, h, w, h_up, w_up, mean3, std3, static_cast<cudaStream_t>(stream)), who);
}

int e2f_spynet_level_input_backward(const float* d_in, const float* dflow, const float* level_img, const float* flow_up,
                                    float* dprev, int b, int l_t, int hk, int wk, void* stream) {
  const char* who = "e2f_spynet_level_input_backward";
  if (!d_in || !dflow || !level_img || !flow_up || !dprev) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || l_t < 2 || hk < 2 || wk < 2 || ((hk | wk) & 1)) { set_error("%s: bad shape b=%d l_t=%d %dx%d (even sizes >= 2)", who, b, l_t, hk, wk); return E2F_ERR_BAD_ARG; }
  if (!aligned(d_in, 4) || !aligned(dflow, 8) || !aligned(flow_up, 8) || !aligned(dprev, 8)) { set_error("%s: alignment (dflow, flow_up, dprev 8 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_spynet_level_input_backward(d_in, dflow, level_img, flow_up, dprev, b, l_t, hk, wk, static_cast<cudaStream_t>(stream)), who);
}

int e2f_spynet_final_backward(const float* d_forward, const float* d_backward, float* dflow, int b, int l_t, int h, int w,
                              int h_up, int w_up, void* stream) {
  const char* who = "e2f_spynet_final_backward";
  if (!d_forward || !d_backward || !dflow) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || l_t < 2 || h <= 0 || w <= 0 || h_up < h || w_up < w) { set_error("%s: bad shape", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(dflow, 8)) { set_error("%s: dflow needs 8-byte alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_spynet_final_backward(d_forward, d_backward, dflow, b, l_t, h, w, h_up, w_up, static_cast<cudaStream_t>(stream)), who);
}

int e2f_video_prepare_clip(const uint8_t* frames, const uint8_t* masks, const int* ids, float* out, int t, int h, int w,
                           int hp, int wp, void* stream) {
  if (!frames || !masks || !ids || !out) { set_error("e2f_video_prepare_clip: null pointer"); return E2F_ERR_BAD_ARG; }
  if (t < 0 || h <= 0 || w <= 0 || hp < h || wp < w || hp > 2 * h || wp > 2 * w) {
    set_error("e2f_video_prepare_clip: bad shape t=%d h=%d w=%d hp=%d wp=%d (mirror padding needs h <= hp <= 2h, w <= wp <= 2w)", t, h, w, hp, wp);
    return E2F_ERR_BAD_ARG;
  }
  return finish(launch_video_prepare_clip(frames, masks, ids, out, t, h, w, hp, wp, static_cast<cudaStream_t>(stream)), "e2f_video_prepare_clip");
}

int e2f_video_compose(const float* pred, const uint8_t* frames, const uint8_t* masks, const int* ids, uint8_t* img,
                      int n_local, int h, int w, int hp, int wp, void* stream) {
  if (!pred || !frames || !masks || !ids || !img) { set_error("e2f_video_compose: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n_local < 0 || h <= 0 || w <= 0 || hp < h || wp < w) { set_error("e2f_video_compose: bad shape n_local=%d h=%d w=%d hp=%d wp=%d", n_local, h, w, hp, wp); return E2F_ERR_BAD_ARG; }
  return finish(launch_video_compose(pred, frames, masks, ids, img, n_local, h, w, hp, wp, static_cast<cudaStream_t>(stream)), "e2f_video_compose");
}

int e2f_video_blend(const uint8_t* img, const int* ids, const int* first, float* comp, int n_local, int64_t frame_elems,
                    void* stream) {
  if (!img || !ids || !first || !comp) { set_error("e2f_video_blend: null pointer"); return E2F_ERR_BAD_ARG; }
  if (n_local < 0 || frame_elems <= 0) { set_error("e2f_video_blend: bad shape"); return E2F_ERR_BAD_ARG; }
  return finish(launch_video_blend(img, ids, first, comp, n_local, static_cast<long long>(frame_elems), static_cast<cudaStream_t>(stream)), "e2f_video_blend");
}

int e2f_video_finalize(const float* comp, uint8_t* out, int64_t count, void* stream) {
  if (!comp || !out) { set_error("e2f_video_finalize: null pointer"); return E2F_ERR_BAD_ARG; }
  if (count < 0) { set_error("e2f_video_finalize: bad count"); return E2F_ERR_BAD_ARG; }
  return finish(launch_video_finalize(comp, out, static_cast<long long>(count), static_cast<cudaStream_t>(stream)), "e2f_video_finalize");
}

// widest frame the bicubic resize takes: one input row is staged in shared memory
static const int kResizeMaxWidth = 65536;

int e2f_video_resize_bicubic(const uint8_t* src, uint8_t* dst, uint8_t* scratch, const int* xtab, int xtaps,
                             const int* ytab, int ytaps, int n, int h, int w, int h2, int w2, void* stream) {
  const char* who = "e2f_video_resize_bicubic";
  if (!src || !dst) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || h2 <= 0 || w2 <= 0 || w > kResizeMaxWidth || w2 > kResizeMaxWidth ||
      static_cast<long long>(n) * (h > h2 ? h : h2) > 0x7fffffffLL) {
    set_error("%s: bad shape n=%d %dx%d -> %dx%d (widths up to %d)", who, n, h, w, h2, w2, kResizeMaxWidth);
    return E2F_ERR_BAD_ARG;
  }
  const bool horiz = w2 != w, vert = h2 != h;
  if (horiz && (!xtab || xtaps <= 0)) { set_error("%s: width changes but xtab is null or xtaps=%d", who, xtaps); return E2F_ERR_BAD_ARG; }
  if (vert && (!ytab || ytaps <= 0)) { set_error("%s: height changes but ytab is null or ytaps=%d", who, ytaps); return E2F_ERR_BAD_ARG; }
  if (horiz && vert && !scratch) { set_error("%s: null scratch (both passes run)", who); return E2F_ERR_BAD_ARG; }
  return finish(launch_video_resize_bicubic(src, dst, scratch, xtab, xtaps, ytab, ytaps, n, h, w, h2, w2, static_cast<cudaStream_t>(stream)), who);
}

int e2f_video_prepare_masks(const uint8_t* src, uint8_t* dst, const int* rows, const int* cols, int n, int hm, int wm,
                            int h, int w, void* stream) {
  const char* who = "e2f_video_prepare_masks";
  if (!src || !dst || !rows || !cols) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || hm <= 0 || wm <= 0 || h <= 0 || w <= 0 || (h + 31) / 32 > 65535) {
    set_error("%s: bad shape n=%d %dx%d -> %dx%d", who, n, hm, wm, h, w);
    return E2F_ERR_BAD_ARG;
  }
  return finish(launch_video_prepare_masks(src, dst, rows, cols, n, hm, wm, h, w, static_cast<cudaStream_t>(stream)), who);
}

// ----------------------------------------------------------------------------- I3D (VFID)
static bool pad_ok(const int* pad, int k, int t, int h, int w) {
  const int sz[3] = {t, h, w};
  for (int a = 0; a < 3; ++a)
    if (pad[2 * a] < 0 || pad[2 * a + 1] < 0 || pad[2 * a] >= k || pad[2 * a + 1] >= k ||
        sz[a] + pad[2 * a] + pad[2 * a + 1] < k)
      return false;
  return true;
}

int e2f_conv3d_bf16x3(const void* src_hi, const void* src_lo, int cin, const void* w_hi, const void* w_lo, const float* bias,
                      float* out, void* out_hi, void* out_lo, int out_cs, int b, int t, int h, int w, int cout, int ksize,
                      const int* pad, int relu, void* stream) {
  const char* who = "e2f_conv3d_bf16x3";
  if (!src_hi || !src_lo || !w_hi || !w_lo || !pad) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || cin <= 0 || cout <= 0 || cout > 512) { set_error("%s: bad shape b=%d t=%d h=%d w=%d cin=%d cout=%d", who, b, t, h, w, cin, cout); return E2F_ERR_BAD_ARG; }
  if (cin % 8 || cout % 8 || out_cs < cout || out_cs % 8) { set_error("%s: cin, cout and out_cs must be multiples of 8 with out_cs >= cout (cin=%d cout=%d out_cs=%d)", who, cin, cout, out_cs); return E2F_ERR_UNSUPPORTED; }
  if (ksize != 1 && ksize != 3) { set_error("%s: ksize=%d (1 or 3)", who, ksize); return E2F_ERR_UNSUPPORTED; }
  if (!pad_ok(pad, ksize, t, h, w)) { set_error("%s: padding must be 0..ksize-1 per side and leave a non-empty output", who); return E2F_ERR_BAD_ARG; }
  if (relu != 0 && relu != 1) { set_error("%s: relu=%d", who, relu); return E2F_ERR_BAD_ARG; }
  if (!aligned(src_hi, 16) || !aligned(src_lo, 16) || !aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) ||
      (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (bias && !aligned(bias, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_conv3d(src_hi, src_lo, cin, 0, w_hi, w_lo, bias, out, out_hi, out_lo, out_cs, b, t, h, w, cout, ksize, 1,
                              pad, relu ? 0.f : 1.f, static_cast<cudaStream_t>(stream)), who);
}

int64_t e2f_i3d_stem_elems(int b, int t, int h, int w) {
  if (b < 0 || t <= 0 || h <= 0 || w <= 0) return E2F_ERR_BAD_ARG;
  return static_cast<int64_t>(i3d_stem_elems(b, t, h, w));
}

int e2f_i3d_stem_pack(const void* x, int x_u8, void* hi, void* lo, int b, int t, int h, int w, void* stream) {
  const char* who = "e2f_i3d_stem_pack";
  if (!x || !hi || !lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || (x_u8 != 0 && x_u8 != 1)) { set_error("%s: bad shape b=%d t=%d h=%d w=%d x_u8=%d", who, b, t, h, w, x_u8); return E2F_ERR_BAD_ARG; }
  if (!aligned(hi, 16) || !aligned(lo, 16) || (!x_u8 && !aligned(x, 4))) { set_error("%s: alignment", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_i3d_stem_pack(x, x_u8, hi, lo, b, t, h, w, static_cast<cudaStream_t>(stream)), who);
}

int e2f_i3d_stem_conv(const void* hi, const void* lo, const void* w_hi, const void* w_lo, const float* bias, float* out,
                      void* out_hi, void* out_lo, int out_cs, int b, int t, int h, int w, int cout, void* stream) {
  const char* who = "e2f_i3d_stem_conv";
  if (!hi || !lo || !w_hi || !w_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || cout <= 0 || cout > 512 || cout % 8 || out_cs < cout || out_cs % 8) { set_error("%s: bad shape b=%d t=%d h=%d w=%d cout=%d out_cs=%d", who, b, t, h, w, cout, out_cs); return E2F_ERR_BAD_ARG; }
  if (!aligned(hi, 16) || !aligned(lo, 16) || !aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) ||
      (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (bias && !aligned(bias, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_i3d_stem_conv(hi, lo, w_hi, w_lo, bias, out, out_hi, out_lo, out_cs, b, t, h, w, cout,
                                     static_cast<cudaStream_t>(stream)), who);
}

int e2f_maxpool3d(const float* x, float* out, void* out_hi, void* out_lo, int b, int t, int h, int w, int c, const int* ksize,
                  const int* stride, const int* pad, void* stream) {
  const char* who = "e2f_maxpool3d";
  if (!x || !ksize || !stride || !pad) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || c <= 0 || c % 4 || (out_hi && c % 8)) { set_error("%s: bad shape b=%d t=%d h=%d w=%d c=%d", who, b, t, h, w, c); return E2F_ERR_BAD_ARG; }
  const int sz[3] = {t, h, w};
  for (int a = 0; a < 3; ++a) {
    if (ksize[a] < 1 || ksize[a] > 3 || stride[a] < 1 || stride[a] > 2 || pad[2 * a] < 0 || pad[2 * a + 1] < 0 ||
        pad[2 * a] >= ksize[a] || pad[2 * a + 1] >= ksize[a] || sz[a] + pad[2 * a] + pad[2 * a + 1] < ksize[a]) {
      set_error("%s: unsupported window on axis %d (k=%d s=%d pad=%d,%d)", who, a, ksize[a], stride[a], pad[2 * a], pad[2 * a + 1]);
      return E2F_ERR_UNSUPPORTED;
    }
  }
  if (!aligned(x, 16) || (out && !aligned(out, 16)) || (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16)))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_i3d_maxpool(x, out, out_hi, out_lo, b, t, h, w, c, ksize, stride, pad, static_cast<cudaStream_t>(stream)), who);
}

int e2f_mean_thw(const float* x, float* out, int b, int t, int h, int w, int c, void* stream) {
  const char* who = "e2f_mean_thw";
  if (!x || !out) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (b < 0 || t <= 0 || h <= 0 || w <= 0 || c <= 0) { set_error("%s: bad shape b=%d t=%d h=%d w=%d c=%d", who, b, t, h, w, c); return E2F_ERR_BAD_ARG; }
  return finish(launch_i3d_mean(x, out, b, t, h, w, c, static_cast<cudaStream_t>(stream)), who);
}

// ----------------------------------------------------------------------------- PSNR / SSIM (evaluate.py)
static constexpr size_t kMetricsMaxSmem = 227 * 1024;   // sm_90 opt-in shared memory per block, static included

// win = 0 asks for the SSE alone
static long long metrics_ctas(int n, int h, int w, int c, int win) {
  return static_cast<long long>(n) * (win ? frame_metrics_tiles(w, win) : frame_sse_blocks(h, w, c));
}

static bool metrics_shape_ok(const char* who, int n, int h, int w, int c, int win) {
  if (n < 1 || h < 1 || w < 1 || c < 1 || c > 4) { set_error("%s: bad shape n=%d h=%d w=%d c=%d (n >= 1, 1 <= c <= 4)", who, n, h, w, c); return false; }
  if (win != 0 && (win < 3 || !(win & 1) || win > h || win > w)) { set_error("%s: win=%d must be 0 (SSE only) or odd, >= 3 and <= min(h, w) = %d", who, win, h < w ? h : w); return false; }
  if (metrics_ctas(n, h, w, c, win) > 0x7fffffffLL) { set_error("%s: n=%d frames of %dx%dx%d are too many for one call", who, n, h, w, c); return false; }
  return true;
}

int64_t e2f_frame_metrics_work_elems(int n, int h, int w, int c, int win) {
  if (!metrics_shape_ok("e2f_frame_metrics_work_elems", n, h, w, c, win)) return E2F_ERR_BAD_ARG;
  return static_cast<int64_t>(metrics_ctas(n, h, w, c, win)) * (win ? 1 + c : 1);
}

int e2f_frame_metrics(const void* a, int a_u8, const void* b, int b_u8, double* sse, double* ssim, double* work, int n,
                      int h, int w, int c, int win, double data_range, void* stream) {
  const char* who = "e2f_frame_metrics";
  if (!a || !b || !sse || (win && !ssim)) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((a_u8 != 0 && a_u8 != 1) || (b_u8 != 0 && b_u8 != 1)) { set_error("%s: a_u8=%d b_u8=%d (0 = fp32, 1 = uint8)", who, a_u8, b_u8); return E2F_ERR_BAD_ARG; }
  if (!metrics_shape_ok(who, n, h, w, c, win)) return E2F_ERR_BAD_ARG;
  if (!(data_range > 0.0) || data_range > 1e300) { set_error("%s: data_range=%g must be > 0 and finite", who, data_range); return E2F_ERR_BAD_ARG; }
  if (!work) { set_error("%s: null workspace (e2f_frame_metrics_work_elems doubles needed)", who); return E2F_ERR_BAD_ARG; }
  if (win && frame_metrics_smem(c, win) > kMetricsMaxSmem) { set_error("%s: win=%d with c=%d needs %zu bytes of shared memory (at most %zu)", who, win, c, frame_metrics_smem(c, win), kMetricsMaxSmem); return E2F_ERR_UNSUPPORTED; }
  if ((!a_u8 && !aligned(a, 4)) || (!b_u8 && !aligned(b, 4)) || !aligned(sse, 8) || (ssim && !aligned(ssim, 8)) || !aligned(work, 8)) { set_error("%s: alignment (fp32 operands 4 bytes, outputs and workspace 8)", who); return E2F_ERR_ALIGNMENT; }
  if (!win) return finish(launch_frame_sse(a, a_u8, b, b_u8, sse, work, n, h, w, c, static_cast<cudaStream_t>(stream)), who);
  return finish(launch_frame_metrics(a, a_u8, b, b_u8, sse, ssim, work, n, h, w, c, win, data_range,
                                     static_cast<cudaStream_t>(stream)), who);
}

// ----------------------------------------------------------------------------- Temporal PatchGAN discriminator
static int dis_out_size(int s, int pad) { return (s + 2 * pad - 5) / 2 + 1; }

static bool dis_shape_ok(const char* who, int b, int t, int h_in, int w_in, int pad) {
  if (b < 1 || t < 1 || h_in + 2 * pad < 5 || w_in + 2 * pad < 5 || (pad != 1 && pad != 2) || dis_out_size(h_in, pad) < 1 ||
      dis_out_size(w_in, pad) < 1 || static_cast<long long>(b) * t > 0x7fffffffLL) {
    set_error("%s: bad shape b=%d t=%d h=%d w=%d pad=%d (a 5x5 window at stride 2 needs h, w >= %d)", who, b, t, h_in, w_in,
              pad, 5 - 2 * pad);
    return false;
  }
  return true;
}

int e2f_dis_conv3d(const void* x_hi, const void* x_lo, int cin, const void* w_hi, const void* w_lo, const float* bias,
                   float* out, void* out_hi, void* out_lo, int b, int t, int h_in, int w_in, int cout, int pad, int leaky,
                   void* stream) {
  const char* who = "e2f_dis_conv3d";
  if (!x_hi || !x_lo || !w_hi || !w_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!out && !out_hi) || (!out_hi) != (!out_lo)) { set_error("%s: need out and/or both of out_hi/out_lo", who); return E2F_ERR_BAD_ARG; }
  if (!dis_shape_ok(who, b, t, h_in, w_in, pad)) return E2F_ERR_BAD_ARG;
  if (cin < 8 || cin % 8 || cout < 8 || cout % 8 || cout > 128) { set_error("%s: cin=%d must be a multiple of 8, cout=%d a multiple of 8 <= 128", who, cin, cout); return E2F_ERR_UNSUPPORTED; }
  if (leaky != 0 && leaky != 1) { set_error("%s: leaky=%d", who, leaky); return E2F_ERR_BAD_ARG; }
  if (!aligned(x_hi, 16) || !aligned(x_lo, 16) || !aligned(w_hi, 16) || !aligned(w_lo, 16) || (out && !aligned(out, 16)) ||
      (out_hi && (!aligned(out_hi, 16) || !aligned(out_lo, 16))) || (bias && !aligned(bias, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dis_conv(x_hi, x_lo, cin, w_hi, w_lo, bias, out, out_hi, out_lo, b, t, h_in, w_in, dis_out_size(h_in, pad),
                                dis_out_size(w_in, pad), cout, pad, 0, leaky ? 0.2f : 1.f, nullptr, 0.f,
                                static_cast<cudaStream_t>(stream)), who);
}

int e2f_dis_conv3d_dgrad(const void* dy_hi, const void* dy_lo, int cout, const void* wt_hi, const void* wt_lo, float* dx,
                         void* dx_hi, void* dx_lo, const void* act, int b, int t, int h_in, int w_in, int cin, int pad,
                         void* stream) {
  const char* who = "e2f_dis_conv3d_dgrad";
  if (!dy_hi || !dy_lo || !wt_hi || !wt_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!dx && !dx_hi) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dx and/or both of dx_hi/dx_lo", who); return E2F_ERR_BAD_ARG; }
  if (!dis_shape_ok(who, b, t, h_in, w_in, pad)) return E2F_ERR_BAD_ARG;
  if (cout < 8 || cout % 8 || cin < 8 || cin % 8 || cin > 128) { set_error("%s: cout=%d must be a multiple of 8, cin=%d a multiple of 8 <= 128", who, cout, cin); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(dy_hi, 16) || !aligned(dy_lo, 16) || !aligned(wt_hi, 16) || !aligned(wt_lo, 16) || (dx && !aligned(dx, 16)) ||
      (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16))) || (act && !aligned(act, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dis_conv(dy_hi, dy_lo, cout, wt_hi, wt_lo, nullptr, dx, dx_hi, dx_lo, b, t, dis_out_size(h_in, pad),
                                dis_out_size(w_in, pad), h_in, w_in, cin, pad, 1, 1.f, act, 0.2f,
                                static_cast<cudaStream_t>(stream)), who);
}

int64_t e2f_dis_conv3d_wgrad_work_elems(int b, int t, int h_in, int w_in, int cin, int cout, int pad) {
  if (!dis_shape_ok("e2f_dis_conv3d_wgrad_work_elems", b, t, h_in, w_in, pad)) return E2F_ERR_BAD_ARG;
  if (cin < 8 || cin % 8 || cin > 512 || cout < 8 || cout % 8 || cout > 512) { set_error("e2f_dis_conv3d_wgrad_work_elems: cin=%d cout=%d (multiples of 8, <= 512)", cin, cout); return E2F_ERR_BAD_ARG; }
  return static_cast<int64_t>(dis_wgrad_work_elems(b, t, dis_out_size(h_in, pad), dis_out_size(w_in, pad), cout, cin));
}

int e2f_dis_conv3d_wgrad(const float* dy, const void* x_hi, const void* x_lo, float* dw, float* db, float* work, int b,
                         int t, int h_in, int w_in, int cin, int cout, int pad, void* stream) {
  const char* who = "e2f_dis_conv3d_wgrad";
  if (!dy || !x_hi || !x_lo || !dw) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (!dis_shape_ok(who, b, t, h_in, w_in, pad)) return E2F_ERR_BAD_ARG;
  if (cin < 8 || cin % 8 || cin > 512 || cout < 8 || cout % 8 || cout > 512) { set_error("%s: cin=%d cout=%d (multiples of 8, <= 512)", who, cin, cout); return E2F_ERR_BAD_ARG; }
  if (!work) { set_error("%s: null workspace (e2f_dis_conv3d_wgrad_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy, 16) || !aligned(x_hi, 16) || !aligned(x_lo, 16) || !aligned(dw, 4) || (db && !aligned(db, 4)) ||
      !aligned(work, 4)) { set_error("%s: alignment (dy, x_hi, x_lo 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_dis_wgrad(dy, x_hi, x_lo, dw, db, work, b, t, h_in, w_in, cin, dis_out_size(h_in, pad),
                                 dis_out_size(w_in, pad), cout, pad, static_cast<cudaStream_t>(stream)), who);
}

static bool rows_c(int c) { return c == 4 || c == 8 || c == 16 || c == 32; }

int e2f_conv2d_dgrad_bf16x3(const void* dy_hi, const void* dy_lo, int dy_c, int dy_lead, const void* wt_hi, const void* wt_lo,
                            const void* act, int act_lead, float* dx, void* dx_hi, void* dx_lo, int dx_lead, int n, int h,
                            int w, int cin, void* stream) {
  const char* who = "e2f_conv2d_dgrad_bf16x3";
  if (!dy_hi || !dy_lo || !wt_hi || !wt_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!dx && !dx_hi) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dx and/or both of dx_hi/dx_lo", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0) { set_error("%s: bad shape n=%d h=%d w=%d", who, n, h, w); return E2F_ERR_BAD_ARG; }
  if (dy_lead != 0 && dy_lead != 3) { set_error("%s: dy_lead=%d (0: dense, 3: row-gapped for the 7x7 / pad 3 conv)", who, dy_lead); return E2F_ERR_BAD_ARG; }
  if (act_lead < 0 || act_lead > 8 || dx_lead < 0 || dx_lead > 8 || (dx_lead && !dx_hi)) { set_error("%s: act_lead=%d dx_lead=%d (0..8; a row-gapped dx needs the split)", who, act_lead, dx_lead); return E2F_ERR_BAD_ARG; }
  // row-gapped: the tensor map steps one pixel per row element, a 16-byte multiple from 8 channels on
  if (dy_lead ? (!rows_c(dy_c) || dy_c < 8) : (dy_c < 8 || dy_c % 8)) { set_error("%s: dy_c=%d (row-gapped: 8, 16 or 32; dense: a multiple of 8)", who, dy_c); return E2F_ERR_UNSUPPORTED; }
  if (cin < 8 || cin % 8 || cin > 64 || ((dx_lead || act_lead) && !rows_c(cin))) { set_error("%s: cin=%d (a multiple of 8 <= 64; 8, 16 or 32 when dx or act is row-gapped)", who, cin); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(dy_hi, 16) || !aligned(dy_lo, 16) || !aligned(wt_hi, 16) || !aligned(wt_lo, 16) || (dx && !aligned(dx, 16)) ||
      (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16))) || (act && !aligned(act, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  const void* srch[1] = {dy_hi};
  const void* srcl[1] = {dy_lo};
  const int ch[1] = {dy_c};
  return finish(launch_conv3x3(1, srch, srcl, ch, wt_hi, wt_lo, nullptr, nullptr, dx, dx_hi, dx_lo, n, h, w, cin, 1, 1.f, 7,
                               1, 3, dy_lead ? 1 : 0, dx_lead, static_cast<cudaStream_t>(stream), nullptr, 0, act, act_lead), who);
}

int64_t e2f_conv2d_wgrad_work_elems(int n, int h, int w, int cin, int cout) {
  if (n < 0 || h <= 0 || w <= 0 || cin < 8 || cin % 8 || cin > 512 || cout < 8 || cout % 8 || cout > 512) { set_error("e2f_conv2d_wgrad_work_elems: n=%d %dx%d cin=%d cout=%d (multiples of 8, <= 512)", n, h, w, cin, cout); return E2F_ERR_BAD_ARG; }
  return static_cast<int64_t>(conv2d_wgrad_work_elems(n, h, w, cin, cout));
}

int e2f_conv2d_wgrad_bf16x3(const float* dy, const void* x_hi, const void* x_lo, int x_lead, float* dw, float* db, float* work,
                            int n, int h, int w, int cin, int cout, void* stream) {
  const char* who = "e2f_conv2d_wgrad_bf16x3";
  if (!dy || !x_hi || !x_lo || !dw) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || x_lead < 0 || x_lead > 8) { set_error("%s: bad shape n=%d %dx%d x_lead=%d", who, n, h, w, x_lead); return E2F_ERR_BAD_ARG; }
  if (cin < 8 || cin % 8 || cin > 512 || cout < 8 || cout % 8 || cout > 512 || (x_lead && !rows_c(cin))) { set_error("%s: cin=%d cout=%d (multiples of 8, <= 512; cin 8, 16 or 32 when x is row-gapped)", who, cin, cout); return E2F_ERR_BAD_ARG; }
  if (!work) { set_error("%s: null workspace (e2f_conv2d_wgrad_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy, 16) || !aligned(x_hi, 16) || !aligned(x_lo, 16) || !aligned(dw, 4) || (db && !aligned(db, 4)) ||
      !aligned(work, 4)) { set_error("%s: alignment (dy, x_hi, x_lo 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_conv2d_wgrad(dy, x_hi, x_lo, x_lead, dw, db, work, n, h, w, cin, cout, static_cast<cudaStream_t>(stream)), who);
}

static bool groups_ok(int g) { return g == 1 || g == 2 || g == 4 || g == 8; }

int e2f_conv_dgrad_bf16x3(const void* dy_hi, const void* dy_lo, int dy_c, int dy_lead, const void* wt_hi, const void* wt_lo,
                          const void* act, const float* residual, float* dx, void* dx_hi, void* dx_lo, int n, int h_in,
                          int w_in, int cin, int groups, int ks, int stride, void* stream) {
  const char* who = "e2f_conv_dgrad_bf16x3";
  if (!dy_hi || !dy_lo || !wt_hi || !wt_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if ((!dx && !dx_hi) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dx and/or both of dx_hi/dx_lo", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h_in <= 0 || w_in <= 0) { set_error("%s: bad shape n=%d h_in=%d w_in=%d", who, n, h_in, w_in); return E2F_ERR_BAD_ARG; }
  if (!((ks == 3 || ks == 7) && stride == 1) && !(ks == 3 && stride == 2)) { set_error("%s: ks=%d stride=%d (3 or 7 at stride 1, 3 at stride 2)", who, ks, stride); return E2F_ERR_UNSUPPORTED; }
  if (!groups_ok(groups) || (stride == 2 && groups != 1)) { set_error("%s: groups=%d (1, 2, 4 or 8; 1 at stride 2)", who, groups); return E2F_ERR_UNSUPPORTED; }
  if (cin < 8 || cin > 512 || cin % (8 * groups)) { set_error("%s: cin=%d (<= 512, a multiple of 8 per group)", who, cin); return E2F_ERR_UNSUPPORTED; }
  if (dy_lead != 0 && (dy_lead != ks / 2 || stride != 1 || groups != 1)) { set_error("%s: dy_lead=%d (0: dense; %d: row-gapped, stride 1, groups 1)", who, dy_lead, ks / 2); return E2F_ERR_BAD_ARG; }
  if (dy_lead ? !rows_c(dy_c) || dy_c < 8 : (dy_c < 8 || dy_c % (8 * groups))) { set_error("%s: dy_c=%d (row-gapped: 8, 16 or 32; dense: a multiple of 8 per group)", who, dy_c); return E2F_ERR_UNSUPPORTED; }
  if (!aligned(dy_hi, 16) || !aligned(dy_lo, 16) || !aligned(wt_hi, 16) || !aligned(wt_lo, 16) || (dx && !aligned(dx, 16)) ||
      (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16))) || (act && !aligned(act, 16)) || (residual && !aligned(residual, 16))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  if (n == 0) return 0;
  return finish(launch_conv_dgrad(dy_hi, dy_lo, dy_c, dy_lead, wt_hi, wt_lo, act, residual, dx, dx_hi, dx_lo, n, h_in, w_in,
                                  cin, groups, ks, stride, static_cast<cudaStream_t>(stream)), who);
}

static bool linear_wgrad_ok(const char* who, int m, int n, int k) {
  if (m < 0 || n <= 0 || k <= 0) { set_error("%s: bad shape m=%d n=%d k=%d", who, m, n, k); return false; }
  return true;
}

int64_t e2f_linear_wgrad_work_elems(int m, int n, int k) {
  if (!linear_wgrad_ok("e2f_linear_wgrad_work_elems", m, n, k)) return E2F_ERR_BAD_ARG;
  return static_cast<int64_t>(linear_wgrad_work_elems(m, n, k));
}

int e2f_linear_wgrad_bf16x3(const void* dy_hi, const void* dy_lo, int ldy, const void* x_hi, const void* x_lo, int ldx, float* dw,
                            float* db, float* work, int m, int n, int k, void* stream) {
  const char* who = "e2f_linear_wgrad_bf16x3";
  if (!dy_hi || !dy_lo || !x_hi || !x_lo || !dw) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (!linear_wgrad_ok(who, m, n, k)) return E2F_ERR_BAD_ARG;
  if (ldy < n || ldx < k || ldy % 8 || ldx % 8) { set_error("%s: row pitches ldy=%d ldx=%d must be multiples of 8 >= n=%d / k=%d", who, ldy, ldx, n, k); return E2F_ERR_BAD_ARG; }
  if (!work && linear_wgrad_work_elems(m, n, k) > 0) { set_error("%s: null workspace (e2f_linear_wgrad_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy_hi, 16) || !aligned(dy_lo, 16) || !aligned(x_hi, 16) || !aligned(x_lo, 16) || !aligned(dw, 4) || (db && !aligned(db, 4)) || (work && !aligned(work, 4))) { set_error("%s: alignment (operands 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_linear_wgrad(dy_hi, dy_lo, ldy, x_hi, x_lo, ldx, dw, db, work, m, n, k, static_cast<cudaStream_t>(stream)), who);
}

static bool conv3x3_wgrad_ok(const char* who, int n, int h_in, int w_in, int cin, int cout, int groups, int stride) {
  if (n < 0 || h_in <= 0 || w_in <= 0 || (stride != 1 && stride != 2) || !groups_ok(groups)) { set_error("%s: bad shape n=%d %dx%d stride=%d groups=%d", who, n, h_in, w_in, stride, groups); return false; }
  if (cin % (8 * groups) || cin / groups > 512 || cout < 8 || cout > 512 || cout % (8 * groups)) { set_error("%s: cin=%d cout=%d (multiples of 8 per group, <= 512 per group)", who, cin, cout); return false; }
  return true;
}

int64_t e2f_conv3x3_wgrad_work_elems(int n, int h_in, int w_in, int cin, int cout, int groups, int stride) {
  if (!conv3x3_wgrad_ok("e2f_conv3x3_wgrad_work_elems", n, h_in, w_in, cin, cout, groups, stride)) return E2F_ERR_BAD_ARG;
  return static_cast<int64_t>(conv3x3_wgrad_work_elems(n, h_in, w_in, cin / groups, cout, groups, stride));
}

int e2f_conv3x3_wgrad_bf16x3(const float* dy, int nsrc, const void* const* x_hi, const void* const* x_lo, const int* x_c,
                             int x_lead, float* dw, float* db, float* work, int n, int h_in, int w_in, int cout, int groups,
                             int stride, void* stream) {
  const char* who = "e2f_conv3x3_wgrad_bf16x3";
  if (!dy || !x_hi || !x_lo || !x_c || !dw) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (nsrc < 1 || nsrc > 2) { set_error("%s: nsrc=%d (1 or 2)", who, nsrc); return E2F_ERR_BAD_ARG; }
  int cin = 0;
  for (int i = 0; i < nsrc; ++i) {
    if (!x_hi[i] || !x_lo[i]) { set_error("%s: null source %d", who, i); return E2F_ERR_BAD_ARG; }
    if (x_c[i] < 8 || x_c[i] % (8 * groups)) { set_error("%s: source %d has %d channels (a multiple of 8 per group)", who, i, x_c[i]); return E2F_ERR_BAD_ARG; }
    if (!aligned(x_hi[i], 16) || !aligned(x_lo[i], 16)) { set_error("%s: alignment (sources 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
    cin += x_c[i];
  }
  if (!conv3x3_wgrad_ok(who, n, h_in, w_in, cin, cout, groups, stride)) return E2F_ERR_BAD_ARG;
  if (x_lead != 0 && (x_lead != 1 || nsrc != 1 || groups != 1 || !rows_c(x_c[0]))) { set_error("%s: x_lead=%d (0: dense; 1: one row-gapped source of 8, 16 or 32 channels, groups 1)", who, x_lead); return E2F_ERR_BAD_ARG; }
  if (!work) { set_error("%s: null workspace (e2f_conv3x3_wgrad_work_elems floats needed)", who); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy, 16) || !aligned(dw, 4) || (db && !aligned(db, 4)) || !aligned(work, 4)) { set_error("%s: alignment (dy 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_conv3x3_wgrad(dy, nsrc, x_hi, x_lo, x_c, x_lead, dw, db, work, n, h_in, w_in, cout, groups, stride,
                                     static_cast<cudaStream_t>(stream)), who);
}

int e2f_upsample2x_backward(const float* dy, const float* act, float* dx, void* dx_hi, void* dx_lo, int n, int h, int w, int c,
                            void* stream) {
  const char* who = "e2f_upsample2x_backward";
  if (!dy || (!dx && !dx_hi) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dy, and dx and/or both of dx_hi/dx_lo", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c < 8 || c % 8) { set_error("%s: bad shape n=%d %dx%d c=%d (c a multiple of 8)", who, n, h, w, c); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy, 32) || (act && !aligned(act, 32)) || (dx && !aligned(dx, 32)) || (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16)))) { set_error("%s: alignment (fp32 32 bytes, bf16 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_upsample2x_backward(dy, act, dx, dx_hi, dx_lo, n, h, w, c, 0.2f, static_cast<cudaStream_t>(stream)), who);
}

int e2f_tanh_backward_rows(const float* dout, const float* out, float* dy, void* dy_hi, void* dy_lo, int n, int c, int h, int w,
                           int lead, void* stream) {
  const char* who = "e2f_tanh_backward_rows";
  if (!dout || !out || !dy || !dy_hi || !dy_lo) { set_error("%s: null pointer", who); return E2F_ERR_BAD_ARG; }
  if (n < 0 || h <= 0 || w <= 0 || c < 1 || c > 8 || lead < 1 || lead > 8) { set_error("%s: bad shape n=%d c=%d %dx%d lead=%d (c 1..8, lead 1..8)", who, n, c, h, w, lead); return E2F_ERR_BAD_ARG; }
  if (!aligned(dout, 4) || !aligned(out, 4) || !aligned(dy, 16) || !aligned(dy_hi, 16) || !aligned(dy_lo, 16)) { set_error("%s: alignment (dy, dy_hi, dy_lo 16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_tanh_backward_rows(dout, out, dy, dy_hi, dy_lo, n, c, h, w, lead, static_cast<cudaStream_t>(stream)), who);
}

int e2f_leaky_relu_backward(const float* dy, const float* act, float* dx, void* dx_hi, void* dx_lo, int64_t count, float slope,
                            void* stream) {
  const char* who = "e2f_leaky_relu_backward";
  if (!dy || !act || (!dx && !dx_hi) || (!dx_hi) != (!dx_lo)) { set_error("%s: need dy, act, and dx and/or both of dx_hi/dx_lo", who); return E2F_ERR_BAD_ARG; }
  if (count < 0 || count % 8) { set_error("%s: count=%lld (a multiple of 8)", who, static_cast<long long>(count)); return E2F_ERR_BAD_ARG; }
  if (!aligned(dy, 16) || !aligned(act, 16) || (dx && !aligned(dx, 16)) || (dx_hi && (!aligned(dx_hi, 16) || !aligned(dx_lo, 16)))) { set_error("%s: alignment (16 bytes)", who); return E2F_ERR_ALIGNMENT; }
  return finish(launch_leaky_backward(dy, act, dx, dx_hi, dx_lo, count, slope, static_cast<cudaStream_t>(stream)), who);
}

}  // extern "C"
