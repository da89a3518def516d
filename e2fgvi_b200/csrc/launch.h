// Internal host-side launcher declarations shared by api.cu and the kernel translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>

namespace e2f {

// Function attributes (opt-in dynamic shared memory), SM counts and cluster occupancy are PER DEVICE: a process that
// drives several GPUs (model moved to cuda:1, one thread per device) must configure each of them.  One bit per device
// ordinal; devices >= 64 are simply configured on every call.  Setting an attribute twice is idempotent, so two threads
// racing on the same bit are harmless.
struct DeviceOnce {
  std::atomic<unsigned long long> done{0};
};
inline int current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return d;
}
inline bool device_done(const DeviceOnce& o, int dev) {
  return dev >= 0 && dev < 64 && ((o.done.load(std::memory_order_acquire) >> dev) & 1ull);
}
inline void device_mark(DeviceOnce& o, int dev) {
  if (dev >= 0 && dev < 64) o.done.fetch_or(1ull << dev, std::memory_order_release);
}
int num_sms();                             // api.cu: SM count of the CURRENT device (cached per device ordinal)

void count_launch();                       // api.cu: atomic launch counter behind e2f_launch_count()
void set_error(const char* fmt, ...);      // api.cu: thread-local message behind e2f_last_error()

// Opts `kernels` in to `smem` bytes of dynamic shared memory, once per device.  carveout >= 0 also sets the preferred
// shared-memory carve-out (percent); that is a hint, so its result is ignored.  Returns the first cudaFuncSetAttribute
// error, or 0; the device is marked configured only when every kernel took its size, so a failure is reported again on
// the next call.
template <typename... Kernels>
int configure_once_carveout(DeviceOnce& once, int smem, int carveout, Kernels... kernels) {
  const int dev = current_device();
  if (device_done(once, dev)) return 0;
  const void* const list[] = {reinterpret_cast<const void*>(kernels)...};
  for (const void* k : list) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (carveout >= 0)
    for (const void* k : list) cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
  device_mark(once, dev);
  return 0;
}
template <typename... Kernels>
int configure_once(DeviceOnce& once, int smem, Kernels... kernels) {
  return configure_once_carveout(once, smem, -1, kernels...);
}

// api.cu: encodes a tiled TMA tensor map with the settings every kernel here uses: no interleave, 128-byte swizzle,
// 256-byte L2 promotion, zero fill out of bounds.  dims / box / estr have `rank` entries, strides (bytes) rank - 1.  The
// driver's entry point is looked up on the first call, so a launcher that validates its arguments before it encodes a
// map makes no CUDA call for a rejected one.  Returns 0, or -4 with an error naming the map `what` when the driver lacks
// the entry point or rejects the map.
int encode_tmap(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                const cuuint32_t* box, const cuuint32_t* estr, const char* what,
                CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);

int launch_flow_warp_nhwc(const void* x, const float* flow, void* out, int n, int h, int w, int c, int dtype,
                          int pad_mode, cudaStream_t stream);
int launch_flow_warp_nchw(const float* x, const float* flow, float* out, int n, int c, int h, int w, int pad_mode,
                          cudaStream_t stream);

int launch_prop_prologue(const float* prop, const float* feat2, const float* flow1, long long f1_bs, const float* flowp,
                         long long fp_bs, void* c1h, void* c1l, void* c2h, void* c2l, float* f1_out, float* f2_out,
                         void* flh, void* fll, void* xg, int n, int h, int w, int c, cudaStream_t stream);

int launch_dcn_pack_weight(const float* w, void* w_packed, int cout, int cin, int dg, cudaStream_t stream);
// head != nullptr selects the fused (tanh / flow / sigmoid) prologue; otherwise offset+mask are final values.
int launch_dcn(const void* x, const float* offset, const float* mask, const float* head, const float* flow1,
               const float* flow2, const void* w_packed, const float* bias, void* out, int n, int h, int w, int cin,
               int cout, int dg, float max_residue, int out_dtype, int x_grouped, cudaStream_t stream,
               void* out_hi = nullptr, void* out_lo = nullptr);   // optional bf16 split of the fp32 result
int launch_dcn_pack_input(const float* a, const float* b, void* xg, int n, int h, int w, int ca, int cb,
                          cudaStream_t stream);
// Deformable alignment backward (dcn_grad.cu): the sampler's adjoint (d head / offset part of d flow, the split sample
// rows A, the dx scatter list in `work`) and the sort + gather of dx; workspace of dcn_backward_work_elems 32-bit words.
long long dcn_backward_work_elems(int n, int h, int w);
int launch_dcn_sample_backward(const void* x, const float* head, const float* flow1, const float* flow2, const float* da,
                               float* dhead, float* dflow, void* a_hi, void* a_lo, void* work, int n, int h, int w,
                               float max_residue, cudaStream_t stream);
int launch_dcn_scatter_backward(const float* da, void* work, float* dx, int n, int h, int w, cudaStream_t stream);

int launch_focal_attention(const void* qkv, const void* qkv_pooled, void* out, int b, int t, int h, int w, int heads,
                           int head_dim, int wh, int ww, int eh, int ew, int fh, int fw, int use_pooled, float scale,
                           int out_dtype, cudaStream_t stream);

int launch_t2t_unfold(const float* img, float* tok, void* tok_hi, void* tok_lo, int bt, int c, int h, int w, int k,
                      int s, int p, int gelu, int nhwc, cudaStream_t stream);
int launch_upsample2x_split(const float* x, void* hi, void* lo, int n, int h, int w, int c, cudaStream_t stream);
int launch_layernorm_split(const float* x, const float* gamma, const float* beta, float* out, void* hi, void* lo,
                           long long rows, int c, float eps, cudaStream_t stream);
int launch_layernorm_pool_split(const float* x, const float* gamma, const float* beta, const float* pool_w,
                                const float* pool_b, void* hi, void* lo, int bt, int h, int w, int c, int wh, int ww,
                                float eps, cudaStream_t stream);
// LayerNorm / LayerNorm + window pooling backward (layernorm_grad.cu): per-CTA partial rows of the parameter gradients
// in `work` (the *_work_elems floats), added in a fixed order by a second launch.
long long layernorm_backward_work_elems(long long rows);
long long layernorm_pool_backward_work_elems(int bt, int h, int w, int wh, int ww);
int launch_layernorm_backward(const float* x, const float* dy, const float* gamma, const float* res, float* out, void* hi,
                              void* lo, float* dgamma, float* dbeta, float* work, long long rows, int c, float eps,
                              cudaStream_t stream);
int launch_layernorm_pool_backward(const float* x, const float* gamma, const float* beta, const float* pool_w,
                                   const float* drows, const float* dx1, float* out, float* dgamma, float* dbeta,
                                   float* dpool_w, float* dpool_b, float* work, int bt, int h, int w, int c, int wh,
                                   int ww, float eps, cudaStream_t stream);
int launch_window_pool(const void* xh, const void* xl, const float* weight, const float* bias, float* out, void* out_hi,
                       void* out_lo, int bt, int h, int w, int c, int wh, int ww, cudaStream_t stream);
// gu != nullptr: the adjoint of the training forward (tin = dz, gu = its saved u); u_out != nullptr (gelu only): the
// training forward, which also writes u = the normalised values before GELU.  Both [BT][L][C*k*k] fp32.
int launch_t2t_fold_unfold(const float* tin, float* tok, void* tok_hi, void* tok_lo, int bt, int c, int h, int w, int k,
                           int s, int p, int gelu, int out_pitch, cudaStream_t stream, const float* gu = nullptr,
                           float* u_out = nullptr);
int launch_t2t_fold_nhwc(const float* tok, const float* bias, const float* residual, float* img, int bt, int c, int h,
                         int w, int k, int s, int p, int normalize, cudaStream_t stream);
int launch_t2t_fold(const float* tok, const float* bias, float* img, int bt, int c, int h, int w, int k, int s,
                    int p, int normalize, cudaStream_t stream);

int launch_split_bf16(const float* x, void* hi, void* lo, long long n, cudaStream_t stream);
int launch_linear_bf16x3(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                         const float* residual, void* out, int m, int n, int k, int out_dtype, cudaStream_t stream);
// Focal attention backward (focal_attn_grad.cu): workspace size in floats (negative: argument error), the (window, key
// slot, multiplicity) sources of one key token, and the launch.
long long focal_attention_backward_work_elems(int b, int t, int h, int w, int heads, int wh, int ww, int eh, int ew,
                                              int fh, int fw, int use_pooled);
int focal_attention_key_sources(int t_count, int h, int w, int wh, int ww, int eh, int ew, int fh, int fw,
                                int use_pooled, int t, int pooled, int y, int x, int* win, int* slot, int* mult, int cap);
int launch_focal_attention_backward(const void* qkv, const void* qkv_pooled, const float* dout, float* dqkv,
                                    float* dqkv_pooled, float* work, int b, int t, int h, int w, int heads, int wh,
                                    int ww, int eh, int ew, int fh, int fw, int use_pooled, float scale,
                                    cudaStream_t stream);
// Linear weight / bias gradient (linear_wgrad.cu): dW [n][k] = dY^T X, db [n] = column sums of dY, from the split
// dY [m][ldy] and X [m][ldx]; split-K workspace of linear_wgrad_work_elems floats (0: none needed).
int linear_wgrad_slices(int m, int n, int k);
long long linear_wgrad_work_elems(int m, int n, int k);
int launch_linear_wgrad(const void* dy_hi, const void* dy_lo, int ldy, const void* x_hi, const void* x_lo, int ldx, float* dw,
                        float* db, float* work, int m, int n, int k, cudaStream_t stream);

// Optional generalised geometry of the implicit-GEMM conv ("gather conv", see conv.cu Params): explicit tap offsets,
// output phases and tile shape.  nullptr = the plain k x k / stride / pad conv.
struct ConvGeom {
  int grid_h, grid_w;            // GEMM grid (per phase): one accumulator row per grid pixel
  int out_h, out_w;              // output image; grid pixel (y, x) of phase ph -> (y*ostep + ph_oy[ph], x*ostep + ph_ox[ph])
  int tile_w, tile_h;            // grid pixels per tile, tile_w * tile_h <= 128
  int ntaps, nphase, ostep;
  const int8_t* tap_dy;          // [ntaps] input offset of tap i relative to (y*stride, x*stride)
  const int8_t* tap_dx;
  const uint8_t* ph_tap0;        // [nphase + 1]
  const uint8_t* ph_oy;          // [nphase]
  const uint8_t* ph_ox;
  const float* bias_map;         // fp32 [out_h][out_w][cout] or null
  const long long* src_nstride;  // [nsrc] pixels between consecutive images of each source (0 / null = dense)
  long long out_nstride;         // pixels between consecutive images of every output and of the residual (0 = dense)
};
int launch_conv3x3(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_channels,
                   const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* out,
                   void* out_hi, void* out_lo, int n, int h_in, int w_in, int cout, int groups, float slope, int ks,
                   int stride, int pad, int in_rows, int out_lead, cudaStream_t stream, const ConvGeom* geom = nullptr,
                   int epi_flags = 0,      // 1: tanh, 2: NCHW fp32 output (3-channel output conv only)
                   const void* dact = nullptr, int dact_lead = 0,    // LeakyReLU(dact_slope) derivative at dact (bf16,
                   float dact_slope = 0.f);                          // Cout channels; row-gapped with that lead, or
                                                                     // dense when 0); slope 0: ReLU
int launch_conv_kxn(int nsrc, const void* const* src_hi, const void* const* src_lo, const int* src_c, const void* w_hi,
                    const void* w_lo, const float* bias, const float* residual, float* out, void* out_hi, void* out_lo, int n,
                    int h, int w, int cout, int groups, int co_pad, int ks, float slope, int flags, cudaStream_t stream);
int conv_rows_tail(int lead, int channels);
int conv_rows_pitch(int w, int lead, int channels);
int launch_pack_rows(const float* x, void* hi, void* lo, int n, int c, int h, int w, int cin, int lead,
                     cudaStream_t stream);

int launch_conv3d(const void* src_hi, const void* src_lo, int cin, int in_rows, const void* w_hi, const void* w_lo,
                  const float* bias, float* out, void* out_hi, void* out_lo, int out_cs, int b, int t_in, int h_in,
                  int w_in, int cout, int ks, int stride, const int* pad, float slope, cudaStream_t stream);
int launch_dis_conv(const void* src_hi, const void* src_lo, int cin, const void* w_hi, const void* w_lo, const float* bias,
                    float* out, void* out_hi, void* out_lo, int b, int t, int h_src, int w_src, int h_out, int w_out,
                    int cout, int pad, int transposed, float slope, const void* dact, float dact_slope, cudaStream_t stream);
int dis_wgrad_slices(int b, int t, int h_o, int w_o, int cout, int cin);
long long dis_wgrad_work_elems(int b, int t, int h_o, int w_o, int cout, int cin);
int launch_dis_wgrad(const float* dy, const void* x_hi, const void* x_lo, float* dw, float* db, float* work, int b, int t,
                     int h_in, int w_in, int cin, int h_o, int w_o, int cout, int pad, cudaStream_t stream);
// SPyNet's 7x7 / stride 1 / pad 3 convs: weight (+ bias) gradient from dy fp32 [n][h][w][cout] and the forward's operand
// x (dense [n][h][w][cin], or row-gapped with x_lead > 0).
long long conv2d_wgrad_work_elems(int n, int h, int w, int cin, int cout);
int launch_conv2d_wgrad(const float* dy, const void* x_hi, const void* x_lo, int x_lead, float* dw, float* db, float* work,
                        int n, int h, int w, int cin, int cout, cudaStream_t stream);
// Encoder / decoder backward (3x3 / pad 1 convs, stride 1 or 2): input gradient on the implicit-GEMM conv (conv.cu,
// also the k = 7 / stride 1 case), weight gradient on the split-K GEMM (dis_wgrad.cu), element-wise adjoints
// (encdec_grad.cu).  See include/e2fgvi_b200.h for the operand layouts.
int launch_conv_dgrad(const void* dy_hi, const void* dy_lo, int dy_c, int dy_lead, const void* w_hi, const void* w_lo,
                      const void* act, const float* residual, float* dx, void* dx_hi, void* dx_lo, int n, int h_in,
                      int w_in, int cin, int groups, int ks, int stride, cudaStream_t stream);
long long conv3x3_wgrad_work_elems(int n, int h_in, int w_in, int cig, int cout, int groups, int stride);
int launch_conv3x3_wgrad(const float* dy, int nsrc, const void* const* x_hi, const void* const* x_lo, const int* x_c,
                         int x_lead, float* dw, float* db, float* work, int n, int h_in, int w_in, int cout, int groups,
                         int stride, cudaStream_t stream);
int launch_upsample2x_backward(const float* dy, const float* act, float* dx, void* hi, void* lo, int n, int h, int w, int c,
                               float slope, cudaStream_t stream);
int launch_tanh_backward_rows(const float* dout, const float* out, float* dy32, void* hi, void* lo, int n, int c, int h, int w,
                              int lead, cudaStream_t stream);
int launch_leaky_backward(const float* dy, const float* act, float* dx, void* hi, void* lo, long long count, float slope,
                          cudaStream_t stream);
constexpr int I3D_STEM_TAIL = 16;         // zero pixels after the stem operand's last row (the last window's overrun)
long long i3d_stem_elems(int b, int t, int h, int w);
int launch_i3d_stem_pack(const void* x, int x_u8, void* hi, void* lo, int b, int t, int h, int w, cudaStream_t stream);
int launch_i3d_stem_conv(const void* hi, const void* lo, const void* w_hi, const void* w_lo, const float* bias, float* out,
                         void* out_hi, void* out_lo, int out_cs, int b, int t, int h, int w, int cout, cudaStream_t stream);
int launch_i3d_maxpool(const float* x, float* out, void* out_hi, void* out_lo, int b, int t, int h, int w, int c,
                       const int* k, const int* s, const int* pad, cudaStream_t stream);
int launch_i3d_mean(const float* x, float* out, int b, int t, int h, int w, int c, cudaStream_t stream);

int frame_metrics_tiles(int w, int win);
size_t frame_metrics_smem(int c, int win);            // all of the kernel's shared memory (dynamic; no static)
long long frame_sse_blocks(int h, int w, int c);
int launch_frame_sse(const void* a, int a_u8, const void* b, int b_u8, double* sse, double* work, int n, int h, int w,
                     int c, cudaStream_t stream);
int launch_frame_metrics(const void* a, int a_u8, const void* b, int b_u8, double* sse, double* ssim, double* work,
                         int n, int h, int w, int c, int win, double data_range, cudaStream_t stream);

int launch_spynet_pyramid(const float* frames, float* pyr, int b, int t, int lt, int H, int W, int h, int w, int hu, int wu,
                          const float* mean3, const float* std3, cudaStream_t stream);
int launch_spynet_level_input(const float* img, const float* prev, void* hi, void* lo, float* flow_up, int b, int lt, int hk,
                              int wk, int lead, cudaStream_t stream);
int launch_spynet_pyramid_unit(const float* frames, float* pyr, int b, int t, int lt, int H, int W, int h, int w, int hu,
                               int wu, const float* mean3, const float* std3, cudaStream_t stream);
int launch_spynet_final(const float* flow, float* out_fwd, float* out_bwd, int b, int lt, int h, int w, int hu, int wu,
                        cudaStream_t stream);
int launch_spynet_level_input_backward(const float* d_in, const float* dflow, const float* img, const float* flow_up,
                                       float* dprev, int b, int lt, int hk, int wk, cudaStream_t stream);
int launch_spynet_final_backward(const float* d_fwd, const float* d_bwd, float* dflow, int b, int lt, int h, int w, int hu,
                                 int wu, cudaStream_t stream);

int launch_video_prepare_clip(const uint8_t* frames, const uint8_t* masks, const int* ids, float* out, int t, int h,
                              int w, int hp, int wp, cudaStream_t stream);
int launch_video_compose(const float* pred, const uint8_t* frames, const uint8_t* masks, const int* ids, uint8_t* img,
                         int n_local, int h, int w, int hp, int wp, cudaStream_t stream);
int launch_video_blend(const uint8_t* img, const int* ids, const int* first, float* comp, int n_local,
                       long long frame_elems, cudaStream_t stream);
int launch_video_finalize(const float* comp, uint8_t* out, long long count, cudaStream_t stream);
int launch_video_resize_bicubic(const uint8_t* src, uint8_t* dst, uint8_t* scratch, const int* xtab, int xtaps,
                                const int* ytab, int ytaps, int n, int h, int w, int h2, int w2, cudaStream_t stream);
int launch_video_prepare_masks(const uint8_t* src, uint8_t* dst, const int* rows, const int* cols, int n, int hm,
                               int wm, int h, int w, cudaStream_t stream);

}  // namespace e2f
