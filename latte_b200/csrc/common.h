// Host-side shared declarations for liblatte_b200.so (internal; the public C ABI is include/latte_b200.h).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/latte_b200.h"

namespace b200 {

// ---- error plumbing (thread-local message; negative enum codes cross the ABI) -----------------
void set_error(const char* fmt, ...);
const char* get_error();

#define B200_CHECK_CUDA(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)

#define B200_REQUIRE(cond, code, ...)   \
  do {                                  \
    if (!(cond)) {                      \
      b200::set_error(__VA_ARGS__);     \
      return (code);                    \
    }                                   \
  } while (0)

#define B200_TRY(expr)          \
  do {                          \
    int _rc = (expr);           \
    if (_rc != B200_OK) return _rc; \
  } while (0)

// ---- TMA tensor maps ---------------------------------------------------------------------------
enum TmapSwizzle { TMAP_SW_NONE = 0, TMAP_SW_32 = 1, TMAP_SW_64 = 2, TMAP_SW_128 = 3 };

// rank-R tiled map over 16-bit elements. dims[0] is the contiguous dimension; strides_bytes[i] is the
// byte stride of dims[i+1] (R-1 entries). box[i] in elements. OOB elements read as zero.
int make_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, TmapSwizzle sw);
int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, TmapSwizzle sw);

// ---- launch with programmatic dependent launch enabled (the kernel MUST call pdl_wait() before touching global memory)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---- device-property cache ----------------------------------------------------------------------
int current_device(int* out);   // ordinal in [0, 64)
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per DEVICE: remember it per (kernel instantiation, device ordinal)
struct PerDeviceOnce {
  bool done[64] = {};
};
#define B200_SET_SMEM_ONCE(kern, bytes)                                                                        \
  do {                                                                                                         \
    static b200::PerDeviceOnce _once;                                                                          \
    int _dev = 0;                                                                                              \
    B200_TRY(b200::current_device(&_dev));                                                                     \
    if (!_once.done[_dev]) {                                                                                   \
      B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (bytes)));       \
      _once.done[_dev] = true;                                                                                 \
    }                                                                                                          \
  } while (0)
int device_sm_count(int* out);
int check_arch();  // B200_ERR_ARCH unless the current device is sm_90 (Hopper)

// ---- kernels (launchers; all enqueue on `stream`, never synchronise) ---------------------------
struct GemmArgs {
  const void* A;        // [M, K] 16-bit row-major
  const void* W;        // [N, K] 16-bit row-major (nn.Linear weight layout)
  const float* bias;    // [N] fp32 or nullptr
  int M, N, K;
  int bf16;             // 0 = fp16 operands, 1 = bf16
  int epilogue;         // B200_EPI_*
  void* out16;          // [M, N] 16-bit   (EPI_BIAS / EPI_BIAS_GELU; EPI_GATE_RESIDUAL_STORE16: acc + bias)
  float* resid;         // [M, N] fp32 in/out (EPI_GATE_RESIDUAL): resid += gate * (acc + bias) (+ row_add)
  const float* gate;    // gate[(row / rows_per_batch) * gate_batch_stride + col]
  long long gate_batch_stride;
  int rows_per_batch;
  const float* row_add; // optional [period, N] fp32 added to resid rows: row_add[((row / row_add_div) % row_add_period) * N + col]
  int row_add_div, row_add_period;
  int block_n;          // 0 = auto
  int mn_major;         // bit 0: A is stored [K, M]; bit 1: W is stored [K, N] (N % 128 == 0).  3 = wgrad (dW[M, N] += dY[K, M]^T X[K, N]),
                        // 2 = dgrad (dX[M, N] = dY[M, K] W[K, N] with the weight in its nn.Linear [out, in] layout);
                        // 1 is rejected (no caller transposes A alone)
  unsigned long long* sk_flags;  // B200_GEMM_SK_FLAGS zeroed u64 (caller's workspace) or nullptr: enables ordered stream-K
  const void* add16;    // EPI_BIAS_ADD16: [M, N] 16-bit tensor added to the result (resnet shortcut); EPI_BIAS_MUL16: the factor
  void* out16b;         // EPI_BIAS_GELU_BOTH: [M, N] 16-bit second output = gelu_tanh(out16)
  // implicit-GEMM convolution (conv_taps > 0): A is an NHWC activation [conv_n, conv_h, conv_w, conv_c] (16-bit), M =
  // conv_n*conv_h*conv_w output pixels, K = conv_taps * conv_c with W laid out [N][tap][c]; tap t reads the input pixel
  // shifted by (conv_dx[t], conv_dy[t]) with zero padding (TMA out-of-bounds fill).
  int conv_taps, conv_n, conv_h, conv_w, conv_c;
  int conv_dx[9], conv_dy[9], conv_dz[9];   // dz shifts the image index (temporal convolution over the frames of one clip)
};
// Internal epilogue (not a b200_linear value): B200_EPI_GATE_RESIDUAL plus out16[M, N] = acc + bias in 16 bits, on
// whole-K tiles (no stream-K).  LatteT2V's attention cache (b200_t2v_forward_cached) stores its entries with it.
constexpr int EPI_GATE_RESIDUAL_STORE16 = 6;
int launch_gemm(const GemmArgs& a, cudaStream_t stream);
// FP8 forward GEMM: out16[M, N] = epi(a_scale[row] * w_scale[col] * (A8[M, K] . W8[N, K]^T) + bias), both operands e4m3
// K-major, epilogue B200_EPI_BIAS or B200_EPI_BIAS_GELU, K % 16 == 0 (16-byte rows), N % 32 == 0
int launch_linear_e4m3(const void* A8, const float* a_scale, const void* W8, const float* w_scale, const float* bias, int M, int N,
                       int K, int bf16, int epilogue, void* out16, cudaStream_t stream);

struct AttnArgs {
  const void* qkv;   // [T, 3*heads*head_dim] 16-bit, row = token (b, f, n), cols [q | k | v] each [head][head_dim]
  void* out;         // [T, heads*head_dim] 16-bit
  int batch, frames, tokens;  // T = batch*frames*tokens
  int heads, head_dim;
  int bf16;
  int temporal;      // 0: sequences over tokens within a frame; 1: sequences over frames at a fixed token
  int any_len;       // spatial: 0 takes the lengths of attention_spatial_len_ok only, 1 any length >= 1
};
int launch_attention(const AttnArgs& a, cudaStream_t stream);
// spatial sequence lengths b200_attention and the ABI v7 shape rules take: a divisor of 128, 128, or a multiple of 256
// (launch_attention with any_len set takes any length >= 1)
bool attention_spatial_len_ok(int tokens);

struct CrossAttnArgs {
  const void* q;      // [batch * q_rows_per_batch, q_row_stride] 16-bit; queries are columns [head][head_dim] of each row
  const void* kv;     // [batch * kv_len, kv_row_stride] 16-bit; columns [k: head][head_dim] then [v: head][head_dim]
  void* out;          // [batch * q_rows_per_batch, heads*head_dim] 16-bit
  int batch, q_rows_per_batch, kv_len;
  int q_row_stride, kv_row_stride;  // elements
  int heads, head_dim;
  int bf16;
  const float* key_bias;  // optional [batch][128] fp32 additive score bias per key (encoder_attention_mask -> (1-m)*-10000,
                          // latte_t2v.py:766-771); entries >= kv_len are ignored
  const float* pos_bias;  // optional [heads][128][128] fp32 additive score bias per (head, query row, key) -- T5's relative
                          // position bias; needs q_rows_per_batch == 128 (one tile per sample)
  float scale;            // score scale; 0 = head_dim^-0.5 (T5 attention is unscaled: 1.0)
  int kv_batch_rows;      // rows of the K/V buffer per sample; 0 = kv_len (T5: sequences padded to 128 rows, kv_len valid)
};
int launch_cross_attention(const CrossAttnArgs& a, cudaStream_t stream);

int launch_ln_modulate(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                       int rows_per_batch, void* out16, int rows, int dim, int bf16, cudaStream_t stream);
// the same LayerNorm + modulate quantized to e4m3 with one fp32 scale per row (out8 [rows, dim] bytes, row_scale [rows])
int launch_ln_modulate_e4m3(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                            int rows_per_batch, void* out8, float* row_scale, int rows, int dim, cudaStream_t stream);
// per-row e4m3 quantization of an fp32 matrix [rows, cols]: scales[r] = amax(|row r|) / 448 (1 if zero), q = e4m3(w / s)
int launch_quantize_rows_e4m3(const float* w, int rows, int cols, void* q8, float* scales, cudaStream_t stream);
int launch_patch_embed(const float* x, int x_batch_mod, const float* w, const float* b, const float* pos, float* out,
                       int batch, int frames, int chans, int grid_h, int grid_w, int patch, int dim, int channels_first,
                       cudaStream_t stream);
int launch_t2v_mod(const float* tables, const float* ts, const float* final_table, const float* emb, float* mod, int batch,
                   int nblocks, int dim, cudaStream_t stream);
int launch_cast16(const float* in, void* out16, long long n, int bf16, cudaStream_t stream);
int launch_fill(float* p, float v, long long n, cudaStream_t stream);
// out[b][j] = act_out(W[j,:] . act_in(in[b,:]) + bias[j] (+ add[add_idx[b]][j]));  W fp32 (wbits=32) or 16-bit
int launch_gemv(const void* W, int wbits, int bf16, const float* bias, const float* in, float* out, int batch, int J,
                int K, int silu_in, int silu_out, const float* add_table, const long long* add_idx, int add_rows,
                cudaStream_t stream);
int launch_timestep_freq(const long long* t, float* out, int batch, cudaStream_t stream);
int launch_final_layer(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                       const float* w, const float* b, float* out, int batch, int frames, int grid_h, int grid_w, int patch,
                       int out_ch, int dim, int channels_first, cudaStream_t stream);
int launch_rms_norm(const float* x, const float* w, void* out16, float* out32, int rows, int dim, float eps, int bf16,
                    cudaStream_t stream);
int launch_embed(const long long* ids, const void* table16, float* x, int rows, int dim, int vocab, int bf16, cudaStream_t stream);
int launch_frames_to_uint8(const void* video, int dtype, int n, int c, int h, int w, int mode, uint8_t* out, cudaStream_t stream);
int launch_unpatchify(const float* y, float* out, int batch, int frames, int grid_h, int grid_w, int patch, int out_ch,
                      int channels_first, cudaStream_t stream);
int launch_cfg_combine(float* out, int batch, long long per_sample, int frames, int out_ch, int guided_ch, int hw,
                       float scale, cudaStream_t stream);

// training-step passes (train.cu)
int launch_transpose16(const void* in, void* out, int rows, int cols, cudaStream_t stream);
int launch_multi_cast(const void* table, int n_entries, long long total_chunks, int bf16, cudaStream_t stream);
int launch_multi_tensor(const void* table, int n_entries, long long total_chunks, int op, float a, float b, const float* scalar,
                        double* accum, cudaStream_t stream);
int launch_gate_residual(const float* x, const void* m16, const float* gate, long long gate_bs, int rows_per_batch,
                         const float* row_add, int tokens, int frames, float* out, int rows, int dim, int bf16, cudaStream_t stream);
int launch_gelu_bwd(const void* da16, const void* u16, void* du16, float* dbias, int rows, int dim, int bf16, cudaStream_t stream);
int launch_gate_bwd(const float* dx, const void* m16, const float* gate, long long gate_bs, int rows_per_batch, void* dm16,
                    float* dgate, long long dgate_bs, float* dbias, int rows, int dim, int bf16, cudaStream_t stream);
int launch_colsum(const void* a, int dtype, float* out, int rows, int dim, cudaStream_t stream);
int launch_ln_modulate_bwd(const void* dh16, const float* x, const float* scale, long long mod_bs, int rows_per_batch, float* dx,
                           float* dshift, float* dscale, long long dmod_bs, int rows, int dim, int bf16, cudaStream_t stream);
int launch_attention_bwd(const void* qkv, const void* o, const void* d_o, void* dqkv, float* stats, int batch, int frames, int tokens,
                         int heads, int head_dim, int bf16, int temporal, cudaStream_t stream);
// backward of launch_cross_attention (no pos_bias, default scale, kv_batch_rows = kv_len)
struct CrossAttnBwdArgs {
  const void* q;          // as CrossAttnArgs
  const void* kv;
  const float* key_bias;
  const void* o;          // the forward's output [batch * q_rows_per_batch, heads*head_dim] 16-bit
  const void* d_o;        // its gradient, same layout
  void* dq;               // [batch * q_rows_per_batch, heads*head_dim] 16-bit
  void* dkv;              // [batch * kv_len, dkv_row_stride] 16-bit; columns [dkv_col0, dkv_col0 + 2*heads*head_dim) are written
  int dkv_row_stride, dkv_col0;
  int batch, q_rows_per_batch, kv_len;
  int q_row_stride, kv_row_stride;
  int heads, head_dim;
  int bf16;
  void* workspace;
  size_t workspace_bytes;
};
size_t cross_attention_bwd_workspace_bytes(int batch, int q_rows_per_batch, int kv_len, int heads, int head_dim);
int launch_cross_attention_bwd(const CrossAttnBwdArgs& a, cudaStream_t stream);
int launch_ada_outer(const float* dmod, long long dmod_bs, const void* sc16, float* dW, int batch, int NA, int dim, int bf16, cudaStream_t stream);
int launch_ada_dsc(const float* dmod, long long dmod_bs, const void* w16, float* dsc, int batch, int NA, int dim, int bf16, cudaStream_t stream);

// VAE passes (vae.cu)
int launch_gn(const void* x, float* part, const float* gamma, const float* beta, void* y, int n_img, int hw, int C, int groups,
              float eps, int do_silu, int bf16, cudaStream_t stream);
int launch_upsample2x(const void* x, void* y, int n_img, int h, int w, int C, cudaStream_t stream);
int launch_conv_in(const float* z, const float* pq_w, const float* pq_b, const float* w, const float* b, void* y, int n_img, int C,
                   int h, int wd, int Cout, int bf16, cudaStream_t stream);
int launch_softmax_rows(const float* s, void* p, int rows, int n, float scale, int bf16, cudaStream_t stream);
int launch_to_nchw(const void* x, float* y, int n_img, int c, int cpad, int hw, int bf16, cudaStream_t stream);
int gemm_schedule(int M, int N, int K, int epilogue, int block_n, int sms, int* bn_out, int* pairs_out, int* streamk_out,
                  int* segments, int max_segments, int wgrad = 0);
int launch_sampler_step(const B200SamplerTables* tab, int method, int clip_denoised, const long long* t,
                        const float* x, const void* model_out, int model_out_dtype, const float* noise, int batch,
                        int frames, int channels, int hw, float* x_prev, float* pred_xstart, float* mean,
                        float* log_variance, cudaStream_t stream);
int launch_training_loss(const B200SamplerTables* tab, const long long* t, const float* x0, const float* xt, const float* noise,
                         const float* model_out, int batch, int frames, int channels, int hw, float* sums, float* dmo, cudaStream_t stream);
int launch_time_conv(const float* x, const float* w, const float* b, float* y, int frames, int c, int hw, cudaStream_t stream);

}  // namespace b200
