// extern "C" surface of liblatte_b200.so (declared in include/latte_b200.h) and the forward orchestration.
#include "common.h"

#include <mutex>
#include <vector>

namespace b200 {
namespace {

// ---- optional per-kernel-class timing (bench.py roofline): CUDA events recorded on the launching stream
// around every launch of b200_latte_forward while enabled. Off by default: zero cost, no events.
enum { PROF_GEMM = 0, PROF_ATTN = 1, PROF_LN = 2, PROF_OTHER = 3, PROF_CLASSES = 4 };
struct ProfRec { int cls; cudaEvent_t e0, e1; };
struct Profiler {
  std::mutex mu;
  bool on = false;
  std::vector<ProfRec> recs;
  std::vector<cudaEvent_t> pool;
  cudaEvent_t get() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
  }
} g_prof;

struct ProfScope {
  cudaStream_t s;
  cudaEvent_t e1 = nullptr;
  ProfScope(int cls, cudaStream_t stream) : s(stream) {
    if (!g_prof.on) return;
    std::lock_guard<std::mutex> lk(g_prof.mu);
    ProfRec r{cls, g_prof.get(), g_prof.get()};
    cudaEventRecord(r.e0, s);
    e1 = r.e1;
    g_prof.recs.push_back(r);
  }
  ~ProfScope() { if (e1) cudaEventRecord(e1, s); }
};
#define B200_PROF(cls, expr) do { ProfScope _ps(cls, stream); B200_TRY(expr); } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- workspace arena: consecutive buffers from `base`, each starting on a 1024-byte boundary; base == NULL only sizes them
struct Arena {
  uint8_t* base;
  size_t off = 0;
  template <class T>
  T* take(size_t bytes) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(bytes, 1024);
    return p;
  }
};

// ---- shape rules Latte and LatteT2V share: head_dim, the GEMM K tile, the patch grid, the operand type and the head width.
// `who` prefixes the message ("" for Latte, "t2v: " for LatteT2V).
template <class Shape>
int block_shape_ok(const char* who, const Shape* s, int batch) {
  B200_REQUIRE(s != nullptr && batch > 0, B200_ERR_SHAPE, "%sshape is NULL or batch %d is not positive", who, batch);
  B200_REQUIRE(s->heads > 0 && s->hidden % s->heads == 0, B200_ERR_SHAPE, "%shidden %d not divisible by heads %d", who, s->hidden,
               s->heads);
  const int hd = s->hidden / s->heads;
  B200_REQUIRE(hd == 64 || hd == 72 || hd == 80, B200_ERR_UNSUPPORTED, "%shead_dim %d unsupported", who, hd);
  B200_REQUIRE(s->hidden % 64 == 0 && s->mlp_hidden % 64 == 0, B200_ERR_UNSUPPORTED,
               "%shidden %d and mlp_hidden %d must be multiples of 64 (GEMM K tile)", who, s->hidden, s->mlp_hidden);
  B200_REQUIRE(s->patch > 0 && s->input_size % s->patch == 0, B200_ERR_SHAPE, "%sinput_size %d not divisible by patch %d", who,
               s->input_size, s->patch);
  // checked here so that a grid the attention does not take fails before the forward launches anything
  const int grid = s->input_size / s->patch;
  B200_REQUIRE(attention_spatial_len_ok(grid * grid), B200_ERR_UNSUPPORTED,
               "%s%d x %d patches per frame: spatial attention takes a divisor of 128, 128 or a multiple of 256 tokens", who, grid,
               grid);
  B200_REQUIRE(s->dtype == B200_FP16 || s->dtype == B200_BF16, B200_ERR_DTYPE, "%sdtype %d unknown", who, s->dtype);
  return B200_OK;
}

// ---- the forwards' two GEMM shapes.  linear16: out16[M, N] = epilogue(A[M, K] . W[N, K]^T + bias) in 16 bits
// (B200_EPI_BIAS, B200_EPI_BIAS_GELU, or B200_EPI_BIAS_MUL16, which multiplies by mul16 [M, N]).
int linear16(const void* A, const void* W, const float* bias, int M, int N, int K, int bf16, int epilogue, void* out16,
             cudaStream_t stream, const void* mul16 = nullptr) {
  GemmArgs g{};
  g.A = A; g.W = W; g.bias = bias; g.M = M; g.N = N; g.K = K; g.bf16 = bf16; g.epilogue = epilogue; g.out16 = out16; g.add16 = mul16;
  return launch_gemm(g, stream);
}

// linear_resid: the gated residual into an fp32 stream, resid[M, N] += gate[(row / rows_per_batch) * gate_bs + col] *
// (A . W^T + bias), plus row_add[((row / row_add_div) % row_add_period) * N + col] when row_add is set.
int linear_resid(const void* A, const void* W, const float* bias, int M, int N, int K, int bf16, float* resid,
                 const float* gate, long long gate_bs, int rows_per_batch, unsigned long long* sk_flags, cudaStream_t stream,
                 const float* row_add = nullptr, int row_add_div = 0, int row_add_period = 0) {
  GemmArgs g{};
  g.A = A; g.W = W; g.bias = bias; g.M = M; g.N = N; g.K = K; g.bf16 = bf16; g.epilogue = B200_EPI_GATE_RESIDUAL;
  g.resid = resid; g.gate = gate; g.gate_batch_stride = gate_bs; g.rows_per_batch = rows_per_batch; g.sk_flags = sk_flags;
  g.row_add = row_add; g.row_add_div = row_add_div; g.row_add_period = row_add_period;
  return launch_gemm(g, stream);
}

// ---- timestep embedding of n rows, both models: c = Linear(D, D)(SiLU(Linear(256, D)(tfreq = sincos(t)))) (+ y_table[y])
template <class Weights>
int timestep_embedding(const Weights* w, const int64_t* t, const float* y_table, const int64_t* y, int num_embed, int n,
                       int D, float* tfreq, float* th, float* c, cudaStream_t stream) {
  B200_PROF(PROF_OTHER, launch_timestep_freq(reinterpret_cast<const long long*>(t), tfreq, n, stream));
  B200_PROF(PROF_OTHER, launch_gemv(w->t_w0, 32, 0, w->t_b0, tfreq, th, n, D, 256, 0, 1, nullptr, nullptr, 0, stream));
  B200_PROF(PROF_OTHER, launch_gemv(w->t_w2, 32, 0, w->t_b2, th, c, n, D, D, 0, 0, y_table, reinterpret_cast<const long long*>(y),
                                    num_embed, stream));
  return B200_OK;
}

// ====================================================================================================== transformer block
// The launch sequence of one Latte block, and of each LatteT2V spatial and temporal block:
//   attention half: LN + modulate -> QKV -> self-attention -> x += gate * out-projection
//   mlp half:       LN + modulate -> fc1 (+GELU) -> x += gate * fc2 (+ row_add)
// A LatteT2V spatial block runs its cross-attention step between the two halves.

// The forward's fp32 residual stream x [T = batch*F*N, D], its scratch h [T, D] (LN + modulate output, then attention output),
// qkv [T, 3D] and g [T, mlp_hidden], and its geometry; mod_bs is the per-sample stride of the modulation rows.
struct Step {
  float* x; uint16_t* h; uint16_t* qkv; uint16_t* g; unsigned long long* sk_flags;
  int batch, F, N, heads, D, mlp_hidden;
  long long mod_bs;
  int bf16;
  cudaStream_t stream;
  int T() const { return batch * F * N; }
};

// One block's operands, offset to its layer (`layer`): weights [N, K] 16-bit or e4m3, per-channel e4m3 scales and fp32
// biases [N].  A 16-bit QKV or fc1 copy may be NULL beside an e4m3 one.
struct BlockWeights {
  const void* qkv_w16; const void* qkv_w8; const float* qkv_ws; const float* qkv_b;
  const void* out_w16; const float* out_b;
  const void* fc1_w16; const void* fc1_w8; const float* fc1_ws; const float* fc1_b;
  const void* fc2_w16; const float* fc2_b;
};

// a block's QKV and fc1 stacks each need a 16-bit copy or an e4m3 one with its per-channel scales (`who`: message prefix)
int e4m3_stacks_ok(const char* who, const BlockWeights& b) {
  B200_REQUIRE(b.qkv_w8 ? b.qkv_ws != nullptr : b.qkv_w16 != nullptr, B200_ERR_SHAPE,
               "%sqkv needs a 16-bit weight copy or an e4m3 one with its scales", who);
  B200_REQUIRE(b.fc1_w8 ? b.fc1_ws != nullptr : b.fc1_w16 != nullptr, B200_ERR_SHAPE,
               "%sfc1 needs a 16-bit weight copy or an e4m3 one with its scales", who);
  return B200_OK;
}

// layer i of the stacks [layers][...] that `stack` points at
BlockWeights layer(const BlockWeights& stack, int i, size_t D, size_t HID) {
  auto w16 = [i](const void* p, size_t n) -> const void* { return p ? static_cast<const uint16_t*>(p) + i * n : nullptr; };
  auto w8 = [i](const void* p, size_t n) -> const void* { return p ? static_cast<const uint8_t*>(p) + i * n : nullptr; };
  auto f32 = [i](const float* p, size_t n) -> const float* { return p ? p + i * n : nullptr; };
  return {w16(stack.qkv_w16, 3 * D * D), w8(stack.qkv_w8, 3 * D * D), f32(stack.qkv_ws, 3 * D), f32(stack.qkv_b, 3 * D),
          w16(stack.out_w16, D * D), f32(stack.out_b, D),
          w16(stack.fc1_w16, HID * D), w8(stack.fc1_w8, HID * D), f32(stack.fc1_ws, HID), f32(stack.fc1_b, HID),
          w16(stack.fc2_w16, D * HID), f32(stack.fc2_b, D)};
}

// LayerNorm + modulate of the residual stream, then the GEMM it feeds (QKV with B200_EPI_BIAS, fc1 with B200_EPI_BIAS_GELU)
// -> out16 [T, N].  With an e4m3 weight copy (w8, w_scale [N]) the LN output is quantized per token and the GEMM runs on
// e4m3 tensor cores; else the 16-bit LN output and weight.  The e4m3 operand and its row scales (T*D + 4T bytes) live in h
// (T*D*2 bytes), which the GEMM consumes before anything else writes h.
int ln_modulate_linear(const Step& s, const float* shift, const float* scale, const void* w16, const void* w8,
                       const float* w_scale, const float* bias, int N, int epilogue, void* out16) {
  cudaStream_t stream = s.stream;
  const int T = s.T();
  if (w8) {
    uint8_t* h8 = reinterpret_cast<uint8_t*>(s.h);
    float* h8_scale = reinterpret_cast<float*>(h8 + static_cast<size_t>(T) * s.D);
    B200_PROF(PROF_LN, launch_ln_modulate_e4m3(s.x, shift, scale, s.mod_bs, s.F * s.N, h8, h8_scale, T, s.D, stream));
    B200_PROF(PROF_GEMM, launch_linear_e4m3(h8, h8_scale, w8, w_scale, bias, T, N, s.D, s.bf16, epilogue, out16, stream));
    return B200_OK;
  }
  B200_PROF(PROF_LN, launch_ln_modulate(s.x, shift, scale, s.mod_bs, s.F * s.N, s.h, T, s.D, s.bf16, stream));
  B200_PROF(PROF_GEMM, linear16(s.h, w16, bias, T, N, s.D, s.bf16, epilogue, out16, stream));
  return B200_OK;
}

// m: the block's modulation rows [shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp], each [D]
int attention_half(const Step& s, const BlockWeights& b, const float* m, int temporal) {
  const int D = s.D;
  cudaStream_t stream = s.stream;
  B200_TRY(ln_modulate_linear(s, m + 0 * D, m + 1 * D, b.qkv_w16, b.qkv_w8, b.qkv_ws, b.qkv_b, 3 * D, B200_EPI_BIAS, s.qkv));
  AttnArgs aa{};
  aa.qkv = s.qkv; aa.out = s.h; aa.batch = s.batch; aa.frames = s.F; aa.tokens = s.N; aa.heads = s.heads; aa.head_dim = D / s.heads;
  aa.bf16 = s.bf16; aa.temporal = temporal;
  B200_PROF(PROF_ATTN, launch_attention(aa, stream));
  B200_PROF(PROF_GEMM, linear_resid(s.h, b.out_w16, b.out_b, s.T(), D, D, s.bf16, s.x, m + 2 * D, s.mod_bs, s.F * s.N, s.sk_flags,
                                    stream));
  return B200_OK;
}

// row_add: NULL, or a [frames, D] table added to every token of each frame in fc2's epilogue
int mlp_half(const Step& s, const BlockWeights& b, const float* m, const float* row_add) {
  const int D = s.D;
  cudaStream_t stream = s.stream;
  B200_TRY(ln_modulate_linear(s, m + 3 * D, m + 4 * D, b.fc1_w16, b.fc1_w8, b.fc1_ws, b.fc1_b, s.mlp_hidden, B200_EPI_BIAS_GELU,
                              s.g));
  B200_PROF(PROF_GEMM, linear_resid(s.g, b.fc2_w16, b.fc2_b, s.T(), D, s.mlp_hidden, s.bf16, s.x, m + 5 * D, s.mod_bs, s.F * s.N,
                                    s.sk_flags, stream, row_add, row_add ? s.N : 0, row_add ? s.F : 0));
  return B200_OK;
}

// ---- output head (latte.py:197-201,297-310,374-376): LayerNorm + modulate -> Linear(D, n_out = p*p*C_out) -> unpatchify.
// With a 16-bit weight copy and n_out == 32, or any n_out > 32 (patch 4 and 8), the Linear runs on the tensor cores: the
// GEMM's gated-residual epilogue on a zeroed fp32 buffer with gate = 1 IS "fp32 out = acc + bias".  n_out < 32, or 32
// without a 16-bit copy, takes the fp32 CUDA-core kernel, which holds at most 32 outputs per token.
int head_width(int patch, int out_ch) { return patch * patch * out_ch; }

// `head` workspace: the fp32 [T, n_out] buffer and its n_out ones; never smaller than the 32-wide one of patch 2
size_t head_floats(size_t T, int n_out) { return (T + 1) * (n_out > 32 ? n_out : 32); }

int head_ok(const char* who, int n_out, const void* w16) {
  B200_REQUIRE(n_out <= 32 || (n_out % 32 == 0 && w16 != nullptr), B200_ERR_UNSUPPORTED,
               "%sp*p*out_channels = %d: a head wider than 32 needs a multiple of 32 and a 16-bit weight copy", who, n_out);
  return B200_OK;
}

int output_head(const float* x, uint16_t* h, float* head, const float* shift, const float* scale, long long mod_bs,
                const float* w32, const void* w16, const float* bias, float* out, int batch, int F, int grid, int patch,
                int out_ch, int D, int bf16, int channels_first, unsigned long long* sk_flags, cudaStream_t stream) {
  const int n_out = head_width(patch, out_ch);
  const int T = batch * F * grid * grid;
  if (w16 == nullptr || n_out < 32) {
    B200_PROF(PROF_OTHER, launch_final_layer(x, shift, scale, mod_bs, w32, bias, out, batch, F, grid, patch, out_ch, D, channels_first, stream));
    return B200_OK;
  }
  float* ones = head + static_cast<size_t>(T) * n_out;
  B200_CHECK_CUDA(cudaMemsetAsync(head, 0, static_cast<size_t>(T) * n_out * 4, stream));
  B200_PROF(PROF_OTHER, launch_fill(ones, 1.0f, n_out, stream));
  B200_PROF(PROF_LN, launch_ln_modulate(x, shift, scale, mod_bs, F * grid * grid, h, T, D, bf16, stream));
  B200_PROF(PROF_GEMM, linear_resid(h, w16, bias, T, n_out, D, bf16, head, ones, 0, T, sk_flags, stream));
  B200_PROF(PROF_OTHER, launch_unpatchify(head, out, batch, F, grid, patch, out_ch, channels_first, stream));
  return B200_OK;
}

// ====================================================================================================== Latte
struct Workspace {
  float* x;          // [T, D]   fp32 residual stream, rows (b, f, n)
  uint16_t* h;       // [T, D]   16-bit: LN+modulate output, then attention output
  uint16_t* qkv;     // [T, 3D]  16-bit
  uint16_t* g;       // [T, 4D]  16-bit MLP hidden
  float* tfreq;      // [B, 256]
  float* th;         // [B, D]   SiLU(Linear(256, D))
  float* c;          // [B, D]   t_emb (+ y_emb)
  float* mod;        // [B, depth*6D + 2D]
  unsigned long long* sk_flags;   // [B200_GEMM_SK_FLAGS] stream-K ordering flags (zeroed at the start of every forward)
  float* head;       // [T, n_out] fp32 output of the head GEMM (zeroed, then reduce-added into), then n_out ones (its "gate");
                     // sized by head_floats
};

int shape_ok(const B200LatteShape* s, int batch) {
  B200_TRY(block_shape_ok("", s, batch));
  if (s->wide_patch) {
    B200_REQUIRE(s->patch == 2 || s->patch == 4 || s->patch == 8, B200_ERR_UNSUPPORTED, "patch size %d not built (2, 4, 8)",
                 s->patch);
  } else {   // the rules of ABI v6
    B200_REQUIRE(s->patch == 2, B200_ERR_UNSUPPORTED, "patch size %d not built (only 2; 4 and 8 need wide_patch)", s->patch);
    B200_REQUIRE(s->out_channels * s->patch * s->patch <= 32, B200_ERR_UNSUPPORTED, "p*p*out_channels > 32");
  }
  B200_REQUIRE(s->depth > 0 && s->depth % 2 == 0, B200_ERR_SHAPE, "depth %d must be even (spatial/temporal pairs)", s->depth);
  return B200_OK;
}

// carves `base` (NULL: sizes only) and returns the bytes it needs
size_t carve(const B200LatteShape* s, int batch, void* base, Workspace* ws) {
  const size_t grid = s->input_size / s->patch;
  const size_t B = batch, T = B * s->frames * grid * grid, D = s->hidden;
  Arena a{static_cast<uint8_t*>(base)};
  ws->x = a.take<float>(T * D * 4);
  ws->h = a.take<uint16_t>(T * D * 2);
  ws->qkv = a.take<uint16_t>(T * 3 * D * 2);
  ws->g = a.take<uint16_t>(T * s->mlp_hidden * 2);
  ws->tfreq = a.take<float>(B * 256 * 4);
  ws->th = a.take<float>(B * D * 4);
  ws->c = a.take<float>(B * D * 4);
  ws->mod = a.take<float>(B * (s->depth * 6 * D + 2 * D) * 4);
  ws->sk_flags = a.take<unsigned long long>(static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8);
  ws->head = a.take<float>(head_floats(T, head_width(s->patch, s->out_channels)) * 4);
  return a.off;
}

// b200_latte_conditioning's scratch: tfreq [n, 256], th [n, D], c [n, D]
size_t conditioning_scratch_bytes(const B200LatteShape* s, int n) {
  return align_up(static_cast<size_t>(n) * 256 * 4, 1024) + 2 * align_up(static_cast<size_t>(n) * s->hidden * 4, 1024);
}

// ---- conditioning, once per SAMPLE (latte.py:332-339): c = t_embedder(t) (+ y_embedder(y)); mod = adaLN(SiLU(c)) for all
// blocks and the final layer.  `n` rows; scratch tfreq [n,256], th [n,D], c [n,D]; mod [n, depth*6D + 2D].
int conditioning(const B200LatteShape* s, const B200LatteWeights* w, const int64_t* t, const int64_t* y, int n, float* tfreq,
                 float* th, float* c, float* mod, cudaStream_t stream) {
  const int D = s->hidden, mod_rows = s->depth * 6 * D + 2 * D;
  B200_TRY(timestep_embedding(w, t, s->num_embed > 0 ? w->y_table : nullptr, y, s->num_embed, n, D, tfreq, th, c, stream));
  B200_PROF(PROF_OTHER, launch_gemv(w->ada_w16, 16, s->dtype == B200_BF16, w->ada_b, c, mod, n, mod_rows, D, 1, 0, nullptr,
                                    nullptr, 0, stream));
  return B200_OK;
}

// premod != NULL: the caller already holds this batch's conditioning rows (b200_latte_conditioning, e.g. for a whole
// sampling trajectory at once -- SURVEY.md 8f rank 2); t is then unused and the adaLN weights are not read.
int forward(const B200LatteShape* s, const B200LatteWeights* w, const float* x, const int64_t* t, const int64_t* y,
            const float* premod, int batch, int use_cfg, float cfg_scale, float* out, void* workspace,
            size_t workspace_bytes, cudaStream_t stream) {
  B200_TRY(shape_ok(s, batch));
  B200_REQUIRE(w && x && (t || premod) && out && workspace, B200_ERR_SHAPE, "NULL argument");
  B200_REQUIRE(premod || (s->num_embed > 0) == (y != nullptr && w->y_table != nullptr), B200_ERR_SHAPE,
               "labels y and y_table must be given iff num_embed > 0 (extras == 2)");
  B200_REQUIRE(!premod || (reinterpret_cast<uintptr_t>(premod) & 15) == 0, B200_ERR_ALIGN, "conditioning rows must be 16-byte aligned");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, B200_ERR_ALIGN, "workspace must be 1024-byte aligned");
  const bool cfg = use_cfg != 0;
  B200_REQUIRE(!cfg || batch % 2 == 0, B200_ERR_SHAPE, "classifier-free guidance needs an even batch (got %d)", batch);
  B200_TRY(check_arch());
  Workspace ws;
  const size_t need = carve(s, batch, workspace, &ws);
  B200_REQUIRE(need <= workspace_bytes, B200_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  const BlockWeights stack{w->qkv_w16, w->qkv_w8, w->qkv_ws, w->qkv_b, w->proj_w16, w->proj_b,
                           w->fc1_w16, w->fc1_w8, w->fc1_ws, w->fc1_b, w->fc2_w16, w->fc2_b};
  B200_TRY(e4m3_stacks_ok("", stack));
  B200_TRY(head_ok("", head_width(s->patch, s->out_channels), w->final_w16));

  const int D = s->hidden, F = s->frames, depth = s->depth;
  const int grid = s->input_size / s->patch, N = grid * grid;
  const int bf16 = s->dtype == B200_BF16;
  const long long mod_bs = static_cast<long long>(depth) * 6 * D + 2 * D;

  // stream-K ordering flags: zero at the start of the step (every stream-K GEMM leaves them zero again; this memset only
  // makes the step independent of whatever the workspace held before -- a fresh allocation, an aborted run)
  B200_CHECK_CUDA(cudaMemsetAsync(ws.sk_flags, 0, static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8, stream));
  if (premod) ws.mod = const_cast<float*>(premod);
  else B200_TRY(conditioning(s, w, t, y, batch, ws.tfreq, ws.th, ws.c, ws.mod, stream));

  // ---- patch embedding + pos_embed -> fp32 residual stream (latte.py:330-331)
  B200_PROF(PROF_OTHER, launch_patch_embed(x, cfg ? batch / 2 : batch, w->patch_w, w->patch_b, w->pos_embed, ws.x, batch, F,
                              s->in_channels, s->input_size, s->patch, D, 0, stream));

  // ---- blocks (latte.py:345-368), alternately spatial and temporal; rows stay in (b, f, n) order for all of them
  const Step st{ws.x, ws.h, ws.qkv, ws.g, ws.sk_flags, batch, F, N, s->heads, D, s->mlp_hidden, mod_bs, bf16, stream};
  for (int i = 0; i < depth; ++i) {
    const float* m = ws.mod + static_cast<size_t>(i) * 6 * D;
    const BlockWeights b = layer(stack, i, D, s->mlp_hidden);
    B200_TRY(attention_half(st, b, m, i & 1));
    // x = x + temp_embed before the first temporal block (latte.py:357-358), folded into block 0's last epilogue
    B200_TRY(mlp_half(st, b, m, i == 0 ? w->temp_embed : nullptr));
  }

  // ---- final layer + unpatchify (latte.py:374-376), then guidance (latte.py:394-398)
  const float* mf = ws.mod + static_cast<size_t>(depth) * 6 * D;  // [shift, scale]
  B200_TRY(output_head(ws.x, ws.h, ws.head, mf, mf + D, mod_bs, w->final_w, w->final_w16, w->final_b, out, batch, F, grid, s->patch,
                       s->out_channels, D, bf16, 0, ws.sk_flags, stream));
  if (cfg) {
    const long long per_sample = static_cast<long long>(F) * s->out_channels * s->input_size * s->input_size;
    B200_PROF(PROF_OTHER, launch_cfg_combine(out, batch, per_sample, F, s->out_channels, s->in_channels, s->input_size * s->input_size,
                                cfg_scale, stream));
  }
  return B200_OK;
}

// ====================================================================================================== LatteT2V
struct T2VWorkspace {
  float* x; uint16_t* h; uint16_t* qkv; uint16_t* g;
  uint16_t* text16; uint16_t* cap_h; uint16_t* cap_o; uint16_t* kv_all;
  float* ones; float* tfreq; float* th; float* emb; float* ts; float* mod;
  unsigned long long* sk_flags;
  float* head;
};

int t2v_shape_ok(const B200T2VShape* s, int batch, int text_len) {
  B200_TRY(block_shape_ok("t2v: ", s, batch));
  B200_REQUIRE(s->patch == 2, B200_ERR_UNSUPPORTED, "t2v: patch size %d not built (only 2)", s->patch);
  B200_REQUIRE(s->out_channels * s->patch * s->patch <= 32, B200_ERR_UNSUPPORTED, "t2v: p*p*out_channels > 32");
  B200_REQUIRE(s->layers > 0, B200_ERR_SHAPE, "t2v: layers %d must be positive", s->layers);
  B200_REQUIRE(s->caption_channels % 64 == 0, B200_ERR_UNSUPPORTED, "t2v: caption_channels %d must be a multiple of 64",
               s->caption_channels);
  B200_REQUIRE(text_len >= 1 && text_len <= 128, B200_ERR_UNSUPPORTED, "t2v: text length %d (1..128 built)", text_len);
  const int grid = s->input_size / s->patch;
  B200_REQUIRE((s->frames * grid * grid) % 128 == 0, B200_ERR_UNSUPPORTED, "t2v: tokens per sample must be a multiple of 128");
  return B200_OK;
}

size_t t2v_carve(const B200T2VShape* s, int batch, int text_len, void* base, T2VWorkspace* ws) {
  const size_t grid = s->input_size / s->patch;
  const size_t B = batch, T = B * s->frames * grid * grid;
  const size_t D = s->hidden, R = B * text_len;
  Arena a{static_cast<uint8_t*>(base)};
  ws->x = a.take<float>(T * D * 4);
  ws->h = a.take<uint16_t>(T * D * 2);
  ws->qkv = a.take<uint16_t>(T * 3 * D * 2);
  ws->g = a.take<uint16_t>(T * s->mlp_hidden * 2);
  ws->text16 = a.take<uint16_t>(R * s->caption_channels * 2);
  ws->cap_h = a.take<uint16_t>(R * D * 2);
  ws->cap_o = a.take<uint16_t>(R * D * 2);
  ws->kv_all = a.take<uint16_t>(R * s->layers * 2 * D * 2);
  ws->ones = a.take<float>(D * 4);
  ws->tfreq = a.take<float>(B * 256 * 4);
  ws->th = a.take<float>(B * D * 4);
  ws->emb = a.take<float>(B * D * 4);
  ws->ts = a.take<float>(B * 6 * D * 4);
  ws->mod = a.take<float>(B * (s->layers * 2 * 6 * D + 2 * D) * 4);
  ws->sk_flags = a.take<unsigned long long>(static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8);
  ws->head = a.take<float>(head_floats(T, head_width(s->patch, s->out_channels)) * 4);
  return a.off;
}

int t2v_forward(const B200T2VShape* s, const B200T2VWeights* w, const float* x, const int64_t* t, const float* text,
                const float* text_bias, int batch, int text_len, int enable_temporal, float* out, void* workspace,
                size_t workspace_bytes, cudaStream_t stream) {
  B200_TRY(t2v_shape_ok(s, batch, text_len));
  B200_REQUIRE(w && x && t && text && out && workspace, B200_ERR_SHAPE, "t2v: NULL argument");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, B200_ERR_ALIGN, "t2v: workspace must be 1024-byte aligned");
  B200_TRY(check_arch());
  T2VWorkspace ws;
  const size_t need = t2v_carve(s, batch, text_len, workspace, &ws);
  B200_REQUIRE(need <= workspace_bytes, B200_ERR_WORKSPACE, "t2v: workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  const BlockWeights spatial{w->s_qkv_w16, w->s_qkv_w8, w->s_qkv_ws, w->s_qkv_b, w->s_out_w16, w->s_out_b,
                             w->s_fc1_w16, w->s_fc1_w8, w->s_fc1_ws, w->s_fc1_b, w->s_fc2_w16, w->s_fc2_b};
  const BlockWeights temporal{w->t_qkv_w16, w->t_qkv_w8, w->t_qkv_ws, w->t_qkv_b, w->t_out_w16, w->t_out_b,
                              w->t_fc1_w16, w->t_fc1_w8, w->t_fc1_ws, w->t_fc1_b, w->t_fc2_w16, w->t_fc2_b};
  B200_TRY(e4m3_stacks_ok("t2v: s_", spatial));
  B200_TRY(e4m3_stacks_ok("t2v: t_", temporal));
  B200_TRY(head_ok("t2v: ", head_width(s->patch, s->out_channels), w->final_w16));

  const int D = s->hidden, H = s->heads, F = s->frames, L = s->layers, HID = s->mlp_hidden;
  const int grid = s->input_size / s->patch, N = grid * grid;
  const int T = batch * F * N, R = batch * text_len;
  const int bf16 = s->dtype == B200_BF16;
  const long long mod_bs = static_cast<long long>(L) * 2 * 6 * D + 2 * D;

  B200_CHECK_CUDA(cudaMemsetAsync(ws.sk_flags, 0, static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8, stream));
  // ---- conditioning (latte_t2v.py:782-784): emb = TimestepEmbedding(sincos(t)); ts = Linear(SiLU(emb)); tables + ts
  B200_TRY(timestep_embedding(w, t, nullptr, nullptr, 0, batch, D, ws.tfreq, ws.th, ws.emb, stream));
  B200_PROF(PROF_OTHER, launch_gemv(w->ada_w16, 16, bf16, w->ada_b, ws.emb, ws.ts, batch, 6 * D, D, 1, 0, nullptr, nullptr, 0, stream));
  B200_PROF(PROF_OTHER, launch_t2v_mod(w->tables, ws.ts, w->final_table, ws.emb, ws.mod, batch, 2 * L, D, stream));
  B200_PROF(PROF_OTHER, launch_fill(ws.ones, 1.0f, D, stream));

  // ---- text: caption projection once per sample (latte_t2v.py:789), then K/V of EVERY layer's cross-attention in one GEMM
  B200_PROF(PROF_OTHER, launch_cast16(text, ws.text16, static_cast<long long>(R) * s->caption_channels, bf16, stream));
  B200_PROF(PROF_GEMM, linear16(ws.text16, w->cap_w1_16, w->cap_b1, R, D, s->caption_channels, bf16, B200_EPI_BIAS_GELU, ws.cap_h, stream));
  B200_PROF(PROF_GEMM, linear16(ws.cap_h, w->cap_w2_16, w->cap_b2, R, D, D, bf16, B200_EPI_BIAS, ws.cap_o, stream));
  B200_PROF(PROF_GEMM, linear16(ws.cap_o, w->c_kv_w16, w->c_kv_b, R, L * 2 * D, D, bf16, B200_EPI_BIAS, ws.kv_all, stream));

  // ---- patch embedding + pos_embed (latte_t2v.py:731,773); x arrives as (b c f h w)
  B200_PROF(PROF_OTHER, launch_patch_embed(x, batch, w->patch_w, w->patch_b, w->pos_embed, ws.x, batch, F, s->in_channels,
                                           s->input_size, s->patch, D, 1, stream));

  const Step st{ws.x, ws.h, ws.qkv, ws.g, ws.sk_flags, batch, F, N, H, D, HID, mod_bs, bf16, stream};
  const size_t DD = static_cast<size_t>(D) * D;
  for (int l = 0; l < L; ++l) {
    // ------------------------------------------------ spatial block (diffusers BasicTransformerBlock; latte_t2v.py:862-870)
    const float* m = ws.mod + static_cast<size_t>(2 * l) * 6 * D;
    const BlockWeights sb = layer(spatial, l, D, HID);
    B200_TRY(attention_half(st, sb, m, 0));
    // cross-attention on the UN-normalised stream (no norm2 before attn2 in ada_norm_single mode), residual without gate
    B200_PROF(PROF_OTHER, launch_cast16(ws.x, ws.h, static_cast<long long>(T) * D, bf16, stream));
    B200_PROF(PROF_GEMM, linear16(ws.h, static_cast<const uint16_t*>(w->c_q_w16) + l * DD, w->c_q_b + static_cast<size_t>(l) * D, T, D,
                                  D, bf16, B200_EPI_BIAS, ws.qkv, stream));
    CrossAttnArgs ca{};
    ca.q = ws.qkv; ca.kv = ws.kv_all + static_cast<size_t>(l) * 2 * D; ca.out = ws.h; ca.batch = batch; ca.q_rows_per_batch = F * N;
    ca.kv_len = text_len; ca.q_row_stride = D; ca.kv_row_stride = L * 2 * D; ca.heads = H; ca.head_dim = D / H; ca.bf16 = bf16;
    ca.key_bias = text_bias;     // padded prompts: (1 - mask) * -10000 per text token (latte_t2v.py:766-771), or NULL
    B200_PROF(PROF_ATTN, launch_cross_attention(ca, stream));
    B200_PROF(PROF_GEMM, linear_resid(ws.h, static_cast<const uint16_t*>(w->c_out_w16) + l * DD, w->c_out_b + static_cast<size_t>(l) * D,
                                      T, D, D, bf16, ws.x, ws.ones, 0, F * N, ws.sk_flags, stream));
    // + temp_pos_embed before the first temporal block (latte_t2v.py:894-895), folded into this epilogue
    B200_TRY(mlp_half(st, sb, m, (l == 0 && enable_temporal && F > 1) ? w->temp_embed : nullptr));
    if (!enable_temporal) continue;
    // ------------------------------------------------ temporal block (BasicTransformerBlock_, latte_t2v.py:897-905)
    const float* mt = ws.mod + static_cast<size_t>(2 * l + 1) * 6 * D;
    const BlockWeights tb = layer(temporal, l, D, HID);
    B200_TRY(attention_half(st, tb, mt, 1));
    B200_TRY(mlp_half(st, tb, mt, nullptr));
  }

  // ---- output head (latte_t2v.py:918-936): table + embedded_timestep -> shift, scale; LN; modulate; proj_out; unpatchify to (b c f h w)
  const float* mf = ws.mod + static_cast<size_t>(2 * L) * 6 * D;
  B200_TRY(output_head(ws.x, ws.h, ws.head, mf, mf + D, mod_bs, w->final_w, w->final_w16, w->final_b, out, batch, F, grid, s->patch,
                       s->out_channels, D, bf16, 1, ws.sk_flags, stream));
  return B200_OK;
}

// ====================================================================================================== T5 encoder
struct T5Workspace {
  float* x; uint16_t* h; uint16_t* qkv; uint16_t* att; uint16_t* g0; uint16_t* g; float* ones; unsigned long long* sk_flags;
};

int t5_shape_ok(const B200T5Shape* s, int batch) {
  B200_REQUIRE(s != nullptr && batch > 0, B200_ERR_SHAPE, "t5: bad shape/batch");
  B200_REQUIRE(s->layers > 0 && s->heads > 0 && s->vocab > 0, B200_ERR_SHAPE, "t5: layers/heads/vocab must be positive");
  B200_REQUIRE(s->d_model % 64 == 0 && s->d_ff % 64 == 0, B200_ERR_UNSUPPORTED, "t5: d_model %d and d_ff %d must be multiples of 64", s->d_model, s->d_ff);
  B200_REQUIRE(s->dtype == B200_FP16 || s->dtype == B200_BF16, B200_ERR_DTYPE, "t5: dtype %d unknown", s->dtype);
  return B200_OK;
}

size_t t5_carve(const B200T5Shape* s, int batch, void* base, T5Workspace* ws) {
  const size_t R = static_cast<size_t>(batch) * 128, D = s->d_model, I = static_cast<size_t>(s->heads) * 64, FF = s->d_ff;
  Arena a{static_cast<uint8_t*>(base)};
  ws->x = a.take<float>(R * D * 4);
  ws->h = a.take<uint16_t>(R * D * 2);
  ws->qkv = a.take<uint16_t>(R * 3 * I * 2);
  ws->att = a.take<uint16_t>(R * I * 2);
  ws->g0 = a.take<uint16_t>(R * FF * 2);
  ws->g = a.take<uint16_t>(R * FF * 2);
  ws->ones = a.take<float>(D * 4);
  ws->sk_flags = a.take<unsigned long long>(static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8);
  return a.off;
}

// T5Stack.forward (encoder): embed -> [T5LayerSelfAttention, T5LayerFF] x layers -> final_layer_norm (transformers
// modeling_t5.py; reached from sample/pipeline_latte.py:214).  Sequences are padded to 128 rows, so one attention tile is one
// (sample, head); masked / padding keys carry a large negative key_bias.
int t5_encode(const B200T5Shape* s, const B200T5Weights* w, const int64_t* ids, const float* key_bias, const float* pos_bias,
              int batch, float* out, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  B200_TRY(t5_shape_ok(s, batch));
  B200_REQUIRE(w && ids && pos_bias && out && workspace, B200_ERR_SHAPE, "t5: NULL argument");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, B200_ERR_ALIGN, "t5: workspace must be 1024-byte aligned");
  B200_TRY(check_arch());
  T5Workspace ws;
  const size_t need = t5_carve(s, batch, workspace, &ws);
  B200_REQUIRE(need <= workspace_bytes, B200_ERR_WORKSPACE, "t5: workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  const int R = batch * 128, D = s->d_model, H = s->heads, I = H * 64, FF = s->d_ff;
  const int bf16 = s->dtype == B200_BF16;
  B200_CHECK_CUDA(cudaMemsetAsync(ws.sk_flags, 0, static_cast<size_t>(B200_GEMM_SK_FLAGS) * 8, stream));
  B200_TRY(launch_fill(ws.ones, 1.0f, D, stream));
  B200_TRY(launch_embed(reinterpret_cast<const long long*>(ids), w->embed16, ws.x, R, D, s->vocab, bf16, stream));
  for (int l = 0; l < s->layers; ++l) {
    const uint16_t* qkv_w = static_cast<const uint16_t*>(w->qkv_w16) + static_cast<size_t>(l) * 3 * I * D;
    const uint16_t* o_w = static_cast<const uint16_t*>(w->o_w16) + static_cast<size_t>(l) * D * I;
    const uint16_t* wi0 = static_cast<const uint16_t*>(w->wi0_w16) + static_cast<size_t>(l) * FF * D;
    const uint16_t* wi1 = static_cast<const uint16_t*>(w->wi1_w16) + static_cast<size_t>(l) * FF * D;
    const uint16_t* wo = static_cast<const uint16_t*>(w->wo_w16) + static_cast<size_t>(l) * D * FF;
    // ---- T5LayerSelfAttention: x += o(attention(q, k, v of T5LayerNorm(x)) with position bias + mask, NO 1/sqrt(d) scale)
    B200_TRY(launch_rms_norm(ws.x, w->ln0_w + static_cast<size_t>(l) * D, ws.h, nullptr, R, D, s->eps, bf16, stream));
    B200_TRY(linear16(ws.h, qkv_w, nullptr, R, 3 * I, D, bf16, B200_EPI_BIAS, ws.qkv, stream));
    CrossAttnArgs ca{};
    ca.q = ws.qkv; ca.kv = ws.qkv + I; ca.out = ws.att; ca.batch = batch; ca.q_rows_per_batch = 128; ca.kv_len = 128;
    ca.kv_batch_rows = 128; ca.q_row_stride = 3 * I; ca.kv_row_stride = 3 * I; ca.heads = H; ca.head_dim = 64; ca.bf16 = bf16;
    ca.key_bias = key_bias; ca.pos_bias = pos_bias; ca.scale = 1.0f;
    B200_TRY(launch_cross_attention(ca, stream));
    B200_TRY(linear_resid(ws.att, o_w, nullptr, R, D, I, bf16, ws.x, ws.ones, 0, R, ws.sk_flags, stream));
    // ---- T5LayerFF (gated-gelu): x += wo(gelu_new(wi_0 h) * wi_1 h), h = T5LayerNorm(x)
    B200_TRY(launch_rms_norm(ws.x, w->ln1_w + static_cast<size_t>(l) * D, ws.h, nullptr, R, D, s->eps, bf16, stream));
    B200_TRY(linear16(ws.h, wi0, nullptr, R, FF, D, bf16, B200_EPI_BIAS_GELU, ws.g0, stream));
    B200_TRY(linear16(ws.h, wi1, nullptr, R, FF, D, bf16, B200_EPI_BIAS_MUL16, ws.g, stream, ws.g0));
    B200_TRY(linear_resid(ws.g, wo, nullptr, R, D, FF, bf16, ws.x, ws.ones, 0, R, ws.sk_flags, stream));
  }
  B200_TRY(launch_rms_norm(ws.x, w->final_w, nullptr, out, R, D, s->eps, bf16, stream));
  return B200_OK;
}

}  // namespace
}  // namespace b200

extern "C" {

B200_API int b200_frames_to_uint8(const void* video, int dtype, int n, int c, int h, int w, int mode, uint8_t* out, void* stream) {
  B200_TRY(b200::check_arch());
  return b200::launch_frames_to_uint8(video, dtype, n, c, h, w, mode, out, static_cast<cudaStream_t>(stream));
}

B200_API size_t b200_t5_workspace_bytes(const B200T5Shape* shape, int batch) {
  if (b200::t5_shape_ok(shape, batch) != B200_OK) return 0;
  b200::T5Workspace ws;
  return b200::t5_carve(shape, batch, nullptr, &ws);
}

B200_API int b200_t5_encode(const B200T5Shape* shape, const B200T5Weights* w, const int64_t* ids, const float* key_bias,
                            const float* pos_bias, int batch, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::t5_encode(shape, w, ids, key_bias, pos_bias, batch, out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

B200_API int b200_sampler_step(const B200SamplerTables* tables, int method, int clip_denoised, const int64_t* t,
                               const float* x, const void* model_out, int model_out_dtype, const float* noise, int batch,
                               int frames, int channels, int hw, float* x_prev, float* pred_xstart, float* mean,
                               float* log_variance, void* stream) {
  return b200::launch_sampler_step(tables, method, clip_denoised, reinterpret_cast<const long long*>(t), x, model_out,
                                   model_out_dtype, noise, batch, frames, channels, hw, x_prev, pred_xstart, mean,
                                   log_variance, static_cast<cudaStream_t>(stream));
}

B200_API int b200_training_loss(const B200SamplerTables* tables, const int64_t* t, const float* x0, const float* xt, const float* noise,
                                const float* model_out, int batch, int frames, int channels, int hw, float* sums, float* dmo, void* stream) {
  return b200::launch_training_loss(tables, reinterpret_cast<const long long*>(t), x0, xt, noise, model_out, batch, frames, channels, hw,
                                    sums, dmo, static_cast<cudaStream_t>(stream));
}

B200_API int b200_wgrad_schedule(int rows, int n_out, int n_in, int num_sms, int* block_n_out, int* pairs_out, int* streamk_out,
                                 int32_t* segments, int max_segments) {
  return b200::gemm_schedule(n_out, n_in, rows, B200_EPI_GATE_RESIDUAL, 0, num_sms, block_n_out, pairs_out, streamk_out, segments, max_segments, 1);
}

B200_API int b200_gemm_schedule(int M, int N, int K, int epilogue, int block_n, int num_sms, int* block_n_out, int* pairs_out,
                                int* streamk_out, int32_t* segments, int max_segments) {
  return b200::gemm_schedule(M, N, K, epilogue, block_n, num_sms, block_n_out, pairs_out, streamk_out, segments, max_segments);
}

B200_API void b200_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(b200::g_prof.mu);
  b200::g_prof.on = on != 0;
}

B200_API int b200_profile_collect(double* ms_per_class, int* launches_per_class, int n_classes) {
  // synchronises on the recorded events, sums elapsed time per class, then clears the records
  std::lock_guard<std::mutex> lk(b200::g_prof.mu);
  for (int i = 0; i < n_classes; ++i) { ms_per_class[i] = 0.0; launches_per_class[i] = 0; }
  for (auto& r : b200::g_prof.recs) {
    B200_CHECK_CUDA(cudaEventSynchronize(r.e1));
    float ms = 0.f;
    B200_CHECK_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
    if (r.cls < n_classes) { ms_per_class[r.cls] += ms; launches_per_class[r.cls] += 1; }
    b200::g_prof.pool.push_back(r.e0);
    b200::g_prof.pool.push_back(r.e1);
  }
  b200::g_prof.recs.clear();
  return B200_OK;
}

B200_API const char* b200_last_error(void) { return b200::get_error(); }
B200_API int b200_abi_version(void) { return B200_ABI_VERSION; }

B200_API size_t b200_latte_workspace_bytes(const B200LatteShape* shape, int batch) {
  if (b200::shape_ok(shape, batch) != B200_OK) return 0;
  b200::Workspace ws;
  return b200::carve(shape, batch, nullptr, &ws);
}

B200_API int b200_latte_forward(const B200LatteShape* shape, const B200LatteWeights* w, const float* x, const int64_t* t,
                       const int64_t* y, int batch, int use_cfg, float cfg_scale, float* out, void* workspace,
                       size_t workspace_bytes, void* stream) {
  return b200::forward(shape, w, x, t, y, nullptr, batch, use_cfg, cfg_scale, out, workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

B200_API size_t b200_latte_conditioning_bytes(const B200LatteShape* shape, int n) {
  if (b200::shape_ok(shape, n) != B200_OK) return 0;
  return static_cast<size_t>(n) * (static_cast<size_t>(shape->depth) * 6 * shape->hidden + 2 * shape->hidden) * sizeof(float);
}

B200_API size_t b200_latte_conditioning_workspace_bytes(const B200LatteShape* shape, int n) {
  if (b200::shape_ok(shape, n) != B200_OK) return 0;
  return b200::conditioning_scratch_bytes(shape, n);
}

B200_API int b200_latte_conditioning(const B200LatteShape* shape, const B200LatteWeights* w, const int64_t* t, const int64_t* y,
                                     int n, float* mod_out, void* workspace, size_t workspace_bytes, void* stream) {
  B200_TRY(b200::shape_ok(shape, n));
  B200_REQUIRE(w && t && mod_out && workspace, B200_ERR_SHAPE, "NULL argument");
  B200_REQUIRE((shape->num_embed > 0) == (y != nullptr && w->y_table != nullptr), B200_ERR_SHAPE,
               "labels y and y_table must be given iff num_embed > 0 (extras == 2)");
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(mod_out)) & 1023) == 0, B200_ERR_ALIGN,
               "workspace and mod_out must be 1024-byte aligned");
  B200_REQUIRE(workspace_bytes >= b200::conditioning_scratch_bytes(shape, n), B200_ERR_WORKSPACE, "conditioning workspace too small");
  B200_TRY(b200::check_arch());
  b200::Arena a{static_cast<uint8_t*>(workspace)};
  float* tfreq = a.take<float>(static_cast<size_t>(n) * 256 * 4);
  float* th = a.take<float>(static_cast<size_t>(n) * shape->hidden * 4);
  float* c = a.take<float>(static_cast<size_t>(n) * shape->hidden * 4);
  return b200::conditioning(shape, w, t, y, n, tfreq, th, c, mod_out, static_cast<cudaStream_t>(stream));
}

B200_API int b200_latte_forward_conditioned(const B200LatteShape* shape, const B200LatteWeights* w, const float* x,
                                            const float* mod, int batch, int use_cfg, float cfg_scale, float* out,
                                            void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(mod != nullptr, B200_ERR_SHAPE, "conditioning rows are NULL");
  return b200::forward(shape, w, x, nullptr, nullptr, mod, batch, use_cfg, cfg_scale, out, workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

B200_API int b200_linear(const void* A, const void* W, const float* bias, int M, int N, int K, int dtype, int epilogue,
                void* out16, float* resid, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                int block_n, void* sk_flags, void* stream) {
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(sk_flags) & 7) == 0, B200_ERR_ALIGN, "sk_flags must be 8-byte aligned");
  b200::GemmArgs a{};
  a.sk_flags = static_cast<unsigned long long*>(sk_flags);
  a.A = A; a.W = W; a.bias = bias; a.M = M; a.N = N; a.K = K; a.bf16 = dtype == B200_BF16; a.epilogue = epilogue;
  a.out16 = out16; a.resid = resid; a.gate = gate; a.gate_batch_stride = gate_batch_stride;
  a.rows_per_batch = rows_per_batch; a.block_n = block_n;
  return b200::launch_gemm(a, static_cast<cudaStream_t>(stream));
}

B200_API int b200_attention(const void* qkv, void* out, int batch, int frames, int tokens, int heads, int head_dim, int dtype,
                   int temporal, void* stream) {
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype);
  b200::AttnArgs a{};
  a.qkv = qkv; a.out = out; a.batch = batch; a.frames = frames; a.tokens = tokens; a.heads = heads;
  a.head_dim = head_dim; a.bf16 = dtype == B200_BF16; a.temporal = temporal;
  return b200::launch_attention(a, static_cast<cudaStream_t>(stream));
}

B200_API size_t b200_t2v_workspace_bytes(const B200T2VShape* shape, int batch, int text_len) {
  if (b200::t2v_shape_ok(shape, batch, text_len) != B200_OK) return 0;
  b200::T2VWorkspace ws;
  return b200::t2v_carve(shape, batch, text_len, nullptr, &ws);
}

B200_API int b200_t2v_forward(const B200T2VShape* shape, const B200T2VWeights* w, const float* x, const int64_t* t,
                              const float* text, const float* text_bias, int batch, int text_len, int enable_temporal,
                              float* out, void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(!text_bias || (reinterpret_cast<uintptr_t>(text_bias) & 15) == 0, B200_ERR_ALIGN, "t2v: text_bias must be 16-byte aligned");
  return b200::t2v_forward(shape, w, x, t, text, text_bias, batch, text_len, enable_temporal, out, workspace, workspace_bytes,
                           static_cast<cudaStream_t>(stream));
}

B200_API int b200_cross_attention(const void* q, const void* kv, const float* key_bias, void* out, int batch, int q_rows_per_batch,
                                  int kv_len, int q_row_stride, int kv_row_stride, int heads, int head_dim, int dtype, void* stream) {
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype);
  b200::CrossAttnArgs a{};
  a.q = q; a.kv = kv; a.out = out; a.batch = batch; a.q_rows_per_batch = q_rows_per_batch; a.kv_len = kv_len;
  a.key_bias = key_bias;
  a.q_row_stride = q_row_stride; a.kv_row_stride = kv_row_stride; a.heads = heads; a.head_dim = head_dim;
  a.bf16 = dtype == B200_BF16;
  return b200::launch_cross_attention(a, static_cast<cudaStream_t>(stream));
}

B200_API int b200_ln_modulate(const float* x, const float* shift, const float* scale, int64_t mod_batch_stride,
                     int rows_per_batch, void* out16, int rows, int dim, int dtype, void* stream) {
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype);
  return b200::launch_ln_modulate(x, shift, scale, mod_batch_stride, rows_per_batch, out16, rows, dim,
                                  dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}

B200_API int b200_quantize_rows_e4m3(const float* w, int rows, int cols, void* q8, float* scales, void* stream) {
  return b200::launch_quantize_rows_e4m3(w, rows, cols, q8, scales, static_cast<cudaStream_t>(stream));
}

B200_API int b200_ln_modulate_e4m3(const float* x, const float* shift, const float* scale, int64_t mod_batch_stride,
                                   int rows_per_batch, void* out8, float* row_scale, int rows, int dim, void* stream) {
  return b200::launch_ln_modulate_e4m3(x, shift, scale, mod_batch_stride, rows_per_batch, out8, row_scale, rows, dim,
                                       static_cast<cudaStream_t>(stream));
}

B200_API int b200_linear_e4m3(const void* A8, const float* a_scale, const void* W8, const float* w_scale, const float* bias, int M,
                              int N, int K, int dtype, int epilogue, void* out16, void* stream) {
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype);
  return b200::launch_linear_e4m3(A8, a_scale, W8, w_scale, bias, M, N, K, dtype == B200_BF16, epilogue, out16,
                                  static_cast<cudaStream_t>(stream));
}

// ---- training-step passes (train.cu) ----
#define B200_DT(dtype) B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "dtype %d unknown", dtype)
B200_API int b200_wgrad(const void* dy16, const void* x16, const float* col_scale, float* dW, int rows, int n_out, int n_in, int dtype,
                        void* sk_flags, void* stream) {
  B200_DT(dtype);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(sk_flags) & 7) == 0, B200_ERR_ALIGN, "sk_flags must be 8-byte aligned");
  B200_REQUIRE(col_scale != nullptr, B200_ERR_SHAPE, "wgrad: col_scale (n_in floats, 1.0 for a plain gradient) is required");
  b200::GemmArgs a{};
  a.A = dy16; a.W = x16; a.M = n_out; a.N = n_in; a.K = rows; a.bf16 = dtype == B200_BF16; a.epilogue = B200_EPI_GATE_RESIDUAL;
  a.resid = dW; a.gate = col_scale; a.gate_batch_stride = 0; a.rows_per_batch = n_out; a.mn_major = 3;
  a.sk_flags = static_cast<unsigned long long*>(sk_flags);
  return b200::launch_gemm(a, static_cast<cudaStream_t>(stream));
}
B200_API int b200_dgrad(const void* dy16, const void* w16, void* dx16, int rows, int n_out, int n_in, int dtype, void* stream) {
  B200_DT(dtype);
  b200::GemmArgs a{};
  a.A = dy16; a.W = w16; a.M = rows; a.N = n_in; a.K = n_out; a.bf16 = dtype == B200_BF16;
  a.epilogue = B200_EPI_BIAS;
  a.out16 = dx16; a.mn_major = 2;
  return b200::launch_gemm(a, static_cast<cudaStream_t>(stream));
}
B200_API int b200_linear_gelu_both(const void* A, const void* W, const float* bias, int M, int N, int K, int dtype, void* u16, void* a16,
                                   void* stream) {
  B200_DT(dtype);
  b200::GemmArgs a{};
  a.A = A; a.W = W; a.bias = bias; a.M = M; a.N = N; a.K = K; a.bf16 = dtype == B200_BF16; a.epilogue = B200_EPI_BIAS_GELU_BOTH;
  a.out16 = u16; a.out16b = a16;
  return b200::launch_gemm(a, static_cast<cudaStream_t>(stream));
}
B200_API int b200_transpose16(const void* in16, void* out16, int rows, int cols, void* stream) {
  return b200::launch_transpose16(in16, out16, rows, cols, static_cast<cudaStream_t>(stream));
}
B200_API int b200_multi_cast(const void* table, int n_entries, int64_t total_chunks, int dtype, void* stream) {
  B200_DT(dtype);
  return b200::launch_multi_cast(table, n_entries, total_chunks, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_multi_tensor(const void* table, int n_entries, int64_t total_chunks, int op, float a, float b, const float* scalar,
                               double* accum, void* stream) {
  return b200::launch_multi_tensor(table, n_entries, total_chunks, op, a, b, scalar, accum, static_cast<cudaStream_t>(stream));
}
B200_API int b200_cast16(const float* in, void* out16, int64_t n, int dtype, void* stream) {
  B200_DT(dtype);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out16) & 7) == 0, B200_ERR_ALIGN, "cast16: misaligned pointer");
  return b200::launch_cast16(in, out16, n, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_gate_residual(const float* x, const void* m16, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                                const float* row_add, int tokens, int frames, float* out, int rows, int dim, int dtype, void* stream) {
  B200_DT(dtype);
  return b200::launch_gate_residual(x, m16, gate, gate_batch_stride, rows_per_batch, row_add, tokens, frames, out, rows, dim,
                                    dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_gelu_bwd(const void* da16, const void* u16, void* du16, float* dbias, int rows, int dim, int dtype, void* stream) {
  B200_DT(dtype);
  return b200::launch_gelu_bwd(da16, u16, du16, dbias, rows, dim, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_gate_bwd(const float* dx, const void* m16, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                           void* dm16, float* dgate, int64_t dgate_batch_stride, float* dbias, int rows, int dim, int dtype,
                           void* stream) {
  B200_DT(dtype);
  return b200::launch_gate_bwd(dx, m16, gate, gate_batch_stride, rows_per_batch, dm16, dgate, dgate_batch_stride, dbias, rows, dim,
                               dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_colsum(const void* a, int a_dtype, float* out, int rows, int dim, void* stream) {
  return b200::launch_colsum(a, a_dtype, out, rows, dim, static_cast<cudaStream_t>(stream));
}
B200_API int b200_ln_modulate_bwd(const void* dh16, const float* x, const float* scale, int64_t mod_batch_stride, int rows_per_batch,
                                  float* dx, float* dshift, float* dscale, int64_t dmod_batch_stride, int rows, int dim, int dtype,
                                  void* stream) {
  B200_DT(dtype);
  return b200::launch_ln_modulate_bwd(dh16, x, scale, mod_batch_stride, rows_per_batch, dx, dshift, dscale, dmod_batch_stride, rows,
                                      dim, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_attention_bwd(const void* qkv16, const void* o16, const void* do16, void* dqkv16, float* stats, int batch,
                                int frames, int tokens, int heads, int head_dim, int dtype, int temporal, void* stream) {
  B200_DT(dtype);
  B200_TRY(b200::check_arch());
  return b200::launch_attention_bwd(qkv16, o16, do16, dqkv16, stats, batch, frames, tokens, heads, head_dim, dtype == B200_BF16,
                                    temporal, static_cast<cudaStream_t>(stream));
}
B200_API size_t b200_cross_attention_bwd_workspace_bytes(int batch, int q_rows_per_batch, int kv_len, int heads, int head_dim) {
  return b200::cross_attention_bwd_workspace_bytes(batch, q_rows_per_batch, kv_len, heads, head_dim);
}
B200_API int b200_cross_attention_bwd(const void* q, const void* kv, const float* key_bias, const void* o16, const void* do16, void* dq16,
                                      void* dkv16, int dkv_row_stride, int dkv_col0, int batch, int q_rows_per_batch, int kv_len,
                                      int q_row_stride, int kv_row_stride, int heads, int head_dim, int dtype, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  B200_DT(dtype);
  B200_TRY(b200::check_arch());
  b200::CrossAttnBwdArgs a{};
  a.q = q; a.kv = kv; a.key_bias = key_bias; a.o = o16; a.d_o = do16; a.dq = dq16; a.dkv = dkv16;
  a.dkv_row_stride = dkv_row_stride; a.dkv_col0 = dkv_col0;
  a.batch = batch; a.q_rows_per_batch = q_rows_per_batch; a.kv_len = kv_len;
  a.q_row_stride = q_row_stride; a.kv_row_stride = kv_row_stride; a.heads = heads; a.head_dim = head_dim;
  a.bf16 = dtype == B200_BF16;
  a.workspace = workspace; a.workspace_bytes = workspace_bytes;
  return b200::launch_cross_attention_bwd(a, static_cast<cudaStream_t>(stream));
}
B200_API int b200_ada_outer(const float* dmod, int64_t dmod_batch_stride, const void* sc16, float* dW, int batch, int NA, int dim,
                            int dtype, void* stream) {
  B200_DT(dtype);
  return b200::launch_ada_outer(dmod, dmod_batch_stride, sc16, dW, batch, NA, dim, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
B200_API int b200_ada_dsc(const float* dmod, int64_t dmod_batch_stride, const void* w16, float* dsc, int batch, int NA, int dim,
                          int dtype, void* stream) {
  B200_DT(dtype);
  return b200::launch_ada_dsc(dmod, dmod_batch_stride, w16, dsc, batch, NA, dim, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}
#undef B200_DT

}  // extern "C"
