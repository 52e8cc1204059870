/* latte_b200 — C ABI of the H100-native (sm_90a) Latte denoiser hot path (liblatte_b200.so).
 *
 * Drop-in boundary (SURVEY.md §8b): the reference's hot path is `Latte.forward` /
 * `Latte.forward_with_cfg` (Vchitect/Latte models/latte.py:314-398), a PyTorch nn.Module.  A binding
 * (ctypes here; see INTEGRATION.md) hands this library raw DEVICE pointers owned by the caller plus the
 * caller's CUDA stream.  Rules:
 *   - plain pointers and sizes only; no torch / C++ types cross the boundary;
 *   - every function enqueues work on `stream` and returns; it never synchronises, never allocates
 *     device memory and keeps no pointer past the call; the only host state is a per-thread cache of encoded
 *     TMA descriptors (pure functions of pointer + shape) and per-device kernel attributes, so a call may be
 *     captured into a CUDA graph and replayed (tests/test_gpu_graph.py);
 *   - return value 0 = ok, negative B200_ERR_* otherwise; text via b200_last_error() (thread-local);
 *   - sm_90 (Hopper) only: any other device returns B200_ERR_ARCH. There is no CPU fallback.
 * All matrices are row-major.  "16-bit" means IEEE fp16 (dtype = B200_FP16) or bfloat16 (B200_BF16).
 */
#ifndef LATTE_B200_H
#define LATTE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 9
#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

enum {
  B200_OK = 0,
  B200_ERR_SHAPE = -1,
  B200_ERR_DTYPE = -2,
  B200_ERR_ALIGN = -3,
  B200_ERR_ARCH = -4,
  B200_ERR_WORKSPACE = -5,
  B200_ERR_CUDA = -6,
  B200_ERR_UNSUPPORTED = -7
};
enum { B200_FP16 = 0, B200_BF16 = 1 };
enum { B200_EPI_BIAS = 0, B200_EPI_BIAS_GELU = 1, B200_EPI_GATE_RESIDUAL = 2, B200_EPI_BIAS_ADD16 = 3, B200_EPI_BIAS_MUL16 = 4,
       B200_EPI_BIAS_GELU_BOTH = 5 }; /* training fc1: out16 = acc + bias (kept for the backward), aux16 (written) = gelu_tanh(out16) */

/* Model geometry: the ctor arguments of reference `Latte` (models/latte.py:208-223). */
typedef struct B200LatteShape {
  int32_t depth;        /* number of TransformerBlocks; even = spatial, odd = temporal (latte.py:345-346) */
  int32_t hidden;       /* D */
  int32_t heads;        /* H; head_dim = D / H must be 64 or in (64, 80] */
  int32_t mlp_hidden;   /* int(D * mlp_ratio) */
  int32_t patch;        /* p: 2; with wide_patch set also 4 or 8 */
  int32_t in_channels;  /* C */
  int32_t out_channels; /* 2C if learn_sigma else C */
  int32_t input_size;   /* latent H = W */
  int32_t frames;       /* F */
  int32_t num_embed;    /* rows of the label table (num_classes + 1); 0 when extras != 2 */
  int32_t dtype;        /* B200_FP16 / B200_BF16: tensor-core operand type of the packed weights */
  int32_t wide_patch;   /* (appended in ABI v7) 0: the rules of ABI v6, patch 2 and p*p*out_channels <= 32 only;
                           nonzero: patch 2, 4 or 8 (Latte-S/B/L/XL /4 and /8).  A head wider than 32 outputs
                           (p*p*out_channels 64 .. 512, a multiple of 32) needs final_w16 and runs on the tensor cores;
                           (input_size / patch)^2 must be a spatial length b200_attention takes (a divisor of 128, 128,
                           or a multiple of 256), checked before anything is launched */
} B200LatteShape;

/* Packed weights (device pointers, torch-owned).  fp32 unless noted.  `*_w16` are 16-bit copies in
 * `shape.dtype`, stacked over blocks in block order.  Names follow the reference state_dict (SURVEY.md App. B). */
typedef struct B200LatteWeights {
  const float* patch_w;    /* x_embedder.proj.weight      [D, C*p*p]                      */
  const float* patch_b;    /* x_embedder.proj.bias        [D]                             */
  const float* pos_embed;  /* pos_embed                   [N, D]                          */
  const float* temp_embed; /* temp_embed                  [F, D]                          */
  const float* t_w0;       /* t_embedder.mlp.0.weight     [D, 256]                        */
  const float* t_b0;       /* t_embedder.mlp.0.bias       [D]                             */
  const float* t_w2;       /* t_embedder.mlp.2.weight     [D, D]                          */
  const float* t_b2;       /* t_embedder.mlp.2.bias       [D]                             */
  const float* y_table;    /* y_embedder.embedding_table.weight [num_embed, D] or NULL    */
  const void* ada_w16;     /* blocks.*.adaLN_modulation.1.weight then final_layer's: [depth*6D + 2D, D] 16-bit */
  const float* ada_b;      /* matching biases             [depth*6D + 2D]                 */
  const void* qkv_w16;     /* blocks.*.attn.qkv.weight    [depth][3D, D] 16-bit (NULL allowed when qkv_w8 is set) */
  const float* qkv_b;      /*                             [depth][3D]                     */
  const void* proj_w16;    /* blocks.*.attn.proj.weight   [depth][D, D] 16-bit            */
  const float* proj_b;     /*                             [depth][D]                      */
  const void* fc1_w16;     /* blocks.*.mlp.fc1.weight     [depth][4D, D] 16-bit (NULL allowed when fc1_w8 is set) */
  const float* fc1_b;      /*                             [depth][4D]                     */
  const void* fc2_w16;     /* blocks.*.mlp.fc2.weight     [depth][D, 4D] 16-bit           */
  const float* fc2_b;      /*                             [depth][D]                      */
  const float* final_w;    /* final_layer.linear.weight   [p*p*out_channels, D]           */
  const float* final_b;    /* final_layer.linear.bias     [p*p*out_channels]              */
  const void* final_w16;   /* 16-bit copy of final_w: the head then runs LN+modulate -> wgmma GEMM (N = p*p*out_channels,
                              fp32 result) -> unpatchify; NULL keeps the fp32 CUDA-core head                 */
  /* FP8 sampling path (opt-in; NULL = the 16-bit GEMM).  e4m3 copies of qkv_w16 / fc1_w16's weights with one fp32 scale per
   * output channel, as b200_quantize_rows_e4m3 makes them.  When set, that block GEMM's LayerNorm + modulate writes e4m3
   * with one scale per token and the GEMM multiplies e4m3 on the tensor cores; every other operand stays 16-bit.
   * The 16-bit copy of a weight that has an e4m3 copy is not read.                                                      */
  const void* qkv_w8;      /* blocks.*.attn.qkv.weight    [depth][3D, D] e4m3             */
  const float* qkv_ws;     /*                             [depth][3D] scales              */
  const void* fc1_w8;      /* blocks.*.mlp.fc1.weight     [depth][4D, D] e4m3             */
  const float* fc1_ws;     /*                             [depth][4D] scales              */
} B200LatteWeights;

/* ---- LatteT2V (reference models/latte_t2v.py:444-944, HF maxin-cn/Latte-1 config: ada_norm_single, gelu-approximate,
 * attention_bias, caption_channels 4096).  Parity: the forward control flow, the temporal block, adaLN-single and the
 * mask -> bias conversion are pinned to goldens generated by the unmodified reference module (oracle/make_golden_t2v.py);
 * the diffusers 0.24.0 leaves it calls (spatial block, Attention, PatchEmbed, CaptionProjection) are shim-restated. */
typedef struct B200T2VShape {
  int32_t layers;           /* num_layers: spatial/temporal block PAIRS (28) */
  int32_t hidden;           /* num_attention_heads * attention_head_dim */
  int32_t heads;
  int32_t mlp_hidden;       /* 4 * hidden */
  int32_t patch;            /* 2 */
  int32_t in_channels;      /* 4 */
  int32_t out_channels;     /* 8 */
  int32_t input_size;       /* latent H (and W when input_width is 0; sample_size, 64 for 512 px) */
  int32_t frames;           /* video_length */
  int32_t caption_channels; /* 4096 */
  int32_t dtype;            /* B200_FP16 / B200_BF16 */
  int32_t input_width;      /* (appended in ABI v8) 0: the rules of ABI v7, a square input_size x input_size latent whose
                               (input_size / patch)^2 patches must be a spatial length of the v7 rule (a divisor of 128, 128,
                               or a multiple of 256).  > 0: the latent width; the latent is input_size x input_width (e.g.
                               40 x 64 for 320 x 512 px), any number of patches per frame, and weights.pos_embed holds the
                               table of that (input_size / patch) x (input_width / patch) grid.  Both: frames * patches per
                               frame must be a multiple of 128 */
} B200T2VShape;

/* Packed weights; `l` runs over layers. fp32 unless the name ends in 16. State-dict names in comments. */
typedef struct B200T2VWeights {
  const float* patch_w;    /* pos_embed.proj.weight [D, C*p*p] */
  const float* patch_b;
  const float* pos_embed;  /* PatchEmbed sin-cos table [N, D] of the call's patch grid, N = grid_h * grid_w */
  const float* temp_embed; /* temp_pos_embed [F, D] */
  const float* t_w0;       /* adaln_single.emb.timestep_embedder.linear_1.weight [D,256] */
  const float* t_b0;
  const float* t_w2;       /* ...linear_2.weight [D,D] */
  const float* t_b2;
  const void* ada_w16;     /* adaln_single.linear.weight [6D, D] */
  const float* ada_b;
  const void* cap_w1_16;   /* caption_projection.linear_1.weight [D, caption_channels] */
  const float* cap_b1;
  const void* cap_w2_16;   /* caption_projection.linear_2.weight [D, D] */
  const float* cap_b2;
  const float* tables;     /* scale_shift_table of every block in execution order s0,t0,s1,t1,...: [2*layers][6][D] */
  const float* final_table;/* scale_shift_table [2][D] */
  const void* s_qkv_w16;   /* transformer_blocks.l.attn1.to_q|to_k|to_v.weight stacked [l][3D, D] (NULL allowed when s_qkv_w8 is set) */
  const float* s_qkv_b;
  const void* s_out_w16;   /* ...attn1.to_out.0.weight [l][D, D] */
  const float* s_out_b;
  const void* c_q_w16;     /* ...attn2.to_q.weight [l][D, D] */
  const float* c_q_b;
  const void* c_kv_w16;    /* ...attn2.to_k|to_v.weight stacked over ALL layers [layers*2D, D] (one GEMM per step) */
  const float* c_kv_b;
  const void* c_out_w16;   /* ...attn2.to_out.0.weight [l][D, D] */
  const float* c_out_b;
  const void* s_fc1_w16;   /* ...ff.net.0.proj.weight [l][4D, D] (NULL allowed when s_fc1_w8 is set) */
  const float* s_fc1_b;
  const void* s_fc2_w16;   /* ...ff.net.2.weight [l][D, 4D] */
  const float* s_fc2_b;
  const void* t_qkv_w16;   /* temporal_transformer_blocks.l.attn1 ... (NULL allowed when t_qkv_w8 is set) */
  const float* t_qkv_b;
  const void* t_out_w16;
  const float* t_out_b;
  const void* t_fc1_w16;   /* (NULL allowed when t_fc1_w8 is set) */
  const float* t_fc1_b;
  const void* t_fc2_w16;
  const float* t_fc2_b;
  const float* final_w;    /* proj_out.weight [p*p*out_channels, D] */
  const float* final_b;
  const void* final_w16;   /* 16-bit copy of final_w (tensor-core head) or NULL */
  /* FP8 sampling path (opt-in; NULL = the 16-bit GEMM), the contract of B200LatteWeights.qkv_w8 ...: e4m3 copies of the four
   * stacks fed by LayerNorm + modulate, stacked over layers like their 16-bit copies, with one fp32 scale per output channel,
   * as b200_quantize_rows_e4m3 makes them.  When a stack's e4m3 copy is set, its LayerNorm + modulate writes e4m3 with one
   * scale per token and the GEMM multiplies e4m3 on the tensor cores; its 16-bit copy is not read and may be NULL.  Every
   * other GEMM (out-projections, attn2's query, the caption projection and K/V, fc2, the head) stays 16-bit. */
  const void* s_qkv_w8;    /* transformer_blocks.l.attn1.to_q|to_k|to_v.weight [l][3D, D] e4m3 */
  const float* s_qkv_ws;   /*                                                 [l][3D] scales */
  const void* s_fc1_w8;    /* transformer_blocks.l.ff.net.0.proj.weight       [l][4D, D] e4m3 */
  const float* s_fc1_ws;   /*                                                 [l][4D] scales */
  const void* t_qkv_w8;    /* temporal_transformer_blocks.l.attn1.to_q|to_k|to_v.weight [l][3D, D] e4m3 */
  const float* t_qkv_ws;   /*                                                 [l][3D] scales */
  const void* t_fc1_w8;    /* temporal_transformer_blocks.l.ff.net.0.proj.weight [l][4D, D] e4m3 */
  const float* t_fc1_ws;   /*                                                 [l][4D] scales */
} B200T2VWeights;

B200_API size_t b200_t2v_workspace_bytes(const B200T2VShape* shape, int batch, int text_len);

/* LatteT2V.forward (latte_t2v.py:677-941, eval):  x [batch, C, F, H, W] fp32, t [batch] int64,
 * text [batch, text_len, caption_channels] fp32 (text_len <= 128)  ->  out [batch, out_channels, F, H, W] fp32;
 * H = input_size, W = input_width (input_size when input_width is 0).
 * text_bias: NULL, or [batch, 128] fp32 = the additive cross-attention bias of encoder_attention_mask,
 * (1 - mask) * -10000 per text token (latte_t2v.py:766-771; columns >= text_len are ignored), 16-byte aligned.  */
B200_API int b200_t2v_forward(const B200T2VShape* shape, const B200T2VWeights* w, const float* x, const int64_t* t,
                              const float* text, const float* text_bias, int batch, int text_len, int enable_temporal,
                              float* out, void* workspace, size_t workspace_bytes, void* stream);

/* (ABI v9) Pyramid Attention Broadcast for b200_t2v_forward: an attention module's output is computed on some sampling
 * steps and reused on others.  One buffer per kind of attention, [layers][T][D] 16-bit in `dtype` (T = batch * frames *
 * patches per frame, rows in the forward's (b, f, n) order), holds each layer's output of the module's out-projection
 * (acc + bias), before the gate:
 *   spatial:  transformer_blocks.l.attn1, added with gate_msa
 *   temporal: temporal_transformer_blocks.l.attn1, added with its gate_msa
 *   cross:    transformer_blocks.l.attn2, added with no gate
 * Modes: COMPUTE runs the module as b200_t2v_forward does and does not touch the buffer; STORE runs it and writes its
 * pre-gate output into the buffer (whole-K GEMM tiles: the residual stream's fp32 sums may differ from COMPUTE's in
 * rounding where the out-projection's K would be split); REUSE skips LayerNorm + modulate, QKV, the attention and the
 * out-projection of every layer and adds gate * buffer into the residual stream.  A cross REUSE also skips the caption
 * projection and the text K/V GEMM.  A mode outside 0..2, a STORE or REUSE without a buffer, or a buffer that is not
 * 16-byte aligned is refused (B200_ERR_SHAPE / B200_ERR_ALIGN) before anything is launched.  */
enum { B200_CACHE_COMPUTE = 0, B200_CACHE_STORE = 1, B200_CACHE_REUSE = 2 };
typedef struct B200T2VCache {
  void* spatial;            /* [layers][T][D] 16-bit, or NULL with spatial_mode COMPUTE */
  void* temporal;
  void* cross;
  int32_t spatial_mode;     /* B200_CACHE_* */
  int32_t temporal_mode;
  int32_t cross_mode;
} B200T2VCache;

/* b200_t2v_forward with each kind of attention computed, stored or reused as `cache` says (NULL: every mode COMPUTE,
 * which is b200_t2v_forward). */
B200_API int b200_t2v_forward_cached(const B200T2VShape* shape, const B200T2VWeights* w, const float* x, const int64_t* t,
                                     const float* text, const float* text_bias, int batch, int text_len, int enable_temporal,
                                     const B200T2VCache* cache, float* out, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* softmax(q k^T / sqrt(hd) + key_bias) v with K/V from another sequence (diffusers Attention attn2, latte_t2v.py:862-870):
 * q [batch*q_rows_per_batch, q_row_stride] 16-bit (first heads*head_dim columns), kv [batch*kv_len, kv_row_stride]
 * 16-bit (columns [k heads][v heads]), kv_len <= 128 keys per sample; key_bias NULL or [batch, 128] fp32 additive bias
 * per key (broadcast over heads and queries); out [rows, heads*head_dim] 16-bit.                                  */
B200_API int b200_cross_attention(const void* q, const void* kv, const float* key_bias, void* out, int batch, int q_rows_per_batch,
                                  int kv_len, int q_row_stride, int kv_row_stride, int heads, int head_dim, int dtype, void* stream);

/* ---- T5 text encoder (SURVEY.md 8f rank 3): the reference obtains prompt embeddings from transformers' T5EncoderModel
 * (sample/pipeline_latte.py:214, `self.text_encoder(ids, attention_mask=mask)[0]`; t5-v1_1-xxl: d_model 4096, 64 heads x 64,
 * d_ff 10240 gated-GELU, 24 layers, relative position bias shared by all layers, no biases, no attention scaling).
 * Parity: oracle/t5_oracle.py is pinned to fixtures generated by transformers' own T5EncoderModel (oracle/make_golden_t5.py). */
typedef struct B200T5Shape {
  int32_t layers;
  int32_t d_model;
  int32_t heads;        /* d_kv is 64: inner = 64 * heads */
  int32_t d_ff;
  int32_t vocab;
  int32_t dtype;        /* B200_FP16 / B200_BF16 operand type of the packed weights */
  float eps;            /* layer_norm_epsilon (1e-6) */
} B200T5Shape;

typedef struct B200T5Weights {
  const void* embed16;    /* shared.weight [vocab, d_model] 16-bit                                                   */
  const void* qkv_w16;    /* block.l.layer.0.SelfAttention.q|k|v.weight stacked [l][3*inner, d_model]                */
  const void* o_w16;      /* ...SelfAttention.o.weight [l][d_model, inner]                                           */
  const float* ln0_w;     /* block.l.layer.0.layer_norm.weight [l][d_model] fp32                                     */
  const void* wi0_w16;    /* block.l.layer.1.DenseReluDense.wi_0.weight [l][d_ff, d_model] (the GELU branch)         */
  const void* wi1_w16;    /* ...wi_1.weight [l][d_ff, d_model]                                                       */
  const void* wo_w16;     /* ...wo.weight [l][d_model, d_ff]                                                         */
  const float* ln1_w;     /* block.l.layer.1.layer_norm.weight [l][d_model]                                          */
  const float* final_w;   /* final_layer_norm.weight [d_model]                                                       */
} B200T5Weights;

B200_API size_t b200_t5_workspace_bytes(const B200T5Shape* shape, int batch);
/* ids [batch, 128] int64 (sequences padded to 128 tokens; any valid id in the padding), key_bias [batch, 128] fp32 =
 * 0 for kept tokens, a large negative number for masked ones (the extended attention mask), pos_bias [heads, 128, 128]
 * fp32 = relative_attention_bias[bucket(j - i)][h] (evaluated by the caller once per model: it depends only on the
 * weights).  out [batch, 128, d_model] fp32 = last_hidden_state (rows of padding tokens are computed but meaningless). */
B200_API int b200_t5_encode(const B200T5Shape* shape, const B200T5Weights* w, const int64_t* ids, const float* key_bias,
                            const float* pos_bias, int batch, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Decoded frames -> uint8 video (SURVEY.md 8f rank 3), fused with the channels-last permute: video [n, c, h, w] in `dtype`
 * (0 fp32, 1 fp16, 2 bf16) -> out [n, h, w, c] uint8 (device).  mode 0 = sample/pipeline_latte.py:775,796
 * `((v / 2.0 + 0.5).clamp(0, 1) * 255).to(uint8)`; mode 1 = sample/sample.py:122, sample_ddp.py:172
 * `((v * 0.5 + 0.5) * 255).add_(0.5).clamp_(0, 255).to(uint8)`.  Every intermediate is rounded to `dtype` as torch does,
 * so the bytes are identical to the reference expression on the same tensor.                                          */
B200_API int b200_frames_to_uint8(const void* video, int dtype, int n, int c, int h, int w, int mode, uint8_t* out, void* stream);

/* ---- AutoencoderKL.decode (diffusers 0.24.0 SD-VAE decoder; reference call sites sample/sample.py:114,
 * sample_ddp.py:167, pipeline_latte.py:758,771).  Parity UNPINNED (diffusers absent offline).
 * Conv weights are 16-bit, repacked from OIHW to [Cout][ky*3+kx][Cin]; 1x1 shortcuts are [Cout][Cin]. */
typedef struct B200VaeResnet {
  const float* gn1_g; const float* gn1_b; const void* conv1_w16; const float* conv1_b;
  const float* gn2_g; const float* gn2_b; const void* conv2_w16; const float* conv2_b;
  const void* short_w16; const float* short_b;   /* NULL when cin == cout */
  int32_t cin, cout;
  /* AutoencoderKLTemporalDecoder only (NULL otherwise): the TemporalResnetBlock of a SpatioTemporalResBlock, Conv3d
   * (3,1,1) weights repacked [C][kt][C]; conv2 weights and bias are pre-multiplied by (1 - alpha) of the AlphaBlender,
   * so blend(x_s, x_s + conv2) == x_s + (1 - alpha) conv2 is the plain "+ shortcut" epilogue. */
  const float* t_gn1_g; const float* t_gn1_b; const void* t_conv1_w16; const float* t_conv1_b;
  const float* t_gn2_g; const float* t_gn2_b; const void* t_conv2_w16; const float* t_conv2_b;
} B200VaeResnet;

typedef struct B200VaeDecoder {
  int32_t latent_channels;      /* 4 */
  int32_t layers_per_block;     /* resnets per up block = layers_per_block + 1 (3) */
  int32_t n_up;                 /* up blocks (4) */
  int32_t up_channels[4];       /* output channels of the up blocks: 512, 512, 256, 128 */
  int32_t groups;               /* 32 */
  int32_t dtype;
  float eps;                    /* 1e-6 */
  const float* pq_w; const float* pq_b;             /* post_quant_conv [C,C], NULL to skip */
  const float* conv_in_w; const float* conv_in_b;   /* [C0, C, 3, 3] fp32 */
  B200VaeResnet mid[2];
  const float* attn_gn_g; const float* attn_gn_b;
  const void* attn_q_w16; const float* attn_q_b; const void* attn_k_w16; const float* attn_k_b;
  const void* attn_v_w16;                           /* v bias is folded into attn_o_b by the packer */
  const void* attn_o_w16; const float* attn_o_b;
  B200VaeResnet up[12];                             /* [block][resnet] row-major, 3 per block */
  const void* ups_w16[3]; const float* ups_b[3];    /* upsampler convs of blocks 0..n_up-2 */
  const float* norm_out_g; const float* norm_out_b;
  const void* conv_out_w16; const float* conv_out_b; /* rows padded to 32: [32][9][C_last], bias [32] */
  int32_t out_channels;                             /* 3 */
  float temporal_eps;                               /* GroupNorm eps of the temporal resnets (1e-5) */
  const float* time_conv_w; const float* time_conv_b; /* time_conv_out Conv3d(3,3,(3,1,1)) [3][3][3] (out, in, kt), or NULL */
} B200VaeDecoder;

B200_API size_t b200_vae_workspace_bytes(const B200VaeDecoder* d, int n_img, int h, int w);
/* z [n_img, C, h, w] fp32 (already divided by scaling_factor, as the callers do) -> out [n_img, 3, 8h, 8w] fp32 */
B200_API int b200_vae_decode(const B200VaeDecoder* d, const float* z, int n_img, int h, int w, float* out, void* workspace,
                             size_t workspace_bytes, void* stream);
/* AutoencoderKLTemporalDecoder.decode(z, num_frames) (pipeline_latte.py:779-798): the n_img frames are ONE clip
 * (n_img == num_frames, as the pipeline's 14-frame chunks are); temporal convolutions zero-pad at the clip ends. */
B200_API int b200_vae_decode_temporal(const B200VaeDecoder* d, const float* z, int n_img, int h, int w, int num_frames, float* out,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- AutoencoderKL.encode (SURVEY.md 8f rank 4; train.py:206-211 `vae.encode(x).latent_dist.sample().mul_(0.18215)`): the
 * diffusers 0.24.0 Encoder -- conv_in, n_down DownEncoderBlock2D (2 resnets each, pad (0,1,0,1) + stride-2 conv except the last),
 * mid block (resnet, 1-head attention, resnet), GroupNorm + SiLU, conv_out -- then quant_conv; the result is the moments tensor
 * [n, 2L, h/f, w/f] (mean | log-variance) of DiagonalGaussianDistribution.  Same kernels as the decoder; a stride-2 conv is a
 * space-to-depth pass + a 2x2-tap implicit GEMM over 4C channels (weights repacked by the host, see latte_b200/vae.py).       */
typedef struct B200VaeEncoder {
  int32_t in_channels;          /* 3 */
  int32_t n_down;               /* 4 */
  int32_t down_channels[4];     /* 128, 256, 512, 512 */
  int32_t groups;               /* 32 */
  int32_t dtype;
  float eps;                    /* 1e-6 */
  int32_t latent_channels;      /* L = 4: conv_out and quant_conv produce 2L channels */
  const float* conv_in_w; const float* conv_in_b;   /* [C0, in, 3, 3] fp32 */
  B200VaeResnet down[8];                            /* [block][resnet] row-major, 2 per block */
  const void* down_w16[3]; const float* down_b[3];  /* stride-2 convs: [Cout][tap = oy*2+ox][phase = py*2+px][Cin], 16-bit */
  B200VaeResnet mid[2];
  const float* attn_gn_g; const float* attn_gn_b;
  const void* attn_q_w16; const float* attn_q_b; const void* attn_k_w16; const float* attn_k_b;
  const void* attn_v_w16;                           /* v bias folded into attn_o_b by the packer */
  const void* attn_o_w16; const float* attn_o_b;
  const float* norm_out_g; const float* norm_out_b;
  const void* conv_out_w16; const float* conv_out_b; /* rows padded to 32: [32][9][C_last], bias [32] */
  const float* quant_w; const float* quant_b;        /* quant_conv [2L, 2L] fp32, NULL to skip */
} B200VaeEncoder;
B200_API size_t b200_vae_encode_workspace_bytes(const B200VaeEncoder* e, int n_img, int h, int w);
/* x [n_img, in_channels, h, w] fp32 -> moments [n_img, 2L, h/f, w/f] fp32, f = 2^(n_down-1) */
B200_API int b200_vae_encode(const B200VaeEncoder* e, const float* x, int n_img, int h, int w, float* moments, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ---- single VAE layers, through the same internal launches b200_vae_decode / b200_vae_encode use (for op-level tests and
 * for callers that assemble their own VAE).  Activations are NHWC 16-bit in `dtype`; weights are packed as by the host
 * packers in latte_b200/vae.py; bias fp32 [cout] or NULL.
 * b200_vae_conv, `kind`:
 *   B200_VAE_CONV3X3     Conv2d 3x3, padding 1: x [n_img, h, w, cin] -> out16 [n_img, h, w, cout]; w16 [cout][ky*3+kx][cin].
 *                        w >= 128: w % 128 == 0; w < 128: 128 % w == 0 and h % (128 / w) == 0.
 *   B200_VAE_CONV_T3     Conv3d (3,1,1), padding (1,0,0) over the n_img frames of ONE clip (zero padding at both ends):
 *                        cin == cout, w16 [cout][kt][cin]; same tiling rule.
 *   B200_VAE_CONV_DOWN2  Downsample2D: F.pad (0,1,0,1) then Conv2d 3x3 stride 2 on an h x w input (h, w even): out16
 *                        [n_img, h/2, w/2, cout]; w16 [cout][tap = oy*2+ox][phase = py*2+px][cin]; scratch receives the
 *                        space-to-depth input, n_img * h * w * cin 16-bit values.  add16 must be NULL.
 * add16: NULL or [n_img, h, w, cout] 16-bit, added after the 16-bit rounding of conv + bias (the resnet "+ shortcut").
 * cin % 64 == 0, cout % 32 == 0; x, out16, add16, scratch 16-byte aligned.                                              */
enum { B200_VAE_CONV3X3 = 0, B200_VAE_CONV_T3 = 1, B200_VAE_CONV_DOWN2 = 2 };
B200_API int b200_vae_conv(const void* x, const void* w16, const float* bias, const void* add16, void* out16, void* scratch, int n_img,
                           int h, int w, int cin, int cout, int kind, int dtype, void* stream);
/* GroupNorm(groups, C, eps) (+ SiLU when silu != 0) over each of n_img images of hw pixels: x, y [n_img, hw, C] 16-bit;
 * gamma, beta fp32 [C]; part: n_img * groups * 2 floats of scratch.  C / groups must be 4 or a multiple of 8, C / 8 must
 * divide 256.  The temporal decoder's GroupNorm over a clip is one image of frames * hw pixels.                         */
B200_API int b200_group_norm(const void* x, void* y, const float* gamma, const float* beta, float* part, int n_img, int hw, int C,
                             int groups, float eps, int silu, int dtype, void* stream);
/* Mid-block attention of the VAE (one head over the h*w pixels of each image):
 * out = x + to_out(softmax(q k^T / sqrt(C)) v) with q, k, v projections of GroupNorm(groups, C, eps)(x).
 * x, out [n_img, h*w, C] 16-bit; *_w16 [C, C] 16-bit nn.Linear weights; o_b = to_out bias + to_out weight . to_v bias (the
 * v bias folded in, latte_b200/vae.py fold_v_bias).  C % 64 == 0, (h*w) % 64 == 0; workspace 1024-byte aligned.          */
B200_API size_t b200_vae_mid_attention_workspace_bytes(int n_img, int h, int w, int C, int groups);
B200_API int b200_vae_mid_attention(const void* x, void* out, const float* gn_g, const float* gn_b, const void* q_w16, const float* q_b,
                                    const void* k_w16, const float* k_b, const void* v_w16, const void* o_w16, const float* o_b, int n_img,
                                    int h, int w, int C, int groups, float eps, int dtype, void* workspace, size_t workspace_bytes,
                                    void* stream);

/* Thread-local description of the last failure on this thread ("" if none). */
B200_API const char* b200_last_error(void);
B200_API int b200_abi_version(void);

/* Bytes of scratch `b200_latte_forward` needs for `batch` videos (0 on invalid shape; see b200_last_error). */
B200_API size_t b200_latte_workspace_bytes(const B200LatteShape* shape, int batch);

/* Whole denoiser forward — replaces Latte.forward (models/latte.py:314-377) and, when use_cfg != 0,
 * Latte.forward_with_cfg (latte.py:379-398: rows [0, batch/2) are the conditional half, x rows
 * [batch/2, batch) are ignored and replaced by a copy of the first half; eps channels [0, in_channels)
 * of BOTH halves become uncond + cfg_scale * (cond - uncond)).
 *   x   [batch, F, C, S, S] fp32        t [batch] int64        y [batch] int64 or NULL (extras != 2)
 *   out [batch, F, out_channels, S, S] fp32
 *   workspace: >= b200_latte_workspace_bytes(shape, batch) bytes, 1024-byte aligned.             */
B200_API int b200_latte_forward(const B200LatteShape* shape, const B200LatteWeights* w, const float* x, const int64_t* t,
                       const int64_t* y, int batch, int use_cfg, float cfg_scale, float* out, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Whole-trajectory conditioning (SURVEY.md 8f rank 2).  The per-sample conditioning -- t_embedder(t) + y_embedder(y)
 * (latte.py:332-339), every block's adaLN_modulation (:160-163,177) and the final layer's (:192-195) -- depends only on
 * (t, y), so a sampler that knows its timesteps can evaluate all of it before the loop: n = steps x batch rows here, then
 * b200_latte_forward_conditioned per step with that step's `batch` rows.  Same kernels and arithmetic as inside
 * b200_latte_forward (bit-identical output); what it saves per step is the 446 MB adaLN weight stream and 4 launches.
 *   mod_out: [n, depth*6*hidden + 2*hidden] fp32 (b200_latte_conditioning_bytes), 1024-byte aligned.            */
B200_API size_t b200_latte_conditioning_bytes(const B200LatteShape* shape, int n);
B200_API size_t b200_latte_conditioning_workspace_bytes(const B200LatteShape* shape, int n);
B200_API int b200_latte_conditioning(const B200LatteShape* shape, const B200LatteWeights* w, const int64_t* t, const int64_t* y,
                                     int n, float* mod_out, void* workspace, size_t workspace_bytes, void* stream);
B200_API int b200_latte_forward_conditioned(const B200LatteShape* shape, const B200LatteWeights* w, const float* x,
                                            const float* mod, int batch, int use_cfg, float cfg_scale, float* out,
                                            void* workspace, size_t workspace_bytes, void* stream);

/* out = epilogue(A @ W^T + bias) on wgmma tensor cores — replaces the nn.Linear calls of the block
 * (latte.py:50 qkv, :75 proj, timm Mlp fc1/fc2 via :171).  A [M,K], W [N,K] 16-bit; bias [N] fp32 or NULL.
 *   B200_EPI_BIAS           out16[M,N] = acc + bias
 *   B200_EPI_BIAS_GELU      out16[M,N] = gelu_tanh(acc + bias)                     (latte.py:169)
 *   B200_EPI_GATE_RESIDUAL  resid[M,N] (fp32, in place) += gate[row / rows_per_batch][col] * (acc + bias)
 *                           (latte.py:179-180); gate row stride = gate_batch_stride floats.
 * K % 64 == 0, N % 32 == 0 required; M arbitrary.
 * sk_flags: NULL, or B200_GEMM_SK_FLAGS 64-bit words of device memory that the caller zeroed ONCE.  With it the
 * residual epilogue may split the last waves of tiles along K across all SMs ("ordered stream-K": partial sums are
 * added into resid in k order, so results stay bit-reproducible); every launch leaves the words zero again.    */
#define B200_GEMM_SK_FLAGS 1024
B200_API int b200_linear(const void* A, const void* W, const float* bias, int M, int N, int K, int dtype, int epilogue,
                void* out16, float* resid, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                int block_n, void* sk_flags, void* stream);

/* softmax(q k^T / sqrt(hd)) v per head — replaces Attention.forward 'math' mode between the qkv and
 * proj Linears (latte.py:50-70).  qkv [T, 3*heads*head_dim] 16-bit with T = batch*frames*tokens rows in
 * (b, f, n) order; out [T, heads*head_dim] 16-bit.  temporal = 0: one sequence per (b, f) over n
 * (latte.py:353); temporal = 1: one sequence per (b, n) over f (latte.py:355-367) — no transpose pass. */
B200_API int b200_attention(const void* qkv, void* out, int batch, int frames, int tokens, int heads, int head_dim,
                   int dtype, int temporal, void* stream);

/* (ABI v8) b200_attention with temporal = 0 at ANY number of tokens per frame >= 1 (b200_attention's spatial lengths are
 * a divisor of 128, 128 or a multiple of 256): the spatial attention b200_t2v_forward runs at latents other than
 * sample_size x sample_size (e.g. 576 tokens per frame at 288 x 512 px).  head_dim 64, 72 or 80. */
B200_API int b200_spatial_attention_any(const void* qkv, void* out, int batch, int frames, int tokens, int heads, int head_dim,
                                        int dtype, void* stream);

/* out16[r, :] = LayerNorm(x[r, :]; no affine, eps 1e-6) * (1 + scale[b]) + shift[b], b = r / rows_per_batch
 * — replaces norm1/norm2 + modulate (latte.py:28-29, 166-168, 179-180). x fp32 [rows, dim].          */
B200_API int b200_ln_modulate(const float* x, const float* shift, const float* scale, int64_t mod_batch_stride,
                     int rows_per_batch, void* out16, int rows, int dim, int dtype, void* stream);

/* ---- FP8 (e4m3) sampling path.  One formula quantizes both operands, row by row:
 *   s = amax(|row|) / 448 (1 for an all-zero row),  q = e4m3_rn_satfinite(row / s)  (fp32, correctly rounded division)
 * b200_quantize_rows_e4m3: w fp32 [rows, cols] -> q8 [rows, cols] e4m3 bytes, scales [rows] fp32 (a weight W[N, K]: one
 *   scale per output channel).  cols % 16 == 0; w, q8 16-byte aligned.
 * b200_ln_modulate_e4m3: b200_ln_modulate's y (in fp32, before any 16-bit rounding) quantized per row -> out8 [rows, dim]
 *   e4m3 bytes, row_scale [rows] fp32.  dim % 16 == 0.
 * b200_linear_e4m3: out16[M, N] = epi(a_scale[row] * w_scale[col] * (A8[M, K] . W8[N, K]^T) + bias), epilogue
 *   B200_EPI_BIAS or B200_EPI_BIAS_GELU, 16-bit output in `dtype`; K % 16 == 0 (else B200_ERR_UNSUPPORTED), N % 32 == 0;
 *   A8, W8, out16, bias 16-byte aligned, w_scale 8-byte aligned.  Partial sums are kept in fp32 (DESIGN.md).            */
B200_API int b200_quantize_rows_e4m3(const float* w, int rows, int cols, void* q8, float* scales, void* stream);
B200_API int b200_ln_modulate_e4m3(const float* x, const float* shift, const float* scale, int64_t mod_batch_stride,
                                   int rows_per_batch, void* out8, float* row_scale, int rows, int dim, void* stream);
B200_API int b200_linear_e4m3(const void* A8, const float* a_scale, const void* W8, const float* w_scale, const float* bias, int M,
                              int N, int K, int dtype, int epilogue, void* out16, void* stream);

/* ---- training step (BASELINE config 5: train.py:206-222, fwd + bwd of models/latte.py under loss.backward()) -------------
 * The reference differentiates Latte.forward with torch autograd; the replacement keeps the same forward kernels, stores the
 * activations, and evaluates the analytic backward with b200_linear (every dgrad: A = dY, W = W^T; every wgrad: A = dY^T,
 * W = X^T, B200_EPI_GATE_RESIDUAL with a unit gate accumulating into the fp32 gradient) plus the passes below.  Host side:
 * latte_b200/training.py (the engine base and TrainEngine; T2VTrainEngine in training_t2v.py adds the cross-attention
 * entries).  All [rows, dim] matrices are row-major; "16" = fp16/bf16 per `dtype`.                                        */
/* dW[n_out, n_in] (fp32, in place) += col_scale[n_in] * (dY16[rows, n_out]^T . X16[rows, n_in]) -- the weight gradient of
 * Y = X W^T, reading both activations as they lie in memory (the GEMM's MN-major operand mode: no transposed copies),
 * accumulated in fp32 through the residual epilogue (sk_flags as in b200_linear).  col_scale: n_in floats, 1.0 for a plain
 * gradient (a loss-scale / per-column factor otherwise).  rows % 64 == 0, n_out % 8 == 0, n_in % 128 == 0.                */
B200_API int b200_wgrad(const void* dy16, const void* x16, const float* col_scale, float* dW, int rows, int n_out, int n_in,
                        int dtype, void* sk_flags, void* stream);
/* dX16[rows, n_in] = dY16[rows, n_out] . W16[n_out, n_in] -- the input gradient of Y = X W^T with the weight in its nn.Linear
 * [out, in] layout (MN-major W operand: no transposed weight copy).  n_out % 64 == 0, n_in % 128 == 0.                    */
B200_API int b200_dgrad(const void* dy16, const void* w16, void* dx16, int rows, int n_out, int n_in, int dtype, void* stream);
/* Training-mode fc1: u16 = A W^T + bias (kept for the backward) and a16 = gelu_tanh(u16) from the same epilogue.              */
B200_API int b200_linear_gelu_both(const void* A, const void* W, const float* bias, int M, int N, int K, int dtype, void* u16, void* a16,
                                   void* stream);
/* out16[cols, rows] = in16[rows, cols]^T (operands of shapes b200_wgrad / b200_dgrad do not take).                          */
B200_API int b200_transpose16(const void* in16, void* out16, int rows, int cols, void* stream);
/* fp32 -> 16-bit elementwise (n % 4 == 0).                                                                                */
/* The same for many tensors in ONE launch (all parameters at the start of a step).  table: device array of n_entries records
 * of four int64 {src fp32 pointer (16-byte aligned), dst 16-bit pointer (8-byte aligned), n4 = element count / 4, first_chunk}
 * with first_chunk[0] = 0, first_chunk[e+1] = first_chunk[e] + ceil(n4[e] / 1024); total_chunks = the sum.                 */
B200_API int b200_multi_cast(const void* table, int n_entries, int64_t total_chunks, int dtype, void* stream);
/* fp32 passes over a LIST of tensors in one launch -- replaces the per-parameter python loops of the reference's
 * `clip_grad_norm_` (utils.py:72-125) and `update_ema` (utils.py:190-200).  table: records of four int64 {src, dst, n elements,
 * first_chunk} with a chunk = 4096 elements (first_chunk as in b200_multi_cast).
 *   B200_MT_SUMSQ  *accum (double, device) += sum over all src of src^2        (dst unused)
 *   B200_MT_SCALE  dst *= *scalar (device float: the clamped clip coefficient, no host sync)   (src unused)
 *   B200_MT_AXPBY  dst = a * dst + b * src                                      (EMA: a = decay, b = 1 - decay)               */
enum { B200_MT_SUMSQ = 1, B200_MT_SCALE = 2, B200_MT_AXPBY = 3 };
B200_API int b200_multi_tensor(const void* table, int n_entries, int64_t total_chunks, int op, float a, float b, const float* scalar,
                               double* accum, void* stream);
B200_API int b200_cast16(const float* in, void* out16, int64_t n, int dtype, void* stream);
/* out[r] = x[r] + gate[r / rows_per_batch] * m16[r] (+ row_add[(r / tokens) % frames] when row_add != NULL): the residual
 * updates of TransformerBlock.forward (latte.py:179-180) with the branch output kept for the backward; row_add = temp_embed
 * (latte.py:357-358).                                                                                                     */
B200_API int b200_gate_residual(const float* x, const void* m16, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                                const float* row_add, int tokens, int frames, float* out, int rows, int dim, int dtype, void* stream);
/* du16 = da16 * gelu_tanh'(u16); dbias[dim] (fp32) += column sums of du = fc1.bias gradient.  (Every reduction output of the
 * training passes ACCUMULATES: the caller zeroes its gradient buffers once per step, so no pass issues a memset.)          */
B200_API int b200_gelu_bwd(const void* da16, const void* u16, void* du16, float* dbias, int rows, int dim, int dtype, void* stream);
/* backward of out = x + gate[b] * m: dm16 = dx * gate[b]; dgate[b] (row stride dgate_batch_stride) += sum over the sample's
 * rows of dx * m; dbias[dim] += column sums of dm = the bias gradient of the Linear that made m.                          */
B200_API int b200_gate_bwd(const float* dx, const void* m16, const float* gate, int64_t gate_batch_stride, int rows_per_batch,
                           void* dm16, float* dgate, int64_t dgate_batch_stride, float* dbias, int rows, int dim, int dtype,
                           void* stream);
/* out[dim] (fp32) += column sums of a [rows, dim]; a_dtype: 0 fp32, 1 fp16, 2 bf16.                                       */
B200_API int b200_colsum(const void* a, int a_dtype, float* out, int rows, int dim, void* stream);
/* backward of h = LayerNorm(x)(1 + scale[b]) + shift[b] (latte.py:28-29, eps 1e-6): dx (fp32, in place) += dL/dx;
 * dshift[b], dscale[b] (row stride dmod_batch_stride) += per-sample sums of dh and dh * xhat.  rows_per_batch % 64 == 0. */
B200_API int b200_ln_modulate_bwd(const void* dh16, const float* x, const float* scale, int64_t mod_batch_stride, int rows_per_batch,
                                  float* dx, float* dshift, float* dscale, int64_t dmod_batch_stride, int rows, int dim, int dtype,
                                  void* stream);
/* backward of b200_attention: dqkv16 [T, 3*heads*head_dim] from qkv16, o16 (its output) and do16.  Scores are recomputed on
 * mma.sync tensor cores; head_dim 64 or 72 at every frame count, other head dims return B200_ERR_UNSUPPORTED.
 * Spatial: tokens % 64 == 0.  Temporal: 1..128 frames.  stats = 2 * batch*frames*heads*tokens floats of scratch (unused by
 * temporal sequences of 16 frames or fewer).                                                                                */
B200_API int b200_attention_bwd(const void* qkv16, const void* o16, const void* do16, void* dqkv16, float* stats, int batch,
                                int frames, int tokens, int heads, int head_dim, int dtype, int temporal, void* stream);
/* backward of b200_cross_attention (default scale, no key/value padding rows): dq16 [batch*q_rows_per_batch, heads*head_dim]
 * and dK / dV written into dkv16 [batch*kv_len, dkv_row_stride] at columns [dkv_col0, dkv_col0 + 2*heads*head_dim) in the kv
 * operand's own order [k heads | v heads]; the other columns are not touched.  q, kv, key_bias as in b200_cross_attention; o16
 * its output, do16 the output's gradient.  head_dim 64 or 72 (others return B200_ERR_UNSUPPORTED), kv_len 1..128,
 * q_rows_per_batch % 128 == 0.  dK / dV sum a fixed number of per-chunk fp32 partials in a fixed order: bit-reproducible.
 * workspace: >= b200_cross_attention_bwd_workspace_bytes(...) bytes, 16-byte aligned (0 = unsupported shape).             */
B200_API size_t b200_cross_attention_bwd_workspace_bytes(int batch, int q_rows_per_batch, int kv_len, int heads, int head_dim);
B200_API int b200_cross_attention_bwd(const void* q, const void* kv, const float* key_bias, const void* o16, const void* do16, void* dq16,
                                      void* dkv16, int dkv_row_stride, int dkv_col0, int batch, int q_rows_per_batch, int kv_len,
                                      int q_row_stride, int kv_row_stride, int heads, int head_dim, int dtype, void* workspace,
                                      size_t workspace_bytes, void* stream);
/* adaLN_modulation Linear on `batch` <= 8 conditioning rows (all blocks stacked, NA = depth*6*dim + 2*dim output features):
 * dW[NA, dim] (fp32, overwritten) = dmod^T . sc16;  dsc[batch, dim] (fp32, overwritten) = dmod . W16.                     */
B200_API int b200_ada_outer(const float* dmod, int64_t dmod_batch_stride, const void* sc16, float* dW, int batch, int NA, int dim,
                            int dtype, void* stream);
B200_API int b200_ada_dsc(const float* dmod, int64_t dmod_batch_stride, const void* w16, float* dsc, int batch, int NA, int dim,
                          int dtype, void* stream);

/* ---- sampler step (SURVEY.md 8f rank 1): the fp32 arithmetic the reference's GaussianDiffusion does around every model
 * call, as ONE kernel with device-resident schedule tables.  Replaces p_mean_variance (diffusion/gaussian_diffusion.py:
 * 254-336, EPSILON mean + LEARNED_RANGE variance), p_sample (:380-419), ddim_sample (:517-564) and the per-call
 * _extract_into_tensor H2D copies (:869-881).                                                                            */
enum { B200_SAMPLER_DDPM = 0, B200_SAMPLER_DDIM = 1 };
typedef struct {
  int num_timesteps;                             /* length of every table (the respaced chain)                           */
  const float* sqrt_recip_alphas_cumprod;        /* device, fp32 = the reference's float64 table cast with .float()      */
  const float* sqrt_recipm1_alphas_cumprod;
  const float* posterior_mean_coef1;
  const float* posterior_mean_coef2;
  const float* posterior_log_variance_clipped;
  const float* log_betas;                        /* np.log(betas)                                                        */
  /* DDIM only (may be NULL for DDPM): the per-timestep scalars of ddim_sample (:544-556) evaluated ONCE by the caller in
   * fp32 with the reference's expressions on the fp32 alphas_cumprod / alphas_cumprod_prev values:
   *   ddim_sqrt_alpha_prev = sqrt(abar_prev);  ddim_sigma = eta * sqrt((1-abar_prev)/(1-abar)) * sqrt(1 - abar/abar_prev);
   *   ddim_dir = sqrt(1 - abar_prev - ddim_sigma^2)                                                                     */
  const float* ddim_sqrt_alpha_prev;
  const float* ddim_sigma;
  const float* ddim_dir;
} B200SamplerTables;

/* x_t (B,F,C,H,W) fp32, t (B,) int64 chain indices (device), model_out (B,F,2C,H,W) in model_out_dtype (0 fp32, 1 fp16,
 * 2 bf16), noise (B,F,C,H,W) fp32 or NULL (= zeros; DDIM with sigma == 0 only).  Outputs, each fp32 (B,F,C,H,W) or NULL:
 * x_prev ('sample'), pred_xstart, mean, log_variance (p_mean_variance's dict).  hw = H*W must be a multiple of 4.       */
B200_API int b200_sampler_step(const B200SamplerTables* tables, int method, int clip_denoised, const int64_t* t,
                               const float* x, const void* model_out, int model_out_dtype, const float* noise, int batch,
                               int frames, int channels, int hw, float* x_prev, float* pred_xstart, float* mean,
                               float* log_variance, void* stream);

/* GaussianDiffusion.training_losses (gaussian_diffusion.py:719-795; LossType.MSE + LEARNED_RANGE, the objective train.py:221
 * uses) in one pass: sums[0][b] = sum over the sample of (noise - eps)^2, sums[1][b] = sum of the variational-bound term in
 * NATS (KL to the true posterior, decoder NLL where t[b] == 0; the mean is frozen: it gets no gradient from this term), and, if
 * dmo != NULL, the gradient of [mean_flat(mse) | mean_flat(vb) / ln 2] with respect to model_out: channels [0, C) of every frame
 * hold d mse / d eps, channels [C, 2C) hold d vb / d var_values.  x0, xt, noise (B,F,C,H,W) fp32; model_out, dmo (B,F,2C,H,W) fp32;
 * t (B,) int64 chain indices; sums 2*B floats (overwritten).                                                                  */
B200_API int b200_training_loss(const B200SamplerTables* tables, const int64_t* t, const float* x0, const float* xt, const float* noise,
                                const float* model_out, int batch, int frames, int channels, int hw, float* sums, float* dmo, void* stream);

/* Host-only introspection (no GPU touched): the work schedule b200_linear would use on a device with `num_sms` SMs --
 * chosen tile width, number of CTA pairs, whether the last waves are split along K (stream-K, residual epilogue), and
 * the (pair, tile, kb0, kb1) segments in each pair's execution order (up to max_segments quadruples; the return value
 * is the total count, negative on error).  The CPU tests check coverage and the ordering invariant on it.            */
B200_API int b200_gemm_schedule(int M, int N, int K, int epilogue, int block_n, int num_sms, int* block_n_out, int* pairs_out,
                                int* streamk_out, int32_t* segments, int max_segments);
/* The same for b200_wgrad(rows, n_out, n_in): a [n_out, n_in] output under a contraction over `rows`.  Outputs with fewer tiles
 * than CTA pairs are cut into several K-segments per tile, executed by consecutive pairs and added in k order.               */
B200_API int b200_wgrad_schedule(int rows, int n_out, int n_in, int num_sms, int* block_n_out, int* pairs_out, int* streamk_out,
                                 int32_t* segments, int max_segments);

/* Measurement hook (bench.py roofline): while enabled, b200_latte_forward brackets every kernel launch with
 * CUDA events on the launching stream.  b200_profile_collect waits for them and returns, per class
 * {0 tensor-core GEMM, 1 attention, 2 LN+modulate, 3 other}, the summed device time in ms and the launch count,
 * then clears the records.  Disabled (default) the forward records nothing.                        */
B200_API void b200_profile_enable(int on);
B200_API int b200_profile_collect(double* ms_per_class, int* launches_per_class, int n_classes);

#ifdef __cplusplus
}
#endif
#endif /* LATTE_B200_H */
