// CUDA-core kernels around the tensor-core GEMMs: everything here is HBM- or latency-bound, so the rules are
// coalesced 16-byte accesses, one pass over the data, fp32 math.
//   ln_modulate   LayerNorm(no affine, eps 1e-6) + adaLN modulate -> 16-bit GEMM operand   (latte.py:28-29,166-168,179-180)
//   patch_embed   Conv2d(k=s=p) as a K=C*p*p dot per token + bias + pos_embed -> fp32 residual stream (latte.py:330-331)
//   timestep_freq sinusoidal features                                                       (latte.py:98-116)
//   gemv          warp-per-output-row mat-vec for the per-SAMPLE conditioning path: t-MLP (latte.py:118-123),
//                 label lookup (:148-153) and ONE batched adaLN for all blocks on B rows instead of B*F / B*N
//                 repeated rows (latte.py:172-178, SURVEY.md F7)
//   final_layer   LN + modulate + Linear(D, p*p*Cout) + unpatchify scatter                   (latte.py:197-201,297-310,374-376)
//   cfg_combine   classifier-free guidance on eps channels                                   (latte.py:394-398)
#include <cstdlib>
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

// ---------------------------------------------------------------------------------- ln_modulate
constexpr int LN_MAXV = 12;  // float4 per lane: dim <= 12*128 = 1536

// One warp per row, the whole row in registers (NV float4 per lane, compile-time so nothing spills), two-pass
// mean/variance in fp32, one read and one write of the data.  (Round 2 tried one 16-byte store per lane per chunk of 8:
// 80 registers instead of 64 cost a quarter of the resident warps and the kernel got SLOWER in the step, 0.91 -> 1.07 ms;
// the 8-byte stores of a warp still fill whole 128-byte lines, so this form stays.)  Work is split so that EVERY warp owns the same number of
// consecutive rows and all warps are resident at once (register-limited to 32 warps/SM): a grid-stride loop left a
// half-empty second wave.  The block's shift/scale vectors are staged in shared memory once, so the only global latency
// on a row's critical path is the row itself.
//
// E4M3: the FP8 sampling path's instance.  The modulated fp32 row is quantized with one scale per row (token),
// s = amax(|y|) / 448 (1 for an all-zero row), q = e4m3_rn_satfinite(y / s) with a correctly rounded division -- the
// formula of quantize_rows_e4m3 -- and `out` receives dim bytes per row, row_scale[row] = s.  The amax is one more warp
// reduction over the registers that already hold the row.
template <bool BF16, int NV, bool E4M3 = false>
__global__ void __launch_bounds__(128) ln_modulate_kernel(const float* __restrict__ x, const float* __restrict__ shift,
                                                          const float* __restrict__ scale, long long mod_bs,
                                                          int rows_per_batch, uint16_t* __restrict__ out, int rows,
                                                          int dim, int rows_per_warp, float* __restrict__ row_scale) {
  extern __shared__ float4 s_mod[];  // [2][dim/4]: shift, scale of the batch row this block starts in
  const int lane = threadIdx.x & 31;
  const int nv = dim >> 2;
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int block_row0 = blockIdx.x * (blockDim.x >> 5) * rows_per_warp;
  pdl_launch_dependents();
  const long long b0 = (block_row0 < rows ? block_row0 : rows - 1) / rows_per_batch;
  // shift / scale come from the conditioning path at the start of the step (a plainly launched kernel that completed
  // before any programmatically-launched one began), not from the kernel just before this one: stage them while that
  // kernel is still draining.  x (the residual stream it updates) is only touched after pdl_wait().
  for (int i = threadIdx.x; i < 2 * nv; i += blockDim.x) {
    const float* src = (i < nv ? shift : scale) + b0 * mod_bs;
    s_mod[i] = __ldg(reinterpret_cast<const float4*>(src) + (i < nv ? i : i - nv));
  }
  __syncthreads();
  pdl_wait();
  const int row0 = warp_global * rows_per_warp;
  float4 v[NV];
  if (row0 < rows) {
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row0) * dim);
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nv) v[i] = xr[lane + i * 32];
  }
  for (int rr = 0; rr < rows_per_warp; ++rr) {
    const int row = row0 + rr;
    if (row >= rows) break;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nv) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) / static_cast<float>(dim);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (lane + i * 32 < nv) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(dim) + 1e-6f);
    const long long b = row / rows_per_batch;
    const bool staged = b == b0;
    const float4* sh = reinterpret_cast<const float4*>(shift + b * mod_bs);
    const float4* sc = reinterpret_cast<const float4*>(scale + b * mod_bs);
    if constexpr (E4M3) {
      // the modulated row replaces x in the registers (the next row is loaded after the stores)
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nv) {
          const float4 h = staged ? s_mod[idx] : __ldg(sh + idx);
          const float4 c = staged ? s_mod[nv + idx] : __ldg(sc + idx);
          v[i].x = fmaf((v[i].x - mean) * rstd, 1.0f + c.x, h.x);
          v[i].y = fmaf((v[i].y - mean) * rstd, 1.0f + c.y, h.y);
          v[i].z = fmaf((v[i].z - mean) * rstd, 1.0f + c.z, h.z);
          v[i].w = fmaf((v[i].w - mean) * rstd, 1.0f + c.w, h.w);
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      const float s = e4m3_scale(amax);
      uint32_t* orow = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(out) + static_cast<size_t>(row) * dim);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nv)
          orow[idx] = pack_e4m3x4(__fdiv_rn(v[i].x, s), __fdiv_rn(v[i].y, s), __fdiv_rn(v[i].z, s), __fdiv_rn(v[i].w, s));
      }
      if (lane == 0) row_scale[row] = s;
    } else {
      uint2* orow = reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * dim);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nv) {
          const float4 h = staged ? s_mod[idx] : __ldg(sh + idx);
          const float4 c = staged ? s_mod[nv + idx] : __ldg(sc + idx);
          const float y0 = fmaf((v[i].x - mean) * rstd, 1.0f + c.x, h.x);
          const float y1 = fmaf((v[i].y - mean) * rstd, 1.0f + c.y, h.y);
          const float y2 = fmaf((v[i].z - mean) * rstd, 1.0f + c.z, h.z);
          const float y3 = fmaf((v[i].w - mean) * rstd, 1.0f + c.w, h.w);
          orow[idx] = make_uint2(pack2<BF16>(y0, y1), pack2<BF16>(y2, y3));
        }
      }
    }
    if (rr + 1 < rows_per_warp && row + 1 < rows) {
      const float4* xn = reinterpret_cast<const float4*>(x + static_cast<size_t>(row + 1) * dim);
#pragma unroll
      for (int i = 0; i < NV; ++i)
        if (lane + i * 32 < nv) v[i] = xn[lane + i * 32];
    }
  }
}

template <bool BF16, int NV, bool E4M3 = false>
int ln_launch(cudaStream_t stream, const float* x, const float* shift, const float* scale, long long mod_bs, int rpb,
              uint16_t* out, int rows, int dim, int sms, float* row_scale = nullptr) {
  auto kern = ln_modulate_kernel<BF16, NV, E4M3>;
  const size_t smem = static_cast<size_t>(dim) * 2 * sizeof(float);
  static int blocks_per_sm_dev[64] = {};   // per instantiation and device: what the register/smem footprint really allows
  int dev = 0;
  B200_TRY(current_device(&dev));
  if (blocks_per_sm_dev[dev] == 0) {
    int n = 0;
    B200_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 128, smem));
    blocks_per_sm_dev[dev] = n > 0 ? n : 1;
  }
  const int blocks_per_sm = blocks_per_sm_dev[dev];
  // every warp gets the same number of consecutive rows and the whole grid is resident in one wave
  const int wpb = 4;
  const int resident_warps = sms * blocks_per_sm * wpb;
  const int rpw = (rows + resident_warps - 1) / resident_warps;
  const int blocks = (rows + wpb * rpw - 1) / (wpb * rpw);
  B200_CHECK_CUDA(launch_pdl(kern, dim3(blocks), dim3(128), smem, stream, x, shift, scale, mod_bs, rpb, out, rows, dim, rpw,
                                    row_scale));
  return B200_OK;
}

template <bool BF16>
int ln_dispatch(int nvmax, cudaStream_t stream, const float* x, const float* shift, const float* scale, long long mod_bs,
                int rpb, uint16_t* out, int rows, int dim, int sms) {
  if (nvmax <= 3) return ln_launch<BF16, 3>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms);
  if (nvmax <= 6) return ln_launch<BF16, 6>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms);
  if (nvmax <= 9) return ln_launch<BF16, 9>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms);
  return ln_launch<BF16, LN_MAXV>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms);
}

// the e4m3 instances (the operand type of the 16-bit template argument does not matter: one instance per width)
int ln_dispatch_e4m3(int nvmax, cudaStream_t stream, const float* x, const float* shift, const float* scale, long long mod_bs,
                     int rpb, uint8_t* out8, float* row_scale, int rows, int dim, int sms) {
  uint16_t* out = reinterpret_cast<uint16_t*>(out8);
  if (nvmax <= 3) return ln_launch<false, 3, true>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms, row_scale);
  if (nvmax <= 6) return ln_launch<false, 6, true>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms, row_scale);
  if (nvmax <= 9) return ln_launch<false, 9, true>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms, row_scale);
  return ln_launch<false, LN_MAXV, true>(stream, x, shift, scale, mod_bs, rpb, out, rows, dim, sms, row_scale);
}

// ---------------------------------------------------------------------------------- quantize_rows_e4m3
// One warp per row of an fp32 matrix [rows, cols] (a weight W[N, K]: one scale per output channel): s = amax(|row|) / 448
// (1 for an all-zero row), q = e4m3_rn_satfinite(w / s), the division correctly rounded.  Two passes over the row in
// global memory: this runs once per weight packing, not per step.
__global__ void __launch_bounds__(256) quantize_rows_e4m3_kernel(const float* __restrict__ w, int rows, int cols,
                                                                 uint32_t* __restrict__ q, float* __restrict__ scales) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* wr = reinterpret_cast<const float4*>(w + static_cast<size_t>(row) * cols);
  const int n4 = cols >> 2;
  float amax = 0.f;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = __ldg(wr + i);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = e4m3_scale(amax);
  uint32_t* qr = q + static_cast<size_t>(row) * n4;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = __ldg(wr + i);
    qr[i] = pack_e4m3x4(__fdiv_rn(v.x, s), __fdiv_rn(v.y, s), __fdiv_rn(v.z, s), __fdiv_rn(v.w, s));
  }
  if (lane == 0) scales[row] = s;
}

// ---------------------------------------------------------------------------------- patch_embed
constexpr int PE_TOK = 16;

// K = C*p*p is a template parameter, 4 to 32 (16 for the 4-channel, patch-2 latents; wider K: patch_embed_wide_kernel).  A thread owns FOUR
// consecutive output channels: their 4 x K weights live in registers, and for each of the block's PE_TOK tokens it does
// 4 x K FMAs, one 16-byte read of pos_embed and ONE 16-byte store of the fp32 residual stream (the only real traffic:
// T*D*4 bytes).  Round 1 stored 4 bytes per thread per token: 42 us for 37.7 MB; this form issues a quarter of the
// load/store instructions.
template <int K>
__global__ void __launch_bounds__(320) patch_embed_kernel(const float* __restrict__ x, int x_batch_mod,
                                                          const float* __restrict__ w, const float* __restrict__ bias,
                                                          const float* __restrict__ pos, float* __restrict__ out,
                                                          int total_tokens, int frames, int chans, int size, int patch,
                                                          int dim, long long sb, long long sf, long long sc) {
  __shared__ float in[PE_TOK][K];
  const int grid = size / patch;
  const int N = grid * grid;
  const int tok0 = blockIdx.x * PE_TOK;
  for (int i = threadIdx.x; i < PE_TOK * K; i += blockDim.x) {
    const int tl = i / K, k = i % K;
    const int tok = tok0 + tl;
    float val = 0.f;
    if (tok < total_tokens) {
      const int n = tok % N, bf = tok / N;
      const int b = bf / frames, f = bf % frames;
      const int bsrc = b % x_batch_mod;
      const int gh = n / grid, gw = n % grid;
      const int c = k / (patch * patch), ij = k % (patch * patch);
      const int ii = ij / patch, jj = ij % patch;
      val = x[bsrc * sb + f * sf + c * sc + static_cast<long long>(gh * patch + ii) * size + gw * patch + jj];
    }
    in[tl][k] = val;
  }
  __syncthreads();
  const int nv = dim >> 2;
  for (int d4 = threadIdx.x; d4 < nv; d4 += blockDim.x) {
    float wk[4][K];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int k = 0; k < K; k += 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(w + static_cast<size_t>(d4 * 4 + r) * K + k));
        wk[r][k] = t.x; wk[r][k + 1] = t.y; wk[r][k + 2] = t.z; wk[r][k + 3] = t.w;
      }
    const float4 bd = __ldg(reinterpret_cast<const float4*>(bias) + d4);
#pragma unroll 2
    for (int tl = 0; tl < PE_TOK; ++tl) {
      const int tok = tok0 + tl;
      if (tok >= total_tokens) break;
      const float4 pe = __ldg(reinterpret_cast<const float4*>(pos + static_cast<size_t>(tok % N) * dim) + d4);
      float a0 = bd.x, a1 = bd.y, a2 = bd.z, a3 = bd.w;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float v = in[tl][k];
        a0 = fmaf(v, wk[0][k], a0); a1 = fmaf(v, wk[1][k], a1); a2 = fmaf(v, wk[2][k], a2); a3 = fmaf(v, wk[3][k], a3);
      }
      reinterpret_cast<float4*>(out + static_cast<size_t>(tok) * dim)[d4] = make_float4(a0 + pe.x, a1 + pe.y, a2 + pe.z, a3 + pe.w);
    }
  }
}

// K = 64 and 256 (patch 4 and 8 of 4-channel latents): 4 x K weights no longer fit in registers (1,024 floats at K = 256), so
// the thread keeps the 4 x PE_TOK accumulators instead and streams K through them PE_KC columns at a time: a chunk's 4 x PE_KC
// weights are loaded once and applied to all PE_TOK tokens of the shared `in` tile.  Each accumulator starts at the bias and
// takes its K products in k order, as in patch_embed_kernel, all in fp32.
constexpr int PE_KC = 16;

template <int K>
__global__ void __launch_bounds__(320) patch_embed_wide_kernel(const float* __restrict__ x, int x_batch_mod,
                                                               const float* __restrict__ w, const float* __restrict__ bias,
                                                               const float* __restrict__ pos, float* __restrict__ out,
                                                               int total_tokens, int frames, int chans, int size, int patch,
                                                               int dim, long long sb, long long sf, long long sc) {
  static_assert(K % PE_KC == 0, "K must be a multiple of the chunk");
  __shared__ float in[PE_TOK][K];
  const int grid = size / patch;
  const int N = grid * grid;
  const int tok0 = blockIdx.x * PE_TOK;
  for (int i = threadIdx.x; i < PE_TOK * K; i += blockDim.x) {
    const int tl = i / K, k = i % K;
    const int tok = tok0 + tl;
    float val = 0.f;
    if (tok < total_tokens) {
      const int n = tok % N, bf = tok / N;
      const int b = bf / frames, f = bf % frames;
      const int bsrc = b % x_batch_mod;
      const int gh = n / grid, gw = n % grid;
      const int c = k / (patch * patch), ij = k % (patch * patch);
      const int ii = ij / patch, jj = ij % patch;
      val = x[bsrc * sb + f * sf + c * sc + static_cast<long long>(gh * patch + ii) * size + gw * patch + jj];
    }
    in[tl][k] = val;
  }
  __syncthreads();
  const int nv = dim >> 2;
  for (int d4 = threadIdx.x; d4 < nv; d4 += blockDim.x) {
    const float4 bd = __ldg(reinterpret_cast<const float4*>(bias) + d4);
    float acc[PE_TOK][4];
#pragma unroll
    for (int tl = 0; tl < PE_TOK; ++tl) { acc[tl][0] = bd.x; acc[tl][1] = bd.y; acc[tl][2] = bd.z; acc[tl][3] = bd.w; }
#pragma unroll 1
    for (int k0 = 0; k0 < K; k0 += PE_KC) {
      float wk[4][PE_KC];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int k = 0; k < PE_KC; k += 4) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(w + static_cast<size_t>(d4 * 4 + r) * K + k0 + k));
          wk[r][k] = t.x; wk[r][k + 1] = t.y; wk[r][k + 2] = t.z; wk[r][k + 3] = t.w;
        }
#pragma unroll
      for (int tl = 0; tl < PE_TOK; ++tl)
#pragma unroll
        for (int k = 0; k < PE_KC; ++k) {
          const float v = in[tl][k0 + k];
#pragma unroll
          for (int r = 0; r < 4; ++r) acc[tl][r] = fmaf(v, wk[r][k], acc[tl][r]);
        }
    }
#pragma unroll
    for (int tl = 0; tl < PE_TOK; ++tl) {
      const int tok = tok0 + tl;
      if (tok < total_tokens) {
        const float4 pe = __ldg(reinterpret_cast<const float4*>(pos + static_cast<size_t>(tok % N) * dim) + d4);
        reinterpret_cast<float4*>(out + static_cast<size_t>(tok) * dim)[d4] =
            make_float4(acc[tl][0] + pe.x, acc[tl][1] + pe.y, acc[tl][2] + pe.z, acc[tl][3] + pe.w);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- timestep features
__global__ void timestep_freq_kernel(const long long* __restrict__ t, float* __restrict__ out, int batch) {
  const int b = blockIdx.x;
  const int k = threadIdx.x;  // 0..255
  if (b >= batch) return;
  const int half = 128;
  const int kk = k % half;
  const float freq = expf(-9.210340371976184f * static_cast<float>(kk) / static_cast<float>(half));  // ln(1e4)
  const float arg = static_cast<float>(t[b]) * freq;
  out[b * 256 + k] = (k < half) ? cosf(arg) : sinf(arg);
}

// ---------------------------------------------------------------------------------- gemv (a warp owns GV_ROWS output rows)
constexpr int GV_MAXB = 8;
constexpr int GV_ROWS = 4;

// HBM-bound on the weight matrix (adaLN: 446 MB per step for XL/2): every lane issues GV_ROWS independent 16-byte
// loads per trip so ~4.6 KB per warp are in flight; the B input vectors live in smem (read as broadcast float4).
template <int WBITS, bool BF16>
__global__ void __launch_bounds__(256) gemv_kernel(const void* __restrict__ W, const float* __restrict__ bias,
                                                   const float* __restrict__ in, float* __restrict__ out, int batch,
                                                   int J, int K, int silu_in, int silu_out,
                                                   const float* __restrict__ add_table,
                                                   const long long* __restrict__ add_idx, int add_rows) {
  extern __shared__ float sin_[];  // [batch][K]
  if (add_table && threadIdx.x < batch) {   // nn.Embedding asserts on an out-of-range index; so does this lookup
    const long long idx = add_idx[threadIdx.x];
    if (idx < 0 || idx >= add_rows) {
      if (blockIdx.x == 0) printf("latte_b200: label %lld out of range [0, %d)\n", idx, add_rows);
      __trap();
    }
  }
  for (int i = threadIdx.x; i < batch * K; i += blockDim.x) {
    const float v = in[i];
    sin_[i] = silu_in ? silu(v) : v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  constexpr int EPC = WBITS == 32 ? 4 : 8;  // elements per 16-byte chunk
  const int nchunk = K / EPC;
  for (int j0 = (blockIdx.x * warps + (threadIdx.x >> 5)) * GV_ROWS; j0 < J; j0 += gridDim.x * warps * GV_ROWS) {
    float acc[GV_ROWS][GV_MAXB];
#pragma unroll
    for (int r = 0; r < GV_ROWS; ++r)
#pragma unroll
      for (int b = 0; b < GV_MAXB; ++b) acc[r][b] = 0.f;
    for (int c = lane; c < nchunk; c += 32) {
      uint4 wv[GV_ROWS];
#pragma unroll
      for (int r = 0; r < GV_ROWS; ++r) {
        const int j = j0 + r < J ? j0 + r : J - 1;
        wv[r] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(W) + (static_cast<size_t>(j) * K + static_cast<size_t>(c) * EPC) * (WBITS / 8)));
      }
#pragma unroll
      for (int b = 0; b < GV_MAXB; ++b) {
        if (b < batch) {
          const float4 x0 = *reinterpret_cast<const float4*>(sin_ + b * K + c * EPC);
          float4 x1 = make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (WBITS == 16) x1 = *reinterpret_cast<const float4*>(sin_ + b * K + c * EPC + 4);
#pragma unroll
          for (int r = 0; r < GV_ROWS; ++r) {
            if constexpr (WBITS == 32) {
              acc[r][b] = fmaf(__uint_as_float(wv[r].x), x0.x, fmaf(__uint_as_float(wv[r].y), x0.y,
                          fmaf(__uint_as_float(wv[r].z), x0.z, fmaf(__uint_as_float(wv[r].w), x0.w, acc[r][b]))));
            } else {
              const float2 w0 = unpack2<BF16>(wv[r].x), w1 = unpack2<BF16>(wv[r].y), w2 = unpack2<BF16>(wv[r].z), w3 = unpack2<BF16>(wv[r].w);
              float a = acc[r][b];
              a = fmaf(w0.x, x0.x, a); a = fmaf(w0.y, x0.y, a); a = fmaf(w1.x, x0.z, a); a = fmaf(w1.y, x0.w, a);
              a = fmaf(w2.x, x1.x, a); a = fmaf(w2.y, x1.y, a); a = fmaf(w3.x, x1.z, a); a = fmaf(w3.y, x1.w, a);
              acc[r][b] = a;
            }
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < GV_ROWS; ++r) {
#pragma unroll
      for (int b = 0; b < GV_MAXB; ++b) {
        if (b < batch) {
          float v = warp_sum(acc[r][b]);
          const int j = j0 + r;
          if (lane == 0 && j < J) {
            if (bias) v += __ldg(bias + j);
            if (add_table) v += __ldg(add_table + static_cast<size_t>(add_idx[b]) * J + j);
            out[static_cast<size_t>(b) * J + j] = silu_out ? silu(v) : v;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------- final layer
constexpr int FL_MAXV = 12;
constexpr int FL_MAXO = 32;

__global__ void __launch_bounds__(512) final_layer_kernel(const float* __restrict__ x, const float* __restrict__ shift,
                                                          const float* __restrict__ scale, long long mod_bs,
                                                          const float* __restrict__ w, const float* __restrict__ bias,
                                                          float* __restrict__ out, int total_tokens, int frames,
                                                          int grid, int patch, int out_ch, int dim, long long osb,
                                                          long long osf, long long osc) {
  extern __shared__ float sw[];  // [n_out][dim]
  const int n_out = patch * patch * out_ch;
  for (int i = threadIdx.x; i < n_out * dim / 4; i += blockDim.x)
    reinterpret_cast<float4*>(sw)[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  const int nv = dim >> 2;
  const int N = grid * grid;
  const int size = grid * patch;
  for (int tok = blockIdx.x * warps + (threadIdx.x >> 5); tok < total_tokens; tok += gridDim.x * warps) {
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(tok) * dim);
    float4 v[FL_MAXV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < FL_MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) {
        v[i] = xr[idx];
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
      }
    }
    const float mean = warp_sum(s) / static_cast<float>(dim);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < FL_MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(dim) + 1e-6f);
    const int n = tok % N, bf = tok / N;
    const long long b = bf / frames;
    const float4* sh = reinterpret_cast<const float4*>(shift + b * mod_bs);
    const float4* sc = reinterpret_cast<const float4*>(scale + b * mod_bs);
#pragma unroll
    for (int i = 0; i < FL_MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) {
        const float4 h = __ldg(sh + idx), c = __ldg(sc + idx);
        v[i].x = fmaf((v[i].x - mean) * rstd, 1.0f + c.x, h.x);
        v[i].y = fmaf((v[i].y - mean) * rstd, 1.0f + c.y, h.y);
        v[i].z = fmaf((v[i].z - mean) * rstd, 1.0f + c.z, h.z);
        v[i].w = fmaf((v[i].w - mean) * rstd, 1.0f + c.w, h.w);
      }
    }
    float mine = 0.f;  // lane o keeps output o
    for (int o = 0; o < n_out; ++o) {
      const float4* wr = reinterpret_cast<const float4*>(sw + static_cast<size_t>(o) * dim);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < FL_MAXV; ++i) {
        const int idx = lane + i * 32;
        if (idx < nv) {
          const float4 wv = wr[idx];
          acc = fmaf(v[i].x, wv.x, fmaf(v[i].y, wv.y, fmaf(v[i].z, wv.z, fmaf(v[i].w, wv.w, acc))));
        }
      }
      acc = warp_sum(acc);
      if (lane == o) mine = acc;
    }
    if (lane < n_out) {
      // unpatchify (latte.py:307-309): o = (pi*patch + qi)*out_ch + c  ->  out[bf][c][gh*patch+pi][gw*patch+qi]
      const int c = lane % out_ch, pq = lane / out_ch;
      const int pi = pq / patch, qi = pq % patch;
      const int gh = n / grid, gw = n % grid;
      out[(bf / frames) * osb + (bf % frames) * osf + c * osc + static_cast<long long>(gh * patch + pi) * size + gw * patch + qi] = mine + __ldg(bias + lane);
    }
  }
}

// ---------------------------------------------------------------------------------- T5 encoder pieces (SURVEY.md 8f rank 3)
// T5LayerNorm (transformers modeling_t5.py): y = x * rsqrt(mean(x^2) + eps) * weight -- no mean subtraction, no bias;
// the variance is taken in fp32.  One warp per row; out16 (GEMM operand) or out32 (the encoder's final_layer_norm).
template <bool BF16>
__global__ void __launch_bounds__(256) rms_norm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                       uint16_t* __restrict__ out16, float* __restrict__ out32, int rows,
                                                       int dim, float eps) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * dim);
  const int nv = dim >> 2;
  float q = 0.f;
  for (int i = lane; i < nv; i += 32) {
    const float4 v = xr[i];
    q += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  const float r = rsqrtf(warp_sum(q) / static_cast<float>(dim) + eps);
  for (int i = lane; i < nv; i += 32) {
    const float4 v = xr[i];
    const float4 g = __ldg(reinterpret_cast<const float4*>(w) + i);
    const float y0 = v.x * r * g.x, y1 = v.y * r * g.y, y2 = v.z * r * g.z, y3 = v.w * r * g.w;
    if (out32) reinterpret_cast<float4*>(out32 + static_cast<size_t>(row) * dim)[i] = make_float4(y0, y1, y2, y3);
    else reinterpret_cast<uint2*>(out16 + static_cast<size_t>(row) * dim)[i] = make_uint2(pack2<BF16>(y0, y1), pack2<BF16>(y2, y3));
  }
}

// x[r, :] = table[ids[r], :]  (nn.Embedding lookup of the token ids; 16-bit table -> fp32 residual stream)
template <bool BF16>
__global__ void __launch_bounds__(256) embed_kernel(const long long* __restrict__ ids, const uint16_t* __restrict__ table,
                                                    float* __restrict__ x, int rows, int dim, int vocab) {
  const int row = blockIdx.x;
  if (row >= rows) return;
  const long long id = ids[row];
  if (id < 0 || id >= vocab) {
    if (threadIdx.x == 0) printf("latte_b200: token id %lld out of range [0, %d)\n", id, vocab);
    __trap();
  }
  const uint2* src = reinterpret_cast<const uint2*>(table + static_cast<size_t>(id) * dim);
  float4* dst = reinterpret_cast<float4*>(x + static_cast<size_t>(row) * dim);
  for (int i = threadIdx.x; i < dim / 4; i += blockDim.x) {
    const uint2 v = __ldg(src + i);
    const float2 a = unpack2<BF16>(v.x), b = unpack2<BF16>(v.y);
    dst[i] = make_float4(a.x, a.y, b.x, b.y);
  }
}

// ---------------------------------------------------------------------------------- decoded frames -> uint8 (SURVEY.md 8f rank 3)
// The two post-processing expressions of the reference, each with ITS rounding, fused with the NCHW -> NHWC permute:
//   mode 0  pipeline_latte.py:775,796   ((v / 2.0 + 0.5).clamp(0, 1) * 255).to(uint8)           (truncation)
//   mode 1  sample.py:122, sample_ddp.py:172   ((v * 0.5 + 0.5) * 255).add_(0.5).clamp_(0, 255).to(uint8)
// torch evaluates every operator in the tensor's own dtype, so for 16-bit inputs each intermediate is rounded to that
// type (`rnd`) -- the result is bit-identical to the reference expression on the same tensor.
template <int DT>   // 0 fp32, 1 fp16, 2 bf16
__device__ __forceinline__ float rnd(float v) {
  if constexpr (DT == 1) return __half2float(__float2half_rn(v));
  if constexpr (DT == 2) return __bfloat162float(__float2bfloat16_rn(v));
  return v;
}
template <int DT>
__global__ void __launch_bounds__(256) frames_to_uint8_kernel(const void* __restrict__ in, uint8_t* __restrict__ out, long long total,
                                                              int c, int hw, int mode) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // i enumerates the OUTPUT [n][h*w][c]; the input is [n][c][h*w]
    const int ch = static_cast<int>(i % c);
    const long long pix = (i / c) % hw;
    const long long img = i / (static_cast<long long>(c) * hw);
    const long long src = (img * c + ch) * hw + pix;
    float v;
    if constexpr (DT == 0) v = static_cast<const float*>(in)[src];
    else if constexpr (DT == 1) v = __half2float(static_cast<const __half*>(in)[src]);
    else v = __bfloat162float(static_cast<const __nv_bfloat16*>(in)[src]);
    float r;
    if (mode == 0) {
      r = rnd<DT>(rnd<DT>(v / 2.0f) + 0.5f);
      r = fminf(fmaxf(r, 0.f), 1.f);
      r = rnd<DT>(r * 255.f);
    } else {
      r = rnd<DT>(rnd<DT>(rnd<DT>(v * 0.5f) + 0.5f) * 255.f);
      r = rnd<DT>(r + 0.5f);
      r = fminf(fmaxf(r, 0.f), 255.f);
    }
    out[i] = static_cast<uint8_t>(static_cast<int>(r));     // float -> uint8 conversion truncates toward zero, like torch
  }
}

// ---------------------------------------------------------------------------------- unpatchify
// y [T, n_out] fp32 (token-major output of the head GEMM, n_out = p*p*out_ch ordered (pi, qi, c)) -> the reference's
// layout out[b][f][c][gh*p + pi][gw*p + qi] (latte.py:297-310) or [b][c][f][..] (LatteT2V).  One thread per output
// element, indexed in OUTPUT order so the 4-byte stores coalesce; the gathers hit 128-byte rows of y that are L2-resident.
__global__ void unpatchify_kernel(const float* __restrict__ y, float* __restrict__ out, long long total, int frames, int grid,
                                  int patch, int out_ch, int n_out, long long osb, long long osf, long long osc) {
  const int size = grid * patch;
  const long long plane = static_cast<long long>(size) * size;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // i enumerates (bf, c, row, col) in the order of an [bf][c][H][W] tensor; osb/osf/osc place it in the real layout
    const long long pix = i % plane;
    const long long t1 = i / plane;
    const int c = static_cast<int>(t1 % out_ch);
    const long long bf = t1 / out_ch;
    const int row = static_cast<int>(pix / size), col = static_cast<int>(pix % size);
    const int gh = row / patch, pi = row % patch, gw = col / patch, qi = col % patch;
    const long long tok = bf * grid * grid + static_cast<long long>(gh) * grid + gw;
    const float v = y[tok * n_out + (pi * patch + qi) * out_ch + c];
    out[(bf / frames) * osb + (bf % frames) * osf + c * osc + pix] = v;
  }
}

// ---------------------------------------------------------------------------------- cfg combine
__global__ void cfg_combine_kernel(float* __restrict__ out, int half_batch, long long per_sample, int out_ch,
                                   int guided_ch, int hw, float scale) {
  // element (b < half, frame/channel/pixel) with channel < guided_ch:
  //   e = uncond + scale * (cond - uncond), written to both halves (latte.py:394-398)
  const long long total = static_cast<long long>(half_batch) * per_sample;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long within = i % per_sample;
    const int c = static_cast<int>((within / hw) % out_ch);
    if (c < guided_ch) {
      const float cond = out[i];
      const float uncond = out[i + total];
      // the product is rounded before the add, as the reference's fp32 tensor expression rounds it (no fma contraction)
      const float e = __fadd_rn(uncond, __fmul_rn(scale, __fsub_rn(cond, uncond)));
      out[i] = e;
      out[i + total] = e;
    }
  }
}

// ---------------------------------------------------------------------------------- LatteT2V helpers
// mod[b][blk][j][:] = table[blk][j][:] + ts[b][j][:]  (scale_shift_table + adaln_single(t), latte_t2v.py:296-298), and
// the output head's table[2][D] + embedded_timestep (latte_t2v.py:919-921) in the last slot.
__global__ void t2v_mod_kernel(const float* __restrict__ tables, const float* __restrict__ ts, const float* __restrict__ final_table,
                               const float* __restrict__ emb, float* __restrict__ mod, int batch, int nblocks, int dim) {
  const long long per_b = static_cast<long long>(nblocks) * 6 * dim + 2 * dim;
  const long long total = per_b * batch;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / per_b);
    const long long w = i % per_b;
    float v;
    if (w < static_cast<long long>(nblocks) * 6 * dim) {
      v = tables[w] + ts[static_cast<long long>(b) * 6 * dim + (w % (6 * dim))];
    } else {
      const long long u = w - static_cast<long long>(nblocks) * 6 * dim;
      v = final_table[u] + emb[static_cast<long long>(b) * dim + (u % dim)];
    }
    mod[i] = v;
  }
}

template <bool BF16>
__global__ void cast16_kernel(const float* __restrict__ in, uint16_t* __restrict__ out, long long n4) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    reinterpret_cast<uint2*>(out)[i] = make_uint2(pack2<BF16>(v.x, v.y), pack2<BF16>(v.z, v.w));
  }
}

__global__ void fill_kernel(float* __restrict__ p, float v, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    p[i] = v;
}

}  // namespace

int launch_t2v_mod(const float* tables, const float* ts, const float* final_table, const float* emb, float* mod, int batch,
                   int nblocks, int dim, cudaStream_t stream) {
  const long long total = (static_cast<long long>(nblocks) * 6 * dim + 2 * dim) * batch;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 2048) blocks = 2048;
  t2v_mod_kernel<<<blocks, 256, 0, stream>>>(tables, ts, final_table, emb, mod, batch, nblocks, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_cast16(const float* in, void* out16, long long n, int bf16, cudaStream_t stream) {
  B200_REQUIRE(n % 4 == 0, B200_ERR_SHAPE, "cast16: element count %lld must be a multiple of 4", n);
  const long long n4 = n / 4;
  int blocks = static_cast<int>((n4 + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (bf16) cast16_kernel<true><<<blocks, 256, 0, stream>>>(in, reinterpret_cast<uint16_t*>(out16), n4);
  else cast16_kernel<false><<<blocks, 256, 0, stream>>>(in, reinterpret_cast<uint16_t*>(out16), n4);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_fill(float* p, float v, long long n, cudaStream_t stream) {
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 1024) blocks = 1024;
  fill_kernel<<<blocks, 256, 0, stream>>>(p, v, n);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_ln_modulate(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                       int rows_per_batch, void* out16, int rows, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && dim <= LN_MAXV * 128, B200_ERR_SHAPE,
               "ln_modulate: dim %d must be a multiple of 4 and <= %d", dim, LN_MAXV * 128);
  B200_REQUIRE(rows_per_batch > 0 && mod_batch_stride % 4 == 0, B200_ERR_SHAPE, "ln_modulate: bad batch geometry");
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(scale)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(out16) & 7) == 0,
               B200_ERR_ALIGN, "ln_modulate: pointers must be 16-byte aligned");
  int sms = 0;
  B200_TRY(device_sm_count(&sms));
  const int nvmax = (dim / 4 + 31) / 32;
  uint16_t* o = reinterpret_cast<uint16_t*>(out16);
  if (bf16) return ln_dispatch<true>(nvmax, stream, x, shift, scale, mod_batch_stride, rows_per_batch, o, rows, dim, sms);
  return ln_dispatch<false>(nvmax, stream, x, shift, scale, mod_batch_stride, rows_per_batch, o, rows, dim, sms);
}

int launch_ln_modulate_e4m3(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                            int rows_per_batch, void* out8, float* row_scale, int rows, int dim, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 16 == 0 && dim <= LN_MAXV * 128, B200_ERR_SHAPE,
               "ln_modulate_e4m3: dim %d must be a multiple of 16 and <= %d", dim, LN_MAXV * 128);
  B200_REQUIRE(rows_per_batch > 0 && mod_batch_stride % 4 == 0, B200_ERR_SHAPE, "ln_modulate_e4m3: bad batch geometry");
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(scale) |
                 reinterpret_cast<uintptr_t>(out8)) & 15) == 0 && row_scale && (reinterpret_cast<uintptr_t>(row_scale) & 3) == 0,
               B200_ERR_ALIGN, "ln_modulate_e4m3: x, shift, scale, out must be 16-byte aligned, row_scale 4-byte");
  int sms = 0;
  B200_TRY(device_sm_count(&sms));
  return ln_dispatch_e4m3((dim / 4 + 31) / 32, stream, x, shift, scale, mod_batch_stride, rows_per_batch,
                          static_cast<uint8_t*>(out8), row_scale, rows, dim, sms);
}

int launch_quantize_rows_e4m3(const float* w, int rows, int cols, void* q8, float* scales, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && cols > 0, B200_ERR_SHAPE, "quantize_rows_e4m3: bad shape %d x %d", rows, cols);
  B200_REQUIRE(cols % 16 == 0, B200_ERR_UNSUPPORTED, "quantize_rows_e4m3: cols %d must be a multiple of 16 (16-byte rows)", cols);
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(q8)) & 15) == 0 && scales &&
                   (reinterpret_cast<uintptr_t>(scales) & 3) == 0,
               B200_ERR_ALIGN, "quantize_rows_e4m3: w and q must be 16-byte aligned, scales 4-byte");
  const int blocks = (rows + 7) / 8;
  quantize_rows_e4m3_kernel<<<blocks, 256, 0, stream>>>(w, rows, cols, static_cast<uint32_t*>(q8), scales);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_patch_embed(const float* x, int x_batch_mod, const float* w, const float* b, const float* pos, float* out,
                       int batch, int frames, int chans, int size, int patch, int dim, int channels_first, cudaStream_t stream) {
  const int K = chans * patch * patch;
  B200_REQUIRE(size % patch == 0, B200_ERR_SHAPE, "patch_embed: size %d not divisible by patch %d", size, patch);
  B200_REQUIRE(K == 4 || K == 8 || K == 16 || K == 32 || K == 64 || K == 256, B200_ERR_UNSUPPORTED,
               "patch_embed: C*p*p = %d unsupported (4, 8, 16, 32, 64, 256)", K);
  const int grid = size / patch;
  const int total = batch * frames * grid * grid;
  const int blocks = (total + PE_TOK - 1) / PE_TOK;
  // x is [b][f][c][h][w] (Latte, latte.py:329) or [b][c][f][h][w] (LatteT2V, latte_t2v.py:731)
  const long long plane = static_cast<long long>(size) * size;
  const long long sb = plane * chans * frames;
  const long long sf = channels_first ? plane : plane * chans;
  const long long sc = channels_first ? plane * frames : plane;
#define B200_PE(KERNEL, KK) KERNEL<KK><<<blocks, 320, 0, stream>>>(x, x_batch_mod, w, b, pos, out, total, frames, chans, size, patch, dim, sb, sf, sc)
  switch (K) {
    case 4: B200_PE(patch_embed_kernel, 4); break;
    case 8: B200_PE(patch_embed_kernel, 8); break;
    case 16: B200_PE(patch_embed_kernel, 16); break;
    case 32: B200_PE(patch_embed_kernel, 32); break;
    case 64: B200_PE(patch_embed_wide_kernel, 64); break;
    default: B200_PE(patch_embed_wide_kernel, 256); break;
  }
#undef B200_PE
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_timestep_freq(const long long* t, float* out, int batch, cudaStream_t stream) {
  timestep_freq_kernel<<<batch, 256, 0, stream>>>(t, out, batch);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_gemv(const void* W, int wbits, int bf16, const float* bias, const float* in, float* out, int batch, int J,
                int K, int silu_in, int silu_out, const float* add_table, const long long* add_idx, int add_rows,
                cudaStream_t stream) {
  B200_REQUIRE(K % 8 == 0 && J > 0, B200_ERR_SHAPE, "gemv: K=%d must be a multiple of 8", K);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(W) & 15) == 0, B200_ERR_ALIGN, "gemv: W must be 16-byte aligned");
  int sms = 0;
  B200_TRY(device_sm_count(&sms));
  for (int b0 = 0; b0 < batch; b0 += GV_MAXB) {
    const int nb = (batch - b0) < GV_MAXB ? (batch - b0) : GV_MAXB;
    const size_t smem = static_cast<size_t>(nb) * K * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, B200_ERR_SHAPE, "gemv: K=%d too large", K);
    const int warps = 8;
    int blocks = (J + warps * GV_ROWS - 1) / (warps * GV_ROWS);
    const int cap = sms * 8;
    if (blocks > cap) blocks = cap;
    const float* inb = in + static_cast<size_t>(b0) * K;
    float* outb = out + static_cast<size_t>(b0) * J;
    const long long* idx = add_idx ? add_idx + b0 : nullptr;
    if (wbits == 32)
      gemv_kernel<32, false><<<blocks, warps * 32, smem, stream>>>(W, bias, inb, outb, nb, J, K, silu_in, silu_out, add_table, idx, add_rows);
    else if (bf16)
      gemv_kernel<16, true><<<blocks, warps * 32, smem, stream>>>(W, bias, inb, outb, nb, J, K, silu_in, silu_out, add_table, idx, add_rows);
    else
      gemv_kernel<16, false><<<blocks, warps * 32, smem, stream>>>(W, bias, inb, outb, nb, J, K, silu_in, silu_out, add_table, idx, add_rows);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  return B200_OK;
}

int launch_final_layer(const float* x, const float* shift, const float* scale, long long mod_batch_stride,
                       const float* w, const float* b, float* out, int batch, int frames, int grid, int patch,
                       int out_ch, int dim, int channels_first, cudaStream_t stream) {
  const int n_out = patch * patch * out_ch;
  B200_REQUIRE(n_out <= FL_MAXO && dim % 4 == 0 && dim <= FL_MAXV * 128, B200_ERR_SHAPE,
               "final_layer: p*p*Cout = %d must be <= %d, dim %d <= %d", n_out, FL_MAXO, dim, FL_MAXV * 128);
  const size_t smem = static_cast<size_t>(n_out) * dim * sizeof(float);
  B200_SET_SMEM_ONCE(final_layer_kernel, 200 * 1024);
  B200_REQUIRE(smem <= 200 * 1024, B200_ERR_SHAPE, "final_layer: weight tile %zu B exceeds shared memory", smem);
  int sms = 0;
  B200_TRY(device_sm_count(&sms));
  const int total = batch * frames * grid * grid;
  const int warps = 16;
  int blocks = (total + warps - 1) / warps;
  if (blocks > sms) blocks = sms;
  const long long plane = static_cast<long long>(grid * patch) * (grid * patch);
  const long long sb = plane * out_ch * frames;
  const long long sf = channels_first ? plane : plane * out_ch;
  const long long sc = channels_first ? plane * frames : plane;
  final_layer_kernel<<<blocks, warps * 32, smem, stream>>>(x, shift, scale, mod_batch_stride, w, b, out, total, frames,
                                                            grid, patch, out_ch, dim, sb, sf, sc);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_rms_norm(const float* x, const float* w, void* out16, float* out32, int rows, int dim, float eps, int bf16,
                    cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim % 4 == 0, B200_ERR_SHAPE, "rms_norm: dim %d must be a multiple of 4", dim);
  B200_REQUIRE((out16 != nullptr) != (out32 != nullptr), B200_ERR_SHAPE, "rms_norm: exactly one of out16 / out32");
  const int blocks = (rows + 7) / 8;
  if (bf16) rms_norm_kernel<true><<<blocks, 256, 0, stream>>>(x, w, static_cast<uint16_t*>(out16), out32, rows, dim, eps);
  else rms_norm_kernel<false><<<blocks, 256, 0, stream>>>(x, w, static_cast<uint16_t*>(out16), out32, rows, dim, eps);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_embed(const long long* ids, const void* table16, float* x, int rows, int dim, int vocab, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim % 4 == 0, B200_ERR_SHAPE, "embed: dim %d must be a multiple of 4", dim);
  if (bf16) embed_kernel<true><<<rows, 256, 0, stream>>>(ids, static_cast<const uint16_t*>(table16), x, rows, dim, vocab);
  else embed_kernel<false><<<rows, 256, 0, stream>>>(ids, static_cast<const uint16_t*>(table16), x, rows, dim, vocab);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_frames_to_uint8(const void* video, int dtype, int n, int c, int h, int w, int mode, uint8_t* out, cudaStream_t stream) {
  B200_REQUIRE(video && out && n > 0 && c > 0 && h > 0 && w > 0, B200_ERR_SHAPE, "frames_to_uint8: bad arguments");
  B200_REQUIRE(dtype >= 0 && dtype <= 2 && (mode == 0 || mode == 1), B200_ERR_UNSUPPORTED, "frames_to_uint8: dtype %d / mode %d", dtype, mode);
  const long long total = static_cast<long long>(n) * c * h * w;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (dtype == 0) frames_to_uint8_kernel<0><<<blocks, 256, 0, stream>>>(video, out, total, c, h * w, mode);
  else if (dtype == 1) frames_to_uint8_kernel<1><<<blocks, 256, 0, stream>>>(video, out, total, c, h * w, mode);
  else frames_to_uint8_kernel<2><<<blocks, 256, 0, stream>>>(video, out, total, c, h * w, mode);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_unpatchify(const float* y, float* out, int batch, int frames, int grid, int patch, int out_ch, int channels_first,
                      cudaStream_t stream) {
  const long long plane = static_cast<long long>(grid * patch) * (grid * patch);
  const long long total = static_cast<long long>(batch) * frames * out_ch * plane;
  const long long sb = plane * out_ch * frames;
  const long long sf = channels_first ? plane : plane * out_ch;
  const long long sc = channels_first ? plane * frames : plane;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  unpatchify_kernel<<<blocks, 256, 0, stream>>>(y, out, total, frames, grid, patch, out_ch, patch * patch * out_ch, sb, sf, sc);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_cfg_combine(float* out, int batch, long long per_sample, int frames, int out_ch, int guided_ch, int hw,
                       float scale, cudaStream_t stream) {
  (void)frames;
  B200_REQUIRE(batch % 2 == 0, B200_ERR_SHAPE, "cfg: batch %d must be even", batch);
  const long long total = static_cast<long long>(batch / 2) * per_sample;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  cfg_combine_kernel<<<blocks, 256, 0, stream>>>(out, batch / 2, per_sample, out_ch, guided_ch, hw, scale);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

}  // namespace b200
