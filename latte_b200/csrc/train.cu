// Backward-pass kernels of the training step (BASELINE config 5; reference train.py:206-222 -> autograd over models/latte.py).
// Every GEMM of the backward (dgrad, wgrad) runs on the wgmma kernel of gemm.cu; this file holds what surrounds them:
//   transpose16                    16-bit [R,C] -> [C,R] operands for wgrad (K = tokens must be the contiguous dimension)
//   multi_cast / multi_tensor      fp32 -> 16-bit operand copies; gradient norm, clipping and EMA, many tensors per launch
//   gate_residual                  x_out = x + gate[b] * m (+ temp_embed row)          forward of latte.py:179-180 residuals
//   gelu_bwd                       tanh-GELU derivative, bias gradient (column sums) fused               (latte.py:169-171)
//   gate_bwd                       dm = dx * gate[b]; dgate[b] = sum_rows dx * m; dbias = sum_rows dm   (latte.py:179-180)
//   colsum                         column sums (bias gradients of the plain Linear layers)
//   ln_modulate_bwd                d/dx of LN(x)(1+scale)+shift accumulated into dx; dshift, dscale per sample (latte.py:28-29)
//   attn_bwd_dq / attn_bwd_dkv     softmax(QK^T hd^-1/2)V backward on mma.sync tensor cores, scores recomputed (latte.py:48-77)
//                                  (also the temporal sequences of 17..128 frames: strided rows, partial last block masked)
//   attn_bwd_temporal_mma          same for the F <= 16 frame sequences (one 16-row tile per (b, n, head))
// The attention backward takes head_dim 64 or 72 only.
//   ada_outer / ada_dsc            gradients of the stacked adaLN_modulation Linear on B rows  (latte.py:160-163,192-195)
// All are HBM-bound passes (one read, one write, fp32 math) except the attention backward (tensor cores, ~2 % of the FLOPs).
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool BF16>
__device__ __forceinline__ float cvt1(uint16_t u) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(u) << 16);
  else return __half2float(*reinterpret_cast<const __half*>(&u));
}
template <bool BF16>
__device__ __forceinline__ uint16_t rnd1(float f) {
  const uint32_t p = pack2<BF16>(f, 0.f);
  return static_cast<uint16_t>(p & 0xffffu);
}

// ------------------------------------------------------------------------------------------------ transposes
// 64x64 tile through shared memory; 4-byte global accesses on both sides.  R, C even.
__global__ void __launch_bounds__(256) transpose16_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, int R, int C) {
  __shared__ uint16_t tile[64][66];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 64; r += 8) {
    const int row = r0 + r, col = c0 + 2 * tx;
    uint32_t v = 0;
    if (row < R && col < C) v = *reinterpret_cast<const uint32_t*>(in + static_cast<size_t>(row) * C + col);
    tile[r][2 * tx] = static_cast<uint16_t>(v & 0xffffu);
    tile[r][2 * tx + 1] = static_cast<uint16_t>(v >> 16);
  }
  __syncthreads();
  for (int c = ty; c < 64; c += 8) {
    const int orow = c0 + c, ocol = r0 + 2 * tx;
    if (orow < C && ocol < R) {
      const uint32_t v = static_cast<uint32_t>(tile[2 * tx][c]) | (static_cast<uint32_t>(tile[2 * tx + 1][c]) << 16);
      *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(orow) * R + ocol) = v;
    }
  }
}

// fp32 -> 16-bit cast of MANY tensors in one launch (the operand copies of all parameters at the start of a training step:
// 116 weights = 116 launches of a few microseconds each otherwise, which left the GPU waiting for the host).
// table[e] = {src, dst, n4 = float4 count, first_chunk}; a chunk = 1024 float4.  Chunks are dealt to blocks grid-stride; the
// owning entry is found by binary search on first_chunk.
struct MultiCastEntry { const float* src; uint16_t* dst; long long n4; long long first_chunk; };
constexpr int MC_CHUNK = 1024;
template <bool BF16>
__global__ void __launch_bounds__(256) multi_cast_kernel(const MultiCastEntry* __restrict__ tab, int n_entries, long long total_chunks) {
  for (long long c = blockIdx.x; c < total_chunks; c += gridDim.x) {
    int lo = 0, hi = n_entries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab[mid].first_chunk <= c) lo = mid; else hi = mid - 1;
    }
    const MultiCastEntry e = tab[lo];
    const long long base = (c - e.first_chunk) * MC_CHUNK;
#pragma unroll
    for (int j = 0; j < MC_CHUNK / 256; ++j) {
      const long long i = base + j * 256 + threadIdx.x;
      if (i < e.n4) {
        const float4 f = __ldg(reinterpret_cast<const float4*>(e.src) + i);
        reinterpret_cast<uint2*>(e.dst)[i] = make_uint2(pack2<BF16>(f.x, f.y), pack2<BF16>(f.z, f.w));
      }
    }
  }
}

// Multi-tensor fp32 passes over lists of parameters / gradients (the reference's python loops `clip_grad_norm_`,
// utils.py:72-125, and `update_ema`, utils.py:190-200: two tiny kernels per parameter tensor = ~1200 launches per step for
// XL/2's 293 tensors).  Same table layout as multi_cast ({src, dst, n elements, first_chunk}, a chunk = 4096 elements).
//   MT_SUMSQ  *accum (double) += sum src^2          MT_SCALE  dst *= *scalar          MT_AXPBY  dst = a * dst + b * src
enum { MT_SUMSQ = 1, MT_SCALE = 2, MT_AXPBY = 3 };
struct MultiTensorEntry { const float* src; float* dst; long long n; long long first_chunk; };
constexpr int MT_CHUNK = 4096;
template <int OP>
__global__ void __launch_bounds__(256) multi_tensor_kernel(const MultiTensorEntry* __restrict__ tab, int n_entries, long long total_chunks,
                                                           float a, float b, const float* __restrict__ scalar, double* __restrict__ accum) {
  float local = 0.f;
  const float sc = (OP == MT_SCALE) ? __ldg(scalar) : 0.f;
  for (long long c = blockIdx.x; c < total_chunks; c += gridDim.x) {
    int lo = 0, hi = n_entries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab[mid].first_chunk <= c) lo = mid; else hi = mid - 1;
    }
    const MultiTensorEntry e = tab[lo];
    const long long base = (c - e.first_chunk) * MT_CHUNK;
    const long long end = min(e.n, base + MT_CHUNK);
    const bool vec = ((reinterpret_cast<uintptr_t>(e.src) | reinterpret_cast<uintptr_t>(e.dst)) & 15) == 0;
    if (vec) {
      const long long v0 = base >> 2, v1 = end >> 2;       // base is a multiple of 4096
      for (long long i = v0 + threadIdx.x; i < v1; i += 256) {
        if constexpr (OP == MT_SUMSQ) {
          const float4 f = __ldg(reinterpret_cast<const float4*>(e.src) + i);
          local += (f.x * f.x + f.y * f.y) + (f.z * f.z + f.w * f.w);
        } else if constexpr (OP == MT_SCALE) {
          float4 d = reinterpret_cast<float4*>(e.dst)[i];
          d.x *= sc; d.y *= sc; d.z *= sc; d.w *= sc;
          reinterpret_cast<float4*>(e.dst)[i] = d;
        } else {
          const float4 f = __ldg(reinterpret_cast<const float4*>(e.src) + i);
          float4 d = reinterpret_cast<float4*>(e.dst)[i];
          d.x = a * d.x + b * f.x; d.y = a * d.y + b * f.y; d.z = a * d.z + b * f.z; d.w = a * d.w + b * f.w;
          reinterpret_cast<float4*>(e.dst)[i] = d;
        }
      }
    }
    for (long long i = (vec ? (end & ~3LL) : base) + threadIdx.x; i < end; i += 256) {     // tail / unaligned tensors
      if constexpr (OP == MT_SUMSQ) { const float f = e.src[i]; local += f * f; }
      else if constexpr (OP == MT_SCALE) e.dst[i] *= sc;
      else e.dst[i] = a * e.dst[i] + b * e.src[i];
    }
  }
  if constexpr (OP == MT_SUMSQ) {
    __shared__ float red[8];
    local = warp_sum(local);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += static_cast<double>(red[w]);
      atomicAdd(accum, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------ gate_residual (forward)
// out[r, :] = x[r, :] + gate[r / rpb, :] * m[r, :] (+ row_add[(r / tokens) % frames, :]).  Thread = 4 columns.
template <bool BF16>
__global__ void __launch_bounds__(256) gate_residual_kernel(const float* __restrict__ x, const uint16_t* __restrict__ m,
                                                            const float* __restrict__ gate, long long gate_bs, int rpb,
                                                            const float* __restrict__ row_add, int tokens, int frames,
                                                            float* __restrict__ out, int rows, int dim) {
  const int nv = dim >> 2;
  const long long total = static_cast<long long>(rows) * nv;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int row = static_cast<int>(i / nv), c4 = static_cast<int>(i % nv);
    const float4 xv = reinterpret_cast<const float4*>(x)[i];
    const uint2 mv = reinterpret_cast<const uint2*>(m)[i];
    const float4 g = __ldg(reinterpret_cast<const float4*>(gate + (row / rpb) * gate_bs) + c4);
    const float2 m0 = unpack2<BF16>(mv.x), m1 = unpack2<BF16>(mv.y);
    float4 o = make_float4(fmaf(g.x, m0.x, xv.x), fmaf(g.y, m0.y, xv.y), fmaf(g.z, m1.x, xv.z), fmaf(g.w, m1.y, xv.w));
    if (row_add != nullptr) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(row_add + static_cast<size_t>((row / tokens) % frames) * dim) + c4);
      o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
    }
    reinterpret_cast<float4*>(out)[i] = o;
  }
}

// ------------------------------------------------------------------------------------------------ GELU (tanh form)
// one MUFU op per element (tanh.approx, relative error 2^-11 -- below the 16-bit rounding of the result), as in the GEMM's
// GELU epilogue: with libm's tanhf the backward pass was ALU-bound (~60 instructions per element on 94 M elements per call)
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_grad(float u) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u2 = u * u;
  const float th = tanh_fast(k0 * fmaf(k1 * u2, u, u));
  const float sech2 = fmaf(-th, th, 1.0f);
  return fmaf(0.5f * u * sech2, k0 * fmaf(3.0f * k1, u2, 1.0f), fmaf(0.5f, th, 0.5f));
}

// du = da * gelu'(u); dbias[c] += sum over the block's rows.  Block = 128 threads x 8 columns.
template <bool BF16>
__global__ void __launch_bounds__(128) gelu_bwd_kernel(const uint16_t* __restrict__ da, const uint16_t* __restrict__ u,
                                                       uint16_t* __restrict__ du, float* __restrict__ dbias, int rows, int dim) {
  // Rows are dealt round-robin to the gridDim.y row-lanes (lane y takes rows y, y + G, ...): at any moment the whole grid
  // works inside one sliding window of G consecutive rows, which DRAM serves far better than G far-apart row slabs.
  const int c8 = blockIdx.x * 128 + threadIdx.x;
  if (c8 * 8 >= dim) return;
  const int G = gridDim.y;
  float acc[8] = {};
  const int nv = dim >> 3;
  // explicit load batches: U rows of both streams are requested before any of them is consumed (left to itself the compiler
  // interleaves load -> math -> store per row and keeps ~2 rows in flight per thread)
  constexpr int U = 4;
  for (int r = blockIdx.y; r < rows; r += U * G) {
    uint4 av[U], bv[U];
#pragma unroll
    for (int t = 0; t < U; ++t) {
      const int rt = r + t * G;
      if (rt < rows) {
        const size_t idx = static_cast<size_t>(rt) * nv + c8;
        av[t] = __ldg(reinterpret_cast<const uint4*>(da) + idx);
        bv[t] = __ldg(reinterpret_cast<const uint4*>(u) + idx);
      }
    }
#pragma unroll
    for (int t = 0; t < U; ++t) {
      const int rt = r + t * G;
      if (rt < rows) {
        const uint32_t aw[4] = {av[t].x, av[t].y, av[t].z, av[t].w}, bw[4] = {bv[t].x, bv[t].y, bv[t].z, bv[t].w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 g = unpack2<BF16>(aw[j]), uu = unpack2<BF16>(bw[j]);
          const float d0 = g.x * gelu_grad(uu.x), d1 = g.y * gelu_grad(uu.y);
          o[j] = pack2<BF16>(d0, d1);
          acc[2 * j] += d0;
          acc[2 * j + 1] += d1;
        }
        reinterpret_cast<uint4*>(du)[static_cast<size_t>(rt) * nv + c8] = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) atomicAdd(dbias + c8 * 8 + j, acc[j]);
}

// ------------------------------------------------------------------------------------------------ gate_bwd
// dm = dx * gate[b] (16-bit); dgate[b, c] += sum_rows dx * m; dbias[c] += sum_rows dm.  Thread = 4 columns.
template <bool BF16>
__global__ void __launch_bounds__(128) gate_bwd_kernel(const float* __restrict__ dx, const uint16_t* __restrict__ m,
                                                       const float* __restrict__ gate, long long gate_bs, int rpb,
                                                       uint16_t* __restrict__ dm, float* __restrict__ dgate, long long dgate_bs,
                                                       float* __restrict__ dbias, int rows, int dim) {
  // grid (column strips, G row-lanes, samples): lane y of sample b takes rows b*rpb + y, + G, ... (sliding window, see gelu_bwd)
  const int c4 = blockIdx.x * 128 + threadIdx.x;
  const int nv = dim >> 2;
  if (c4 >= nv) return;
  const int G = gridDim.y;
  const int b = blockIdx.z;
  const int r0 = b * rpb + blockIdx.y;
  const int r1 = min(rows, (b + 1) * rpb);
  const float4 g = __ldg(reinterpret_cast<const float4*>(gate + b * gate_bs) + c4);
  float ag[4] = {}, ab[4] = {};
  constexpr int U = 8;            // explicit load batches, see gelu_bwd
  for (int r = r0; r < r1; r += U * G) {
    float4 dv[U];
    uint2 mv[U];
#pragma unroll
    for (int t = 0; t < U; ++t) {
      const int rt = r + t * G;
      if (rt < r1) {
        const size_t idx = static_cast<size_t>(rt) * nv + c4;
        dv[t] = __ldg(reinterpret_cast<const float4*>(dx) + idx);
        mv[t] = __ldg(reinterpret_cast<const uint2*>(m) + idx);
      }
    }
#pragma unroll
    for (int t = 0; t < U; ++t) {
      const int rt = r + t * G;
      if (rt < r1) {
        const float4 d = dv[t];
        const float2 m0 = unpack2<BF16>(mv[t].x), m1 = unpack2<BF16>(mv[t].y);
        const float o0 = d.x * g.x, o1 = d.y * g.y, o2 = d.z * g.z, o3 = d.w * g.w;
        reinterpret_cast<uint2*>(dm)[static_cast<size_t>(rt) * nv + c4] = make_uint2(pack2<BF16>(o0, o1), pack2<BF16>(o2, o3));
        ag[0] += d.x * m0.x; ag[1] += d.y * m0.y; ag[2] += d.z * m1.x; ag[3] += d.w * m1.y;
        ab[0] += o0; ab[1] += o1; ab[2] += o2; ab[3] += o3;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    atomicAdd(dgate + b * dgate_bs + c4 * 4 + j, ag[j]);
    atomicAdd(dbias + c4 * 4 + j, ab[j]);
  }
}

// column sums of a [rows, dim] matrix (16-bit or fp32) into fp32 (pre-zeroed)
template <int KIND>   // 0 fp32, 1 fp16, 2 bf16
__global__ void __launch_bounds__(128) colsum_kernel(const void* __restrict__ a, float* __restrict__ out, int rows, int dim) {
  const int c4 = blockIdx.x * 128 + threadIdx.x;
  const int nv = dim >> 2;
  if (c4 >= nv) return;
  const int G = gridDim.y;
  float acc[4] = {};
  constexpr int U = 8;            // explicit load batches, see gelu_bwd
  for (int r = blockIdx.y; r < rows; r += U * G) {
    if constexpr (KIND == 0) {
      float4 d[U];
#pragma unroll
      for (int t = 0; t < U; ++t)
        if (r + t * G < rows) d[t] = __ldg(reinterpret_cast<const float4*>(a) + static_cast<size_t>(r + t * G) * nv + c4);
#pragma unroll
      for (int t = 0; t < U; ++t)
        if (r + t * G < rows) { acc[0] += d[t].x; acc[1] += d[t].y; acc[2] += d[t].z; acc[3] += d[t].w; }
    } else {
      uint2 v[U];
#pragma unroll
      for (int t = 0; t < U; ++t)
        if (r + t * G < rows) v[t] = __ldg(reinterpret_cast<const uint2*>(a) + static_cast<size_t>(r + t * G) * nv + c4);
#pragma unroll
      for (int t = 0; t < U; ++t)
        if (r + t * G < rows) {
          const float2 f0 = unpack2<KIND == 2>(v[t].x), f1 = unpack2<KIND == 2>(v[t].y);
          acc[0] += f0.x; acc[1] += f0.y; acc[2] += f1.x; acc[3] += f1.y;
        }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) atomicAdd(out + c4 * 4 + j, acc[j]);
}

// ------------------------------------------------------------------------------------------------ ln_modulate_bwd
// h = xhat * (1 + scale[b]) + shift[b], xhat = (x - mean) * rstd.  Given dh:
//   dshift[b] += sum_rows dh;  dscale[b] += sum_rows dh * xhat;  g = dh * (1 + scale[b]);
//   dx += rstd * (g - mean(g) - xhat * mean(g * xhat)).
// One warp per row (row in registers); the warps of a block reduce their column sums through shared memory before the
// atomics.

template <bool BF16, int NV>
__global__ void __launch_bounds__(256) ln_modulate_bwd_kernel(const uint16_t* __restrict__ dh, const float* __restrict__ x,
                                                              const float* __restrict__ scale, long long mod_bs, int rpb,
                                                              float* __restrict__ dx, float* __restrict__ dshift,
                                                              float* __restrict__ dscale, long long dmod_bs, int rows, int dim) {
  extern __shared__ float s_red[];   // [warps][2][dim]: per-warp column sums of dh and dh * xhat (each lane owns its columns)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nw = blockDim.x >> 5;
  const int nv = dim >> 2;
  // grid (blocks per sample, samples).  The warps of a sample take its rows round-robin (warp gw: rows gw, gw + W, ...), so the
  // grid sweeps every sample front to back inside a window of W consecutive rows (DRAM locality, see gelu_bwd).
  const int b = blockIdx.y;
  const int W = gridDim.x * nw;
  const int gw = blockIdx.x * nw + warp;
  const float4* sc = reinterpret_cast<const float4*>(scale + b * mod_bs);
  float4* red_sh = reinterpret_cast<float4*>(s_red) + (warp * 2 + 0) * nv;
  float4* red_sc = reinterpret_cast<float4*>(s_red) + (warp * 2 + 1) * nv;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) red_sh[idx] = red_sc[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float inv_d = 1.0f / static_cast<float>(dim);
  for (int rr = gw; rr < rpb; rr += W) {
    const int row = b * rpb + rr;
    if (row >= rows) break;
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * dim);
    const uint2* dr = reinterpret_cast<const uint2*>(dh + static_cast<size_t>(row) * dim);
    float4* dxr = reinterpret_cast<float4*>(dx + static_cast<size_t>(row) * dim);
    float4 v[NV], o[NV];
    uint2 dpk[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {           // all three streams of the row are requested up front
      const int idx = lane + i * 32;
      if (idx < nv) {
        v[i] = xr[idx];
        dpk[i] = dr[idx];
        o[i] = dxr[idx];
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nv) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * inv_d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (lane + i * 32 < nv) {
        v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
        q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_d + 1e-6f);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) {
        v[i].x *= rstd; v[i].y *= rstd; v[i].z *= rstd; v[i].w *= rstd;          // xhat
        const float2 d0 = unpack2<BF16>(dpk[i].x), d1 = unpack2<BF16>(dpk[i].y);
        float4 a = red_sh[idx], c2 = red_sc[idx];
        a.x += d0.x; a.y += d0.y; a.z += d1.x; a.w += d1.y;
        c2.x += d0.x * v[i].x; c2.y += d0.y * v[i].y; c2.z += d1.x * v[i].z; c2.w += d1.y * v[i].w;
        red_sh[idx] = a;
        red_sc[idx] = c2;
        const float4 c = __ldg(sc + idx);
        const float g0 = d0.x * (1.0f + c.x), g1 = d0.y * (1.0f + c.y), g2 = d1.x * (1.0f + c.z), g3 = d1.y * (1.0f + c.w);
        s1 += (g0 + g1) + (g2 + g3);
        s2 += (g0 * v[i].x + g1 * v[i].y) + (g2 * v[i].z + g3 * v[i].w);
      }
    }
    s1 = warp_sum(s1) * inv_d;
    s2 = warp_sum(s2) * inv_d;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) {
        const float2 d0 = unpack2<BF16>(dpk[i].x), d1 = unpack2<BF16>(dpk[i].y);
        const float4 c = __ldg(sc + idx);
        float4 r = o[i];
        r.x += rstd * (d0.x * (1.0f + c.x) - s1 - v[i].x * s2);
        r.y += rstd * (d0.y * (1.0f + c.y) - s1 - v[i].y * s2);
        r.z += rstd * (d1.x * (1.0f + c.z) - s1 - v[i].z * s2);
        r.w += rstd * (d1.y * (1.0f + c.w) - s1 - v[i].w * s2);
        dxr[idx] = r;
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * dim; i += blockDim.x) {
    const int which = i / dim, c = i % dim;
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += s_red[(w * 2 + which) * dim + c];
    atomicAdd((which == 0 ? dshift : dscale) + b * dmod_bs + c, t);
  }
}

// ------------------------------------------------------------------------------------------------ attention backward (spatial)
// mma.sync m16n8k16 building blocks.  Shared-memory tiles are [64 rows][HDP] 16-bit with HDP = KP + 8 (KP = head_dim rounded up
// to 16; the pad columns [HD, KP) are zero so they add nothing to a k = head_dim contraction); the 8-element skew makes the
// eight 16-byte rows of an ldmatrix land in distinct bank groups.
template <bool BF16>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (BF16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

__device__ __forceinline__ void ldsm_x2_t(uint32_t& r0, uint32_t& r1, uint32_t addr) {   // lanes 0-15 supply the row addresses
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

template <int HD>
struct AB {
  static constexpr int KP = (HD + 15) / 16 * 16;   // 64 or 80
  static constexpr int KS = KP / 16;               // k-steps of a head_dim contraction
  static constexpr int HDP = KP + 8;               // row pitch in elements
  static constexpr int NT = HD / 8;                // n-tiles of a head_dim-wide output (8 or 9)
  static constexpr int TILE = 64 * HDP;            // elements per 64-row tile
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

// asynchronous copy of a [64 x HD] block (rows row0.., columns col0..col0+HD) of a row-major 16-bit matrix into a shared tile.
// STRIDED (temporal sequences): tile row r is matrix row row0 + r * rs for r < nvalid; rows r >= nvalid are past the end of the
// sequence and are written with zeros, never left stale (a stale NaN would survive P = 0 in the MMAs).
template <int HD, bool STRIDED = false>
__device__ __forceinline__ void load_tile64(uint16_t* s, const uint16_t* __restrict__ g, size_t row0, int ld, int col0, int rs = 1,
                                            int nvalid = 64) {
  constexpr int CH = HD / 8;          // 16-byte chunks per row
  constexpr int HDP = AB<HD>::HDP;
  for (int i = threadIdx.x; i < 64 * CH; i += blockDim.x) {
    const int r = i / CH, c = i % CH;
    if constexpr (STRIDED) {
      if (r < nvalid) cp_async16(s + r * HDP + c * 8, g + (row0 + static_cast<size_t>(r) * rs) * ld + col0 + c * 8);
      else *reinterpret_cast<uint4*>(s + r * HDP + c * 8) = make_uint4(0, 0, 0, 0);
    } else {
      cp_async16(s + r * HDP + c * 8, g + (row0 + r) * ld + col0 + c * 8);
    }
  }
}
// zero the pad columns [HD, KP) of `ntiles` consecutive tiles once (the copies above never touch them)
template <int HD>
__device__ __forceinline__ void zero_pads(uint16_t* s, int ntiles) {
  if constexpr (AB<HD>::KP > HD) {
    for (int r = threadIdx.x; r < 64 * ntiles; r += blockDim.x) *reinterpret_cast<uint4*>(s + r * AB<HD>::HDP + HD) = make_uint4(0, 0, 0, 0);
  }
}

// acc[16 x 64] = A[16 x KP] . tile[64 x KP]^T: A = rows [r0, r0+16) of shared tile sA (fragments fetched per k-step, so they
// do not occupy registers across the loop), tile rows are the n dimension, its columns the contraction.
template <bool BF16, int HD>
__device__ __forceinline__ void mm_a_tileT(float (&acc)[8][4], const uint16_t* sA, int r0, const uint16_t* s) {
  const int lane = threadIdx.x & 31;
  const int arow = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
  const int acol = (lane >> 4) * 8;
  const int brow = (lane & 7) + (lane >> 4) * 8;
  const int bcol = ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int k = 0; k < AB<HD>::KS; ++k) {
    uint32_t a[4];
    ldsm_x4(a, smem_u32(sA + arow * AB<HD>::HDP + k * 16 + acol));
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm_x4(b, smem_u32(s + (np * 16 + brow) * AB<HD>::HDP + k * 16 + bcol));
      mma16816<BF16>(acc[2 * np], a, b[0], b[1]);
      mma16816<BF16>(acc[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// out[16 x HD] += P[16 x 64] . tile[64 x HD]   (P given as 4 k-steps of A fragments; tile rows are the contraction)
template <bool BF16, int HD>
__device__ __forceinline__ void mm_p_tile(float (&out)[AB<HD>::NT][4], const uint32_t (&p)[4][4], const uint16_t* s) {
  const int lane = threadIdx.x & 31;
  const int brow = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int bcol = (lane >> 4) * 8;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int np = 0; np < AB<HD>::NT / 2; ++np) {
      uint32_t b[4];
      ldsm_x4_t(b, smem_u32(s + (k * 16 + brow) * AB<HD>::HDP + np * 16 + bcol));
      mma16816<BF16>(out[2 * np], p[k], b[0], b[1]);
      mma16816<BF16>(out[2 * np + 1], p[k], b[2], b[3]);
    }
    if constexpr (AB<HD>::NT % 2 == 1) {     // last single n-tile (head_dim 72): columns [HD-8, HD)
      uint32_t b0, b1;
      ldsm_x2_t(b0, b1, smem_u32(s + (k * 16 + brow) * AB<HD>::HDP + (AB<HD>::NT - 1) * 8));
      mma16816<BF16>(out[AB<HD>::NT - 1], p[k], b0, b1);
    }
  }
}

// pack a 16 x 64 fp32 accumulator block into 4 k-steps of A fragments
template <bool BF16>
__device__ __forceinline__ void acc_to_afrag(uint32_t (&p)[4][4], const float (&acc)[8][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    p[k][0] = pack2<BF16>(acc[2 * k][0], acc[2 * k][1]);
    p[k][1] = pack2<BF16>(acc[2 * k][2], acc[2 * k][3]);
    p[k][2] = pack2<BF16>(acc[2 * k + 1][0], acc[2 * k + 1][1]);
    p[k][3] = pack2<BF16>(acc[2 * k + 1][2], acc[2 * k + 1][3]);
  }
}

// write a warp's [16 x HD] fp32 accumulator as 16-bit rows of the output (row pitch ld; STRIDED: tile row r is row row0 + r * rs)
template <bool BF16, int HD, bool STRIDED = false>
__device__ __forceinline__ void store_rows(uint16_t* __restrict__ g, size_t row0, int ld, int col0, const float (&acc)[AB<HD>::NT][4],
                                           int r_in_tile, int nvalid, int rs = 1) {
  const int lane = threadIdx.x & 31;
  const int r = r_in_tile + (lane >> 2);
  if constexpr (STRIDED) {
    const size_t ra = row0 + static_cast<size_t>(r) * rs, rb = ra + static_cast<size_t>(8) * rs;
#pragma unroll
    for (int n = 0; n < AB<HD>::NT; ++n) {
      const int c = col0 + n * 8 + (lane & 3) * 2;
      if (r < nvalid) *reinterpret_cast<uint32_t*>(g + ra * ld + c) = pack2<BF16>(acc[n][0], acc[n][1]);
      if (r + 8 < nvalid) *reinterpret_cast<uint32_t*>(g + rb * ld + c) = pack2<BF16>(acc[n][2], acc[n][3]);
    }
  } else {
#pragma unroll
    for (int n = 0; n < AB<HD>::NT; ++n) {
      const int c = col0 + n * 8 + (lane & 3) * 2;
      if (r < nvalid) *reinterpret_cast<uint32_t*>(g + (row0 + r) * ld + c) = pack2<BF16>(acc[n][0], acc[n][1]);
      if (r + 8 < nvalid) *reinterpret_cast<uint32_t*>(g + (row0 + r + 8) * ld + c) = pack2<BF16>(acc[n][2], acc[n][3]);
    }
  }
}

// -inf for the key columns >= lim of a warp's [16 x 64] score block (the last, partial key block of a temporal sequence).
// The column of accumulator element (n, e) is n * 8 + (lane & 3) * 2 + (e & 1): one compare per score, no division.
__device__ __forceinline__ void mask_keys(float (&acc)[8][4], int lim) {
  const int c0 = (threadIdx.x & 3) * 2;
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (n * 8 + c0 + (e & 1) >= lim) acc[n][e] = -INFINITY;
}

// Kernel A: one CTA = 64 query rows of one (sequence, head).  Pass 1 recomputes the row statistics (log-sum-exp in log2
// units) and delta = sum_d dO.O, stores both for kernel B; pass 2 recomputes P, forms dS = P (dP - delta) * scale and
// accumulates dQ = dS K.  K / V blocks are double-buffered with cp.async so the next block streams in under the MMAs.
// STRIDED: a sequence is the S frames of one (b, n) of the (b, f, n) row layout (row stride rs = tokens per frame, any S);
// rows of the last block at or beyond S are zero-filled, their keys masked to -inf, and nothing of them is stored.
template <bool BF16, int HD, bool STRIDED = false>
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ o,
                                                          const uint16_t* __restrict__ d_o, uint16_t* __restrict__ dqkv,
                                                          float* __restrict__ lse, float* __restrict__ delta, int S, int heads,
                                                          float scale_log2, int rs) {
  using G = AB<HD>;
  extern __shared__ __align__(16) uint16_t sm[];
  uint16_t* sQ = sm;
  uint16_t* sDO = sm + G::TILE;
  uint16_t* sK = sm + 2 * G::TILE;      // [2] buffers
  uint16_t* sV = sm + 4 * G::TILE;      // [2] buffers
  const int qb = blockIdx.x, h = blockIdx.y, seq = blockIdx.z;
  const int D = heads * HD, ld = 3 * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t seq_row0 = STRIDED ? static_cast<size_t>(seq / rs) * S * rs + seq % rs : static_cast<size_t>(seq) * S;
  const int q0 = qb * 64;
  const int nkb = STRIDED ? (S + 63) / 64 : S / 64;
  auto load_rows = [&](uint16_t* s, const uint16_t* g, int first, int ldg, int col0) {     // sequence rows first.. first+63
    if constexpr (STRIDED) load_tile64<HD, true>(s, g, seq_row0 + static_cast<size_t>(first) * rs, ldg, col0, rs, S - first);
    else load_tile64<HD>(s, g, seq_row0 + first, ldg, col0);
  };
  zero_pads<HD>(sm, 6);
  load_rows(sQ, qkv, q0, ld, h * HD);
  load_rows(sDO, d_o, q0, D, h * HD);
  load_rows(sV, o, q0, D, h * HD);            // O block, only for delta
  load_rows(sK, qkv, 0, ld, D + h * HD);      // K block 0
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  // delta for this thread's two rows (quad lanes split the columns)
  const int r_lo = warp * 16 + (lane >> 2);
  float dl[2] = {0.f, 0.f};
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r_lo + hh * 8;
    for (int c = (lane & 3) * 2; c < HD; c += 8) {
      const float2 a = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(sDO + r * G::HDP + c));
      const float2 b = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(sV + r * G::HDP + c));
      dl[hh] += a.x * b.x + a.y * b.y;
    }
    dl[hh] += __shfl_xor_sync(0xffffffffu, dl[hh], 1);
    dl[hh] += __shfl_xor_sync(0xffffffffu, dl[hh], 2);
  }
  // ---- pass 1: row max / sum over all keys
  float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
  for (int kb = 0; kb < nkb; ++kb) {
    const uint16_t* cK = sK + (kb & 1) * G::TILE;
    if (kb + 1 < nkb) load_rows(sK + ((kb + 1) & 1) * G::TILE, qkv, (kb + 1) * 64, ld, D + h * HD);
    else {                                     // last block of pass 1: start pass 2's first K / V block (V buffer 0 held O, now consumed)
      if (nkb > 1) load_rows(sK + ((kb + 1) & 1) * G::TILE, qkv, 0, ld, D + h * HD);
    }
    cp_async_commit();
    float acc[8][4] = {};
    mm_a_tileT<BF16, HD>(acc, sQ, warp * 16, cK);
    if constexpr (STRIDED) { if (S - kb * 64 < 64) mask_keys(acc, S - kb * 64); }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float m = mx[hh];
#pragma unroll
      for (int n = 0; n < 8; ++n) m = fmaxf(m, fmaxf(acc[n][2 * hh], acc[n][2 * hh + 1]) * scale_log2);
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sacc = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n) sacc += exp2f(acc[n][2 * hh] * scale_log2 - m) + exp2f(acc[n][2 * hh + 1] * scale_log2 - m);
      sum[hh] = sum[hh] * exp2f(mx[hh] - m) + sacc;
      mx[hh] = m;
    }
    cp_async_wait<0>();
    __syncthreads();
  }
  float l2[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float t = sum[hh];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    l2[hh] = mx[hh] + log2f(t);
    if ((lane & 3) == 0 && (!STRIDED || q0 + r_lo + hh * 8 < S)) {
      const size_t idx = (static_cast<size_t>(seq) * heads + h) * S + q0 + r_lo + hh * 8;
      lse[idx] = l2[hh];
      delta[idx] = dl[hh];
    }
  }
  // ---- pass 2.  K block 0 sits in K buffer (nkb & 1) when nkb > 1 (prefetched above), else still in buffer 0.
  const int kbase = nkb > 1 ? (nkb & 1) : 0;
  load_rows(sV + kbase * G::TILE, qkv, 0, ld, 2 * D + h * HD);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  // fp16 and STRIDED keep the softmax scale out of the 16-bit dS operand and apply it to the fp32 dQ / dK at the end: dS of a
  // mean loss over a whole video is small enough that another factor hd^-1/2 pushes many values into fp16's subnormal range
  // (bf16 has the exponent range; its spatial instances keep the original order of operations)
  constexpr bool DEFER = STRIDED || !BF16;
  const float scale = DEFER ? 1.0f : scale_log2 * 0.6931471805599453f;
  float dq[G::NT][4] = {};
  for (int kb = 0; kb < nkb; ++kb) {
    const int cur = (kbase + kb) & 1, nxt = cur ^ 1;
    if (kb + 1 < nkb) {
      load_rows(sK + nxt * G::TILE, qkv, (kb + 1) * 64, ld, D + h * HD);
      load_rows(sV + nxt * G::TILE, qkv, (kb + 1) * 64, ld, 2 * D + h * HD);
    }
    cp_async_commit();
    const uint16_t* cK = sK + cur * G::TILE;
    const uint16_t* cV = sV + cur * G::TILE;
    float s_acc[8][4] = {}, p_acc[8][4] = {};
    mm_a_tileT<BF16, HD>(s_acc, sQ, warp * 16, cK);
    mm_a_tileT<BF16, HD>(p_acc, sDO, warp * 16, cV);
    if constexpr (STRIDED) { if (S - kb * 64 < 64) mask_keys(s_acc, S - kb * 64); }     // P = exp2(-inf) = 0 there
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1;
        const float pr = exp2f(s_acc[n][e] * scale_log2 - l2[hh]);
        s_acc[n][e] = pr * (p_acc[n][e] - dl[hh]) * scale;
      }
    uint32_t pds[4][4];
    acc_to_afrag<BF16>(pds, s_acc);
    mm_p_tile<BF16, HD>(dq, pds, cK);
    cp_async_wait<0>();
    __syncthreads();
  }
  if constexpr (DEFER) {
    const float sc = scale_log2 * 0.6931471805599453f;
#pragma unroll
    for (int n = 0; n < G::NT; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) dq[n][e] *= sc;
  }
  if constexpr (STRIDED) store_rows<BF16, HD, true>(dqkv, seq_row0 + static_cast<size_t>(q0) * rs, ld, h * HD, dq, warp * 16, S - q0, rs);
  else store_rows<BF16, HD>(dqkv, seq_row0 + q0, ld, h * HD, dq, warp * 16, 64);
}

// Kernel B: one CTA = 64 keys of one (sequence, head); loops over the query blocks with the statistics of kernel A.
// S^T = K Q^T so that the warp's accumulator rows are keys: P^T and dS^T are then directly the A operands of
// dV = P^T dO and dK = dS^T Q.  Q / dO blocks (and their statistics) are double-buffered with cp.async.
// STRIDED (see kernel A): queries at or beyond S are zero rows with lse = +inf and delta = 0, so their P and dS are exactly 0;
// key rows at or beyond S are zero and never stored.
template <bool BF16, int HD, bool STRIDED = false>
__global__ void __launch_bounds__(128) attn_bwd_dkv_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ d_o,
                                                           uint16_t* __restrict__ dqkv, const float* __restrict__ lse,
                                                           const float* __restrict__ delta, int S, int heads, float scale_log2, int rs) {
  using G = AB<HD>;
  extern __shared__ __align__(16) uint16_t sm[];
  uint16_t* sK = sm;
  uint16_t* sV = sm + G::TILE;
  uint16_t* sQ = sm + 2 * G::TILE;      // [2]
  uint16_t* sDO = sm + 4 * G::TILE;     // [2]
  float* sL = reinterpret_cast<float*>(sm + 6 * G::TILE);   // [2][64] lse, then [2][64] delta
  float* sD = sL + 128;
  const int kb = blockIdx.x, h = blockIdx.y, seq = blockIdx.z;
  const int D = heads * HD, ld = 3 * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t seq_row0 = STRIDED ? static_cast<size_t>(seq / rs) * S * rs + seq % rs : static_cast<size_t>(seq) * S;
  const size_t stat0 = (static_cast<size_t>(seq) * heads + h) * S;
  const int k0 = kb * 64;
  const int nqb = STRIDED ? (S + 63) / 64 : S / 64;
  auto load_rows = [&](uint16_t* s, const uint16_t* g, int first, int ldg, int col0) {
    if constexpr (STRIDED) load_tile64<HD, true>(s, g, seq_row0 + static_cast<size_t>(first) * rs, ldg, col0, rs, S - first);
    else load_tile64<HD>(s, g, seq_row0 + first, ldg, col0);
  };
  auto load_q = [&](int qb, int buf) {
    load_rows(sQ + buf * G::TILE, qkv, qb * 64, ld, h * HD);
    load_rows(sDO + buf * G::TILE, d_o, qb * 64, D, h * HD);
    if constexpr (STRIDED) {             // S need not be a multiple of 4: one float per thread
      const int t = threadIdx.x & 63, qi = qb * 64 + t;
      float* dst = (threadIdx.x < 64 ? sL : sD) + buf * 64 + t;
      if (qi < S) cp_async4(dst, (threadIdx.x < 64 ? lse : delta) + stat0 + qi);
      else *dst = threadIdx.x < 64 ? INFINITY : 0.f;
    } else {
      if (threadIdx.x < 16) cp_async16(sL + buf * 64 + threadIdx.x * 4, lse + stat0 + qb * 64 + threadIdx.x * 4);
      else if (threadIdx.x < 32) cp_async16(sD + buf * 64 + (threadIdx.x - 16) * 4, delta + stat0 + qb * 64 + (threadIdx.x - 16) * 4);
    }
  };
  zero_pads<HD>(sm, 6);
  load_rows(sK, qkv, k0, ld, D + h * HD);
  load_rows(sV, qkv, k0, ld, 2 * D + h * HD);
  load_q(0, 0);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  constexpr bool DEFER = STRIDED || !BF16;        // softmax scale applied to the fp32 dK at the end (see kernel A)
  const float scale = DEFER ? 1.0f : scale_log2 * 0.6931471805599453f;
  float dk[G::NT][4] = {}, dv[G::NT][4] = {};
  for (int qb = 0; qb < nqb; ++qb) {
    const int cur = qb & 1;
    if (qb + 1 < nqb) load_q(qb + 1, cur ^ 1);
    cp_async_commit();
    const uint16_t* cQ = sQ + cur * G::TILE;
    const uint16_t* cDO = sDO + cur * G::TILE;
    const float* cL = sL + cur * 64;
    const float* cD = sD + cur * 64;
    float s_acc[8][4] = {}, p_acc[8][4] = {};
    mm_a_tileT<BF16, HD>(s_acc, sK, warp * 16, cQ);      // [16 keys x 64 queries]
    mm_a_tileT<BF16, HD>(p_acc, sV, warp * 16, cDO);
    uint32_t pp[4][4], pds[4][4];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = n * 8 + (lane & 3) * 2 + (e & 1);
        const float pr = exp2f(s_acc[n][e] * scale_log2 - cL[qi]);
        p_acc[n][e] = pr * (p_acc[n][e] - cD[qi]) * scale;
        s_acc[n][e] = pr;
      }
    acc_to_afrag<BF16>(pp, s_acc);
    acc_to_afrag<BF16>(pds, p_acc);
    mm_p_tile<BF16, HD>(dv, pp, cDO);
    mm_p_tile<BF16, HD>(dk, pds, cQ);
    cp_async_wait<0>();
    __syncthreads();
  }
  if constexpr (DEFER) {
    const float sc = scale_log2 * 0.6931471805599453f;
#pragma unroll
    for (int n = 0; n < G::NT; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) dk[n][e] *= sc;
  }
  if constexpr (STRIDED) {
    const size_t r0 = seq_row0 + static_cast<size_t>(k0) * rs;
    store_rows<BF16, HD, true>(dqkv, r0, ld, D + h * HD, dk, warp * 16, S - k0, rs);
    store_rows<BF16, HD, true>(dqkv, r0, ld, 2 * D + h * HD, dv, warp * 16, S - k0, rs);
  } else {
    store_rows<BF16, HD>(dqkv, seq_row0 + k0, ld, D + h * HD, dk, warp * 16, 64);
    store_rows<BF16, HD>(dqkv, seq_row0 + k0, ld, 2 * D + h * HD, dv, warp * 16, 64);
  }
}

// ------------------------------------------------------------------------------------------------ cross-attention backward
// Backward of b200_cross_attention, softmax(q k^T hd^-1/2 + key_bias) v, on the tile code above.  All kv_len <= 128 keys of a
// sample sit in one or two 64-row tiles; rows at or beyond kv_len are zero-filled and their scores are -inf, so P = 0 exactly
// there.  The key bias (-10000 for a masked prompt token) is added in fp32 exactly as the forward adds it.  The softmax scale is
// applied to the fp32 dQ / dK accumulators, never to the 16-bit dS (see kernel A above).
//   xattn_bwd_dq:     one CTA = 64 query rows of one (sample, head): row statistics from q and k, delta = rowsum(dO.O), dQ = dS K;
//                     writes dQ and the statistics.
//   xattn_bwd_dkv:    one CTA = one of `chunks` contiguous ranges of a sample's query blocks, one head, every key (one warp per 16
//                     keys): an fp32 [dK | dV] partial per chunk.
//   xattn_bwd_reduce: sums the partials in chunk order and writes 16-bit dK / dV.  No atomics: reruns are bit-identical.
struct XAttnBwd {
  const uint16_t* q;        // [batch*q_rows, q_ld]
  const uint16_t* kv;       // [batch*kv_len, kv_ld], columns [k heads | v heads]
  const float* key_bias;    // [batch, 128] or nullptr
  const uint16_t* o;        // [batch*q_rows, heads*HD]
  const uint16_t* d_o;
  uint16_t* dq;             // [batch*q_rows, heads*HD]
  float* lse;               // [batch][heads][q_rows], log2 units
  float* delta;
  float* part;              // [batch][heads][chunks][128][2*HD]
  int q_rows, kv_len, q_ld, kv_ld, heads, chunks;
  float scale_log2;
};

constexpr float kXLog2e = 1.4426950408889634f;

// scores of a warp's [16 queries x 64 keys] block kt in log2 units with the key bias, -inf at keys >= kv_len
__device__ __forceinline__ void xattn_scores(float (&acc)[8][4], const float* sB, int kt, int kv_len, float scale_log2) {
  const int c0 = kt * 64 + (threadIdx.x & 3) * 2;
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + n * 8 + (e & 1);
      acc[n][e] = c < kv_len ? fmaf(sB[c], kXLog2e, acc[n][e] * scale_log2) : -INFINITY;
    }
}

template <bool BF16, int HD>
__global__ void __launch_bounds__(128) xattn_bwd_dq_kernel(const XAttnBwd p) {
  using G = AB<HD>;
  extern __shared__ __align__(16) uint16_t sm[];
  uint16_t* sQ = sm;
  uint16_t* sDO = sm + G::TILE;
  uint16_t* sO = sm + 2 * G::TILE;
  uint16_t* sK = sm + 3 * G::TILE;      // 2 tiles = keys 0..127
  uint16_t* sV = sm + 5 * G::TILE;      // 2 tiles
  float* sB = reinterpret_cast<float*>(sm + 7 * G::TILE);    // [128] key bias
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = p.heads * HD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t qrow0 = static_cast<size_t>(b) * p.q_rows + qb * 64;
  const size_t krow0 = static_cast<size_t>(b) * p.kv_len;
  const int nkt = (p.kv_len + 63) / 64;
  zero_pads<HD>(sm, 7);
  load_tile64<HD>(sQ, p.q, qrow0, p.q_ld, h * HD);
  load_tile64<HD>(sDO, p.d_o, qrow0, D, h * HD);
  load_tile64<HD>(sO, p.o, qrow0, D, h * HD);
  for (int kt = 0; kt < nkt; ++kt) {
    load_tile64<HD, true>(sK + kt * G::TILE, p.kv, krow0 + kt * 64, p.kv_ld, h * HD, 1, p.kv_len - kt * 64);
    load_tile64<HD, true>(sV + kt * G::TILE, p.kv, krow0 + kt * 64, p.kv_ld, D + h * HD, 1, p.kv_len - kt * 64);
  }
  for (int c = threadIdx.x; c < 128; c += blockDim.x) sB[c] = p.key_bias && c < p.kv_len ? p.key_bias[b * 128 + c] : 0.f;
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  const int r_lo = warp * 16 + (lane >> 2);
  float dl[2] = {0.f, 0.f};
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r_lo + hh * 8;
    for (int c = (lane & 3) * 2; c < HD; c += 8) {
      const float2 a = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(sDO + r * G::HDP + c));
      const float2 v = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(sO + r * G::HDP + c));
      dl[hh] += a.x * v.x + a.y * v.y;
    }
    dl[hh] += __shfl_xor_sync(0xffffffffu, dl[hh], 1);
    dl[hh] += __shfl_xor_sync(0xffffffffu, dl[hh], 2);
  }
  // ---- pass 1: row max / sum over the sample's keys
  float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
  for (int kt = 0; kt < nkt; ++kt) {
    float acc[8][4] = {};
    mm_a_tileT<BF16, HD>(acc, sQ, warp * 16, sK + kt * G::TILE);
    xattn_scores(acc, sB, kt, p.kv_len, p.scale_log2);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float m = mx[hh];
#pragma unroll
      for (int n = 0; n < 8; ++n) m = fmaxf(m, fmaxf(acc[n][2 * hh], acc[n][2 * hh + 1]));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sacc = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n) sacc += exp2f(acc[n][2 * hh] - m) + exp2f(acc[n][2 * hh + 1] - m);
      sum[hh] = sum[hh] * exp2f(mx[hh] - m) + sacc;
      mx[hh] = m;
    }
  }
  float l2[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float t = sum[hh];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    l2[hh] = mx[hh] + log2f(t);
    if ((lane & 3) == 0) {
      const size_t idx = (static_cast<size_t>(b) * p.heads + h) * p.q_rows + qb * 64 + r_lo + hh * 8;
      p.lse[idx] = l2[hh];
      p.delta[idx] = dl[hh];
    }
  }
  // ---- pass 2: dS = P (dP - delta), dQ = dS K
  float dq[G::NT][4] = {};
  for (int kt = 0; kt < nkt; ++kt) {
    const uint16_t* cK = sK + kt * G::TILE;
    float s_acc[8][4] = {}, p_acc[8][4] = {};
    mm_a_tileT<BF16, HD>(s_acc, sQ, warp * 16, cK);
    mm_a_tileT<BF16, HD>(p_acc, sDO, warp * 16, sV + kt * G::TILE);
    xattn_scores(s_acc, sB, kt, p.kv_len, p.scale_log2);
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1;
        s_acc[n][e] = exp2f(s_acc[n][e] - l2[hh]) * (p_acc[n][e] - dl[hh]);
      }
    uint32_t pds[4][4];
    acc_to_afrag<BF16>(pds, s_acc);
    mm_p_tile<BF16, HD>(dq, pds, cK);
  }
  const float sc = p.scale_log2 * 0.6931471805599453f;
#pragma unroll
  for (int n = 0; n < G::NT; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) dq[n][e] *= sc;
  store_rows<BF16, HD>(p.dq, qrow0, D, h * HD, dq, warp * 16, 64);
}

// launched with (kv_len + 63) / 64 * 128 threads: warp w owns keys [16w, 16w + 16)
template <bool BF16, int HD>
__global__ void __launch_bounds__(256) xattn_bwd_dkv_kernel(const XAttnBwd p) {
  using G = AB<HD>;
  extern __shared__ __align__(16) uint16_t sm[];
  uint16_t* sK = sm;                    // 2 tiles
  uint16_t* sV = sm + 2 * G::TILE;      // 2 tiles
  uint16_t* sQ = sm + 4 * G::TILE;      // [2] buffers
  uint16_t* sDO = sm + 6 * G::TILE;     // [2] buffers
  float* sL = reinterpret_cast<float*>(sm + 8 * G::TILE);   // [2][64] lse, then [2][64] delta
  float* sD = sL + 128;
  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = p.heads * HD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t qrow0 = static_cast<size_t>(b) * p.q_rows;
  const size_t krow0 = static_cast<size_t>(b) * p.kv_len;
  const size_t stat0 = (static_cast<size_t>(b) * p.heads + h) * p.q_rows;
  const int nqb = p.q_rows / 64, nkt = (p.kv_len + 63) / 64;
  const int qb0 = chunk * nqb / p.chunks, qb1 = (chunk + 1) * nqb / p.chunks;
  auto load_q = [&](int qb, int buf) {
    load_tile64<HD>(sQ + buf * G::TILE, p.q, qrow0 + qb * 64, p.q_ld, h * HD);
    load_tile64<HD>(sDO + buf * G::TILE, p.d_o, qrow0 + qb * 64, D, h * HD);
    if (threadIdx.x < 16) cp_async16(sL + buf * 64 + threadIdx.x * 4, p.lse + stat0 + qb * 64 + threadIdx.x * 4);
    else if (threadIdx.x < 32) cp_async16(sD + buf * 64 + (threadIdx.x - 16) * 4, p.delta + stat0 + qb * 64 + (threadIdx.x - 16) * 4);
  };
  zero_pads<HD>(sm, 8);
  for (int kt = 0; kt < nkt; ++kt) {
    load_tile64<HD, true>(sK + kt * G::TILE, p.kv, krow0 + kt * 64, p.kv_ld, h * HD, 1, p.kv_len - kt * 64);
    load_tile64<HD, true>(sV + kt * G::TILE, p.kv, krow0 + kt * 64, p.kv_ld, D + h * HD, 1, p.kv_len - kt * 64);
  }
  load_q(qb0, 0);
  cp_async_commit();
  // the two keys of this thread's accumulator rows: validity and bias
  bool kvalid[2];
  float kbias[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int k = warp * 16 + (lane >> 2) + hh * 8;
    kvalid[hh] = k < p.kv_len;
    kbias[hh] = p.key_bias && kvalid[hh] ? p.key_bias[b * 128 + k] : 0.f;
  }
  cp_async_wait<0>();
  __syncthreads();
  float dk[G::NT][4] = {}, dv[G::NT][4] = {};
  for (int qb = qb0; qb < qb1; ++qb) {
    const int cur = (qb - qb0) & 1;
    if (qb + 1 < qb1) load_q(qb + 1, cur ^ 1);
    cp_async_commit();
    const uint16_t* cQ = sQ + cur * G::TILE;
    const uint16_t* cDO = sDO + cur * G::TILE;
    const float* cL = sL + cur * 64;
    const float* cD = sD + cur * 64;
    float s_acc[8][4] = {}, p_acc[8][4] = {};
    mm_a_tileT<BF16, HD>(s_acc, sK, warp * 16, cQ);      // [16 keys x 64 queries]
    mm_a_tileT<BF16, HD>(p_acc, sV, warp * 16, cDO);
    uint32_t pp[4][4], pds[4][4];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1, qi = n * 8 + (lane & 3) * 2 + (e & 1);
        const float pr = kvalid[hh] ? exp2f(fmaf(kbias[hh], kXLog2e, s_acc[n][e] * p.scale_log2) - cL[qi]) : 0.f;
        p_acc[n][e] = pr * (p_acc[n][e] - cD[qi]);
        s_acc[n][e] = pr;
      }
    acc_to_afrag<BF16>(pp, s_acc);
    acc_to_afrag<BF16>(pds, p_acc);
    mm_p_tile<BF16, HD>(dv, pp, cDO);
    mm_p_tile<BF16, HD>(dk, pds, cQ);
    cp_async_wait<0>();
    __syncthreads();
  }
  const float sc = p.scale_log2 * 0.6931471805599453f;
  float* dst = p.part + ((static_cast<size_t>(b) * p.heads + h) * p.chunks + chunk) * 128 * (2 * HD);
  const int r = warp * 16 + (lane >> 2);
#pragma unroll
  for (int n = 0; n < G::NT; ++n) {
    const int c = n * 8 + (lane & 3) * 2;
    *reinterpret_cast<float2*>(dst + r * (2 * HD) + c) = make_float2(dk[n][0] * sc, dk[n][1] * sc);
    *reinterpret_cast<float2*>(dst + (r + 8) * (2 * HD) + c) = make_float2(dk[n][2] * sc, dk[n][3] * sc);
    *reinterpret_cast<float2*>(dst + r * (2 * HD) + HD + c) = make_float2(dv[n][0], dv[n][1]);
    *reinterpret_cast<float2*>(dst + (r + 8) * (2 * HD) + HD + c) = make_float2(dv[n][2], dv[n][3]);
  }
}

// dkv[(b*kv_len + j) * ld + col0 + col] = sum over chunks (in order) of the partials; col in [0, 2D): [k heads | v heads]
template <bool BF16>
__global__ void __launch_bounds__(256) xattn_bwd_reduce_kernel(const float* __restrict__ part, uint16_t* __restrict__ dkv, int ld,
                                                               int col0, int kv_len, int heads, int hd, int chunks) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y, b = blockIdx.z;
  const int D = heads * hd;
  if (col >= 2 * D) return;
  const int kind = col >= D, hh = (col - kind * D) / hd, d = col - kind * D - hh * hd;
  const float* src = part + ((static_cast<size_t>(b) * heads + hh) * chunks * 128 + j) * (2 * hd) + kind * hd + d;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += src[static_cast<size_t>(c) * 128 * (2 * hd)];
  dkv[(static_cast<size_t>(b) * kv_len + j) * ld + col0 + col] = rnd1<BF16>(s);
}

// ------------------------------------------------------------------------------------------------ attention backward (temporal)
// Sequences of F <= 16 frames at a fixed token: rows (b, f, n), f = 0..F-1 (row stride `tokens`), head_dim 64 / 72, on tensor
// cores.  ONE WARP per (b, n, head), four heads per CTA, no block-level synchronisation.  The F <= 16 frames of q, k, v, dO
// sit in a [16 x HDP] shared tile each (rows >= F zero); S = Q K^T and dP = dO V^T are one 16x16 accumulator pair, and the transposed pair (K Q^T, V dO^T) is recomputed so that P^T / dS^T come
// out directly as the A operands of dV = P^T dO and dK = dS^T Q (as in the spatial kernel B).  Row statistics go through 32
// floats of shared memory.  Results are staged in the tiles they came from and written back with 16-byte stores.
template <bool BF16, int HD>
__global__ void __launch_bounds__(128) attn_bwd_temporal_mma_kernel(const uint16_t* __restrict__ qkv, const uint16_t* __restrict__ d_o,
                                                                    uint16_t* __restrict__ dqkv, int frames, int tokens, int heads,
                                                                    float scale_log2) {
  using G = AB<HD>;
  constexpr int T16 = 16 * G::HDP;                 // elements per 16-row tile
  extern __shared__ __align__(16) uint16_t sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y * 4 + warp;
  if (h >= heads) return;
  uint16_t* sQ = sm + warp * (4 * T16 + 64);       // + 64 elements = 32 floats of statistics per warp
  uint16_t* sK = sQ + T16;
  uint16_t* sV = sK + T16;
  uint16_t* sG = sV + T16;
  float* sL = reinterpret_cast<float*>(sG + T16);  // [16] lse (log2 units), [16] delta
  const int F = frames;
  const int n = blockIdx.x % tokens, b = blockIdx.x / tokens;
  const int D = heads * HD, ld = 3 * D;
  const size_t row0 = static_cast<size_t>(b) * F * tokens + n;
  constexpr int CH = HD / 8;
  for (int i = lane; i < 4 * 16 * (G::HDP / 8); i += 32) {          // whole tiles incl. pad columns: zero where nothing is loaded
    const int which = i / (16 * (G::HDP / 8)), rem = i % (16 * (G::HDP / 8));
    const int f = rem / (G::HDP / 8), c = rem % (G::HDP / 8);
    uint16_t* dst = sQ + which * T16 + f * G::HDP + c * 8;
    if (f < F && c < CH) {
      const size_t r = row0 + static_cast<size_t>(f) * tokens;
      const uint16_t* src = which < 3 ? qkv + r * ld + which * D + h * HD + c * 8 : d_o + r * D + h * HD + c * 8;
      cp_async16(dst, src);
    } else {
      *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
    }
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();
  const int arow = (lane & 7) + ((lane >> 3) & 1) * 8, acol = (lane >> 4) * 8;      // A-fragment lane address
  const int brow = (lane & 7) + (lane >> 4) * 8, bcol = ((lane >> 3) & 1) * 8;      // B-fragment ([n][k] tile) lane address
  auto mm16 = [&](float (&acc)[2][4], const uint16_t* sA, const uint16_t* sB) {     // acc[16 x 16] = A[16 x KP] . B[16 x KP]^T
#pragma unroll
    for (int k = 0; k < G::KS; ++k) {
      uint32_t a[4], bb[4];
      ldsm_x4(a, smem_u32(sA + arow * G::HDP + k * 16 + acol));
      ldsm_x4(bb, smem_u32(sB + brow * G::HDP + k * 16 + bcol));
      mma16816<BF16>(acc[0], a, bb[0], bb[1]);
      mma16816<BF16>(acc[1], a, bb[2], bb[3]);
    }
  };
  const float scale = scale_log2 * 0.6931471805599453f;
  // fp16 keeps the softmax scale out of the 16-bit dS operands and applies it to the fp32 dQ / dK (see kernel A above)
  constexpr bool DEFER = !BF16;
  const float ds_scale = DEFER ? 1.0f : scale;
  const int c_lo = (lane & 3) * 2;                 // this thread's columns: c_lo, c_lo+1 (n-tile 0), +8 (n-tile 1)
  // ---- orientation 1: rows = queries
  float s[2][4] = {}, dp[2][4] = {};
  mm16(s, sQ, sK);
  mm16(dp, sG, sV);
  float l2[2], dl[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float m = -INFINITY;
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = t * 8 + c_lo + e;
        float& v = s[t][2 * hh + e];
        v = col < F ? v * scale_log2 : -INFINITY;
        m = fmaxf(m, v);
      }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 2; ++e) sum += exp2f(s[t][2 * hh + e] - m);
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    l2[hh] = m + log2f(sum);
    float d = 0.f;
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float pr = exp2f(s[t][2 * hh + e] - l2[hh]);      // exp2(-inf) = 0 for masked keys
        s[t][2 * hh + e] = pr;
        d += pr * dp[t][2 * hh + e];
      }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    dl[hh] = d;
    if ((lane & 3) == 0) {
      sL[(lane >> 2) + hh * 8] = l2[hh];
      sL[16 + (lane >> 2) + hh * 8] = d;
    }
  }
  uint32_t ds_a[4];
  {
    float t0[2][4];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) t0[t][e] = s[t][e] * (dp[t][e] - dl[e >> 1]) * ds_scale;
    ds_a[0] = pack2<BF16>(t0[0][0], t0[0][1]); ds_a[1] = pack2<BF16>(t0[0][2], t0[0][3]);
    ds_a[2] = pack2<BF16>(t0[1][0], t0[1][1]); ds_a[3] = pack2<BF16>(t0[1][2], t0[1][3]);
  }
  __syncwarp();
  // out[16 x HD] = A-frag(16 x 16) . tile[16 x HD]   (tile rows = contraction)
  auto mm_out = [&](float (&out)[G::NT][4], const uint32_t (&a)[4], const uint16_t* sB) {
#pragma unroll
    for (int np = 0; np < G::NT / 2; ++np) {
      uint32_t bb[4];
      ldsm_x4_t(bb, smem_u32(sB + arow * G::HDP + np * 16 + acol));
      mma16816<BF16>(out[2 * np], a, bb[0], bb[1]);
      mma16816<BF16>(out[2 * np + 1], a, bb[2], bb[3]);
    }
    if constexpr (G::NT % 2 == 1) {
      uint32_t b0, b1;
      ldsm_x2_t(b0, b1, smem_u32(sB + arow * G::HDP + (G::NT - 1) * 8));
      mma16816<BF16>(out[G::NT - 1], a, b0, b1);
    }
  };
  float dq[G::NT][4] = {};
  mm_out(dq, ds_a, sK);
  // ---- orientation 2: rows = keys
  float st[2][4] = {}, dpt[2][4] = {};
  mm16(st, sK, sQ);
  mm16(dpt, sV, sG);
  uint32_t pt_a[4], dst_a[4];
  {
    float pv[2][4], dv_[2][4];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = t * 8 + c_lo + (e & 1);
        const float pr = exp2f(st[t][e] * scale_log2 - sL[qi]);
        pv[t][e] = pr;
        dv_[t][e] = pr * (dpt[t][e] - sL[16 + qi]) * ds_scale;
      }
    pt_a[0] = pack2<BF16>(pv[0][0], pv[0][1]); pt_a[1] = pack2<BF16>(pv[0][2], pv[0][3]);
    pt_a[2] = pack2<BF16>(pv[1][0], pv[1][1]); pt_a[3] = pack2<BF16>(pv[1][2], pv[1][3]);
    dst_a[0] = pack2<BF16>(dv_[0][0], dv_[0][1]); dst_a[1] = pack2<BF16>(dv_[0][2], dv_[0][3]);
    dst_a[2] = pack2<BF16>(dv_[1][0], dv_[1][1]); dst_a[3] = pack2<BF16>(dv_[1][2], dv_[1][3]);
  }
  float dk[G::NT][4] = {}, dv[G::NT][4] = {};
  mm_out(dv, pt_a, sG);
  mm_out(dk, dst_a, sQ);
  if constexpr (DEFER) {
#pragma unroll
    for (int nn = 0; nn < G::NT; ++nn)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dq[nn][e] *= scale;
        dk[nn][e] *= scale;
      }
  }
  __syncwarp();
  // ---- stage the three results in the q / k / v tiles, then 16-byte stores
  auto stage = [&](uint16_t* tile, const float (&acc)[G::NT][4]) {
    const int r = lane >> 2;
#pragma unroll
    for (int nn = 0; nn < G::NT; ++nn) {
      *reinterpret_cast<uint32_t*>(tile + r * G::HDP + nn * 8 + c_lo) = pack2<BF16>(acc[nn][0], acc[nn][1]);
      *reinterpret_cast<uint32_t*>(tile + (r + 8) * G::HDP + nn * 8 + c_lo) = pack2<BF16>(acc[nn][2], acc[nn][3]);
    }
  };
  stage(sQ, dq);
  stage(sK, dk);
  stage(sV, dv);
  __syncwarp();
  for (int i = lane; i < 3 * F * CH; i += 32) {
    const int which = i / (F * CH), rem = i % (F * CH);
    const int f = rem / CH, c = rem % CH;
    const size_t r = row0 + static_cast<size_t>(f) * tokens;
    *reinterpret_cast<uint4*>(dqkv + r * ld + which * D + h * HD + c * 8) =
        *reinterpret_cast<const uint4*>(sQ + which * T16 + f * G::HDP + c * 8);
  }
}

// ------------------------------------------------------------------------------------------------ adaLN gradients
// dW[n, k] = sum_b dmod[b, n] * sc[b, k]   (B <= 8 rows; pure write bandwidth: the gradient buffer itself)
template <bool BF16>
__global__ void __launch_bounds__(256) ada_outer_kernel(const float* __restrict__ dmod, long long dmod_bs, const uint16_t* __restrict__ sc,
                                                        float* __restrict__ dW, int batch, int NA, int dim) {
  extern __shared__ float s_sc[];   // [batch][dim]
  for (int i = threadIdx.x; i < batch * dim; i += blockDim.x) s_sc[i] = cvt1<BF16>(sc[i]);
  __syncthreads();
  const int nv = dim >> 2;
  for (int n = blockIdx.x; n < NA; n += gridDim.x) {
    float dm[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) dm[b] = b < batch ? dmod[b * dmod_bs + n] : 0.f;
    float4* row = reinterpret_cast<float4*>(dW + static_cast<size_t>(n) * dim);
    for (int c = threadIdx.x; c < nv; c += blockDim.x) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b < batch) {
          const float4 s = reinterpret_cast<const float4*>(s_sc + b * dim)[c];
          a.x = fmaf(dm[b], s.x, a.x); a.y = fmaf(dm[b], s.y, a.y); a.z = fmaf(dm[b], s.z, a.z); a.w = fmaf(dm[b], s.w, a.w);
        }
      }
      row[c] = a;
    }
  }
}

// dsc[b, k] += sum_{n in slab} dmod[b, n] * W[n, k]     (W 16-bit [NA, dim]; one read of the adaLN weights)
template <bool BF16>
__global__ void __launch_bounds__(256) ada_dsc_kernel(const float* __restrict__ dmod, long long dmod_bs, const uint16_t* __restrict__ w,
                                                      float* __restrict__ dsc, int batch, int NA, int dim, int slab) {
  const int n0 = blockIdx.x * slab;
  const int n1 = min(NA, n0 + slab);
  const int half = dim >> 1;
  for (int c = threadIdx.x; c < half; c += blockDim.x) {
    float acc[8][2] = {};
    for (int n = n0; n < n1; ++n) {
      const float2 wv = unpack2<BF16>(*reinterpret_cast<const uint32_t*>(w + static_cast<size_t>(n) * dim + 2 * c));
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b < batch) {
          const float d = __ldg(dmod + b * dmod_bs + n);
          acc[b][0] = fmaf(d, wv.x, acc[b][0]);
          acc[b][1] = fmaf(d, wv.y, acc[b][1]);
        }
      }
    }
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      if (b < batch) {
        atomicAdd(dsc + static_cast<size_t>(b) * dim + 2 * c, acc[b][0]);
        atomicAdd(dsc + static_cast<size_t>(b) * dim + 2 * c + 1, acc[b][1]);
      }
    }
  }
}

inline int grid_for(long long items, int per_block, int cap) {
  long long b = (items + per_block - 1) / per_block;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace

// ================================================================================================ launchers
#define ALIGNED16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

int launch_transpose16(const void* in, void* out, int rows, int cols, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && cols > 0 && rows % 2 == 0 && cols % 2 == 0, B200_ERR_SHAPE, "transpose16: %d x %d must be even", rows, cols);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(in) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0, B200_ERR_ALIGN,
               "transpose16: pointers must be 4-byte aligned");
  dim3 grid((cols + 63) / 64, (rows + 63) / 64);
  transpose16_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(in), static_cast<uint16_t*>(out), rows, cols);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_multi_cast(const void* table, int n_entries, long long total_chunks, int bf16, cudaStream_t stream) {
  B200_REQUIRE(table != nullptr && n_entries > 0 && total_chunks > 0, B200_ERR_SHAPE, "multi_cast: empty table");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(table) & 7) == 0, B200_ERR_ALIGN, "multi_cast: table must be 8-byte aligned");
  const int blocks = static_cast<int>(total_chunks < 132 * 8 ? total_chunks : 132 * 8);
  const MultiCastEntry* tab = static_cast<const MultiCastEntry*>(table);
  if (bf16) multi_cast_kernel<true><<<blocks, 256, 0, stream>>>(tab, n_entries, total_chunks);
  else multi_cast_kernel<false><<<blocks, 256, 0, stream>>>(tab, n_entries, total_chunks);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_multi_tensor(const void* table, int n_entries, long long total_chunks, int op, float a, float b, const float* scalar,
                        double* accum, cudaStream_t stream) {
  B200_REQUIRE(table != nullptr && n_entries > 0 && total_chunks > 0, B200_ERR_SHAPE, "multi_tensor: empty table");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(table) & 7) == 0, B200_ERR_ALIGN, "multi_tensor: table must be 8-byte aligned");
  B200_REQUIRE(op == MT_SUMSQ || op == MT_SCALE || op == MT_AXPBY, B200_ERR_UNSUPPORTED, "multi_tensor: op %d unknown", op);
  B200_REQUIRE(op != MT_SUMSQ || (accum != nullptr && (reinterpret_cast<uintptr_t>(accum) & 7) == 0), B200_ERR_ALIGN, "multi_tensor: accum missing");
  B200_REQUIRE(op != MT_SCALE || scalar != nullptr, B200_ERR_SHAPE, "multi_tensor: scalar missing");
  const int blocks = static_cast<int>(total_chunks < 132 * 8 ? total_chunks : 132 * 8);
  const MultiTensorEntry* tab = static_cast<const MultiTensorEntry*>(table);
  if (op == MT_SUMSQ) multi_tensor_kernel<MT_SUMSQ><<<blocks, 256, 0, stream>>>(tab, n_entries, total_chunks, a, b, scalar, accum);
  else if (op == MT_SCALE) multi_tensor_kernel<MT_SCALE><<<blocks, 256, 0, stream>>>(tab, n_entries, total_chunks, a, b, scalar, accum);
  else multi_tensor_kernel<MT_AXPBY><<<blocks, 256, 0, stream>>>(tab, n_entries, total_chunks, a, b, scalar, accum);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_gate_residual(const float* x, const void* m16, const float* gate, long long gate_bs, int rows_per_batch,
                         const float* row_add, int tokens, int frames, float* out, int rows, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && rows_per_batch > 0 && gate_bs % 4 == 0, B200_ERR_SHAPE, "gate_residual: bad shape");
  B200_REQUIRE(row_add == nullptr || (tokens > 0 && frames > 0), B200_ERR_SHAPE, "gate_residual: row_add needs tokens and frames");
  B200_REQUIRE(ALIGNED16(x) && ALIGNED16(gate) && ALIGNED16(out) && (reinterpret_cast<uintptr_t>(m16) & 7) == 0 &&
                   (row_add == nullptr || ALIGNED16(row_add)), B200_ERR_ALIGN, "gate_residual: misaligned pointer");
  const long long total = static_cast<long long>(rows) * (dim / 4);
  const int blocks = grid_for(total, 256, 132 * 16);
  const uint16_t* m = static_cast<const uint16_t*>(m16);
  if (bf16) gate_residual_kernel<true><<<blocks, 256, 0, stream>>>(x, m, gate, gate_bs, rows_per_batch, row_add, tokens, frames, out, rows, dim);
  else gate_residual_kernel<false><<<blocks, 256, 0, stream>>>(x, m, gate, gate_bs, rows_per_batch, row_add, tokens, frames, out, rows, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

// Row-lanes of the column-sum passes (gridDim.y = rows / rows per lane) and the warps of ln_modulate_bwd
constexpr int kGeluBwdRowsPerLane = 32, kGateBwdRowsPerLane = 32, kColsumRowsPerLane = 64;
constexpr int kLnbWarps = 4, kLnbRowsPerWarp = 8;

int launch_gelu_bwd(const void* da16, const void* u16, void* du16, float* dbias, int rows, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 8 == 0, B200_ERR_SHAPE, "gelu_bwd: dim %d must be a multiple of 8", dim);
  B200_REQUIRE(ALIGNED16(da16) && ALIGNED16(u16) && ALIGNED16(du16), B200_ERR_ALIGN, "gelu_bwd: pointers must be 16-byte aligned");
  dim3 grid((dim / 8 + 127) / 128, (rows + kGeluBwdRowsPerLane - 1) / kGeluBwdRowsPerLane);
  const uint16_t *a = static_cast<const uint16_t*>(da16), *u = static_cast<const uint16_t*>(u16);
  if (bf16) gelu_bwd_kernel<true><<<grid, 128, 0, stream>>>(a, u, static_cast<uint16_t*>(du16), dbias, rows, dim);
  else gelu_bwd_kernel<false><<<grid, 128, 0, stream>>>(a, u, static_cast<uint16_t*>(du16), dbias, rows, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_gate_bwd(const float* dx, const void* m16, const float* gate, long long gate_bs, int rows_per_batch, void* dm16,
                    float* dgate, long long dgate_bs, float* dbias, int rows, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && rows_per_batch > 0 && gate_bs % 4 == 0, B200_ERR_SHAPE, "gate_bwd: bad shape");
  B200_REQUIRE(ALIGNED16(dx) && ALIGNED16(gate) && (reinterpret_cast<uintptr_t>(m16) & 7) == 0 && (reinterpret_cast<uintptr_t>(dm16) & 7) == 0,
               B200_ERR_ALIGN, "gate_bwd: misaligned pointer");
  const int batch = (rows + rows_per_batch - 1) / rows_per_batch;
  dim3 grid((dim / 4 + 127) / 128, (rows_per_batch + kGateBwdRowsPerLane - 1) / kGateBwdRowsPerLane, batch);
  const uint16_t* m = static_cast<const uint16_t*>(m16);
  if (bf16) gate_bwd_kernel<true><<<grid, 128, 0, stream>>>(dx, m, gate, gate_bs, rows_per_batch, static_cast<uint16_t*>(dm16), dgate, dgate_bs, dbias, rows, dim);
  else gate_bwd_kernel<false><<<grid, 128, 0, stream>>>(dx, m, gate, gate_bs, rows_per_batch, static_cast<uint16_t*>(dm16), dgate, dgate_bs, dbias, rows, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_colsum(const void* a, int dtype, float* out, int rows, int dim, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && dtype >= 0 && dtype <= 2, B200_ERR_SHAPE, "colsum: bad shape / dtype");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(a) & (dtype == 0 ? 15 : 7)) == 0, B200_ERR_ALIGN, "colsum: misaligned input");
  dim3 grid((dim / 4 + 127) / 128, (rows + kColsumRowsPerLane - 1) / kColsumRowsPerLane);
  if (dtype == 0) colsum_kernel<0><<<grid, 128, 0, stream>>>(a, out, rows, dim);
  else if (dtype == 1) colsum_kernel<1><<<grid, 128, 0, stream>>>(a, out, rows, dim);
  else colsum_kernel<2><<<grid, 128, 0, stream>>>(a, out, rows, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

template <bool BF16, int NV>
static int lnb_launch(cudaStream_t stream, const uint16_t* dh, const float* x, const float* scale, long long mod_bs, int rpb, float* dx,
                      float* dshift, float* dscale, long long dmod_bs, int rows, int dim) {
  // [warps][2][dim] fp32 column sums: at most 48 KiB for dim <= 1536, within the default dynamic shared memory limit
  const size_t smem = static_cast<size_t>(dim) * 2 * kLnbWarps * sizeof(float);
  const int batch = (rows + rpb - 1) / rpb;
  dim3 grid((rpb + kLnbWarps * kLnbRowsPerWarp - 1) / (kLnbWarps * kLnbRowsPerWarp), batch);
  ln_modulate_bwd_kernel<BF16, NV><<<grid, kLnbWarps * 32, smem, stream>>>(dh, x, scale, mod_bs, rpb, dx, dshift, dscale, dmod_bs, rows, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_ln_modulate_bwd(const void* dh16, const float* x, const float* scale, long long mod_bs, int rows_per_batch, float* dx,
                           float* dshift, float* dscale, long long dmod_bs, int rows, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && dim <= 12 * 128, B200_ERR_SHAPE, "ln_modulate_bwd: dim %d must be a multiple of 4 and <= 1536", dim);
  B200_REQUIRE(rows_per_batch > 0 && mod_bs % 4 == 0, B200_ERR_SHAPE, "ln_modulate_bwd: bad batch geometry");
  B200_REQUIRE(ALIGNED16(x) && ALIGNED16(scale) && ALIGNED16(dx) && (reinterpret_cast<uintptr_t>(dh16) & 7) == 0, B200_ERR_ALIGN,
               "ln_modulate_bwd: misaligned pointer");
  const int nvmax = (dim / 4 + 31) / 32;
  const uint16_t* dh = static_cast<const uint16_t*>(dh16);
#define LNB(BF, NVV) return lnb_launch<BF, NVV>(stream, dh, x, scale, mod_bs, rows_per_batch, dx, dshift, dscale, dmod_bs, rows, dim)
  if (bf16) {
    if (nvmax <= 3) LNB(true, 3);
    if (nvmax <= 6) LNB(true, 6);
    if (nvmax <= 9) LNB(true, 9);
    LNB(true, 12);
  }
  if (nvmax <= 3) LNB(false, 3);
  if (nvmax <= 6) LNB(false, 6);
  if (nvmax <= 9) LNB(false, 9);
  LNB(false, 12);
#undef LNB
}

// Spatial sequences (STRIDED = false): nseq = batch * frames sequences of S = tokens consecutive rows, S % 64 == 0.
// Temporal sequences (STRIDED = true): nseq = batch * tokens sequences of S = frames rows at stride rs = tokens.
template <bool BF16, int HD, bool STRIDED = false>
static int attn_bwd_two_pass(const uint16_t* qkv, const uint16_t* o, const uint16_t* d_o, uint16_t* dqkv, float* lse, float* delta,
                            int nseq, int S, int heads, cudaStream_t stream, int rs = 1) {
  using G = AB<HD>;
  auto ka = attn_bwd_dq_kernel<BF16, HD, STRIDED>;
  auto kb = attn_bwd_dkv_kernel<BF16, HD, STRIDED>;
  const size_t smem_a = static_cast<size_t>(6) * G::TILE * 2;
  const size_t smem_b = smem_a + 256 * sizeof(float);
  B200_SET_SMEM_ONCE(ka, static_cast<int>(smem_a));
  B200_SET_SMEM_ONCE(kb, static_cast<int>(smem_b));
  const float scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(HD));
  dim3 grid((S + 63) / 64, heads, nseq);
  ka<<<grid, 128, smem_a, stream>>>(qkv, o, d_o, dqkv, lse, delta, S, heads, scale_log2, rs);
  B200_CHECK_CUDA(cudaGetLastError());
  kb<<<grid, 128, smem_b, stream>>>(qkv, d_o, dqkv, lse, delta, S, heads, scale_log2, rs);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_attention_bwd(const void* qkv, const void* o, const void* d_o, void* dqkv, float* stats, int batch, int frames, int tokens,
                         int heads, int head_dim, int bf16, int temporal, cudaStream_t stream) {
  B200_REQUIRE(batch > 0 && frames > 0 && tokens > 0 && heads > 0, B200_ERR_SHAPE, "attention_bwd: bad shape");
  B200_REQUIRE(ALIGNED16(qkv) && ALIGNED16(o) && ALIGNED16(d_o) && ALIGNED16(dqkv), B200_ERR_ALIGN, "attention_bwd: pointers must be 16-byte aligned");
  const uint16_t *q = static_cast<const uint16_t*>(qkv), *oo = static_cast<const uint16_t*>(o), *g = static_cast<const uint16_t*>(d_o);
  uint16_t* dq = static_cast<uint16_t*>(dqkv);
  if (temporal && frames > 16) {                  // 17..128 frames: the two-kernel tensor-core backward over strided rows
    B200_REQUIRE(frames <= 128 && (head_dim == 64 || head_dim == 72), B200_ERR_UNSUPPORTED,
                 "attention_bwd: temporal sequences of 17..128 frames need head_dim 64 or 72 (got %d frames, head_dim %d)", frames, head_dim);
    B200_REQUIRE(stats != nullptr && ALIGNED16(stats), B200_ERR_ALIGN, "attention_bwd: stats workspace missing");
    const int nseq = batch * tokens;
    B200_REQUIRE(nseq <= 65535 && heads <= 65535, B200_ERR_UNSUPPORTED, "attention_bwd: batch * tokens = %d sequences exceed the grid's z extent", nseq);
    float* lse = stats;
    float* delta = stats + static_cast<size_t>(nseq) * heads * frames;
    if (head_dim == 72) {
      if (bf16) return attn_bwd_two_pass<true, 72, true>(q, oo, g, dq, lse, delta, nseq, frames, heads, stream, tokens);
      return attn_bwd_two_pass<false, 72, true>(q, oo, g, dq, lse, delta, nseq, frames, heads, stream, tokens);
    }
    if (bf16) return attn_bwd_two_pass<true, 64, true>(q, oo, g, dq, lse, delta, nseq, frames, heads, stream, tokens);
    return attn_bwd_two_pass<false, 64, true>(q, oo, g, dq, lse, delta, nseq, frames, heads, stream, tokens);
  }
  if (!temporal && tokens <= 16) {
    // Spatial sequences of N <= 16 tokens (patch 8 at 256^2, small grids): N consecutive rows per (b, f) are exactly the
    // temporal kernel's input with batch' = batch * frames, frames' = N and tokens' = 1 -- one sequence of <= 16 rows per warp
    // at row stride 1.
    batch *= frames;
    frames = tokens;
    tokens = 1;
    temporal = 1;
  }
  if (temporal) {                                 // 1..16 frames: one warp per (b, n, head) on tensor cores
    B200_REQUIRE(head_dim == 64 || head_dim == 72, B200_ERR_UNSUPPORTED,
                 "attention_bwd: temporal sequences of 1..16 frames need head_dim 64 or 72 (got %d frames, head_dim %d)", frames, head_dim);
    const float scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(head_dim));
    dim3 grid_w(batch * tokens, (heads + 3) / 4);
    const int hdp = (head_dim + 15) / 16 * 16 + 8;
    const size_t smem_w = static_cast<size_t>(4) * (4 * 16 * hdp + 64) * 2;
#define TMMA(BF, HDV)                                                                                                          \
    do {                                                                                                                        \
      auto kern = attn_bwd_temporal_mma_kernel<BF, HDV>;                                                                        \
      B200_SET_SMEM_ONCE(kern, static_cast<int>(smem_w));                                                                       \
      kern<<<grid_w, 128, smem_w, stream>>>(q, g, dq, frames, tokens, heads, scale_log2);                                       \
    } while (0)
    if (head_dim == 72) { if (bf16) TMMA(true, 72); else TMMA(false, 72); }
    else { if (bf16) TMMA(true, 64); else TMMA(false, 64); }
#undef TMMA
    B200_CHECK_CUDA(cudaGetLastError());
    return B200_OK;
  }
  B200_REQUIRE(tokens % 64 == 0, B200_ERR_UNSUPPORTED, "attention_bwd: tokens per frame (%d) must be a multiple of 64", tokens);
  B200_REQUIRE(head_dim == 64 || head_dim == 72, B200_ERR_UNSUPPORTED, "attention_bwd: head_dim %d not built (64, 72)", head_dim);
  B200_REQUIRE(stats != nullptr && ALIGNED16(stats), B200_ERR_ALIGN, "attention_bwd: stats workspace missing");
  const int nseq = batch * frames;
  B200_REQUIRE(nseq <= 65535 && heads <= 65535, B200_ERR_UNSUPPORTED, "attention_bwd: batch * frames = %d sequences exceed the grid's z extent", nseq);
  float* lse = stats;
  float* delta = stats + static_cast<size_t>(nseq) * heads * tokens;
  if (head_dim == 72) {
    if (bf16) return attn_bwd_two_pass<true, 72>(q, oo, g, dq, lse, delta, nseq, tokens, heads, stream);
    return attn_bwd_two_pass<false, 72>(q, oo, g, dq, lse, delta, nseq, tokens, heads, stream);
  }
  if (bf16) return attn_bwd_two_pass<true, 64>(q, oo, g, dq, lse, delta, nseq, tokens, heads, stream);
  return attn_bwd_two_pass<false, 64>(q, oo, g, dq, lse, delta, nseq, tokens, heads, stream);
}

// Query chunks per (sample, head) of the dK/dV reduction: at least 4 query blocks (256 rows) per chunk, at most 16 chunks.  A
// function of the shape alone, so the summation order never changes between runs.
static int xattn_chunks(int q_rows_per_batch) {
  const int c = q_rows_per_batch / 64 / 4;
  return c < 1 ? 1 : (c > 16 ? 16 : c);
}

static int xattn_bwd_check(int batch, int q_rows_per_batch, int kv_len, int heads, int head_dim) {
  B200_REQUIRE(batch > 0 && q_rows_per_batch > 0 && heads > 0, B200_ERR_SHAPE, "cross_attention_bwd: bad shape");
  B200_REQUIRE(head_dim == 64 || head_dim == 72, B200_ERR_UNSUPPORTED, "cross_attention_bwd: head_dim %d not built (64, 72)", head_dim);
  B200_REQUIRE(kv_len >= 1 && kv_len <= 128, B200_ERR_UNSUPPORTED, "cross_attention_bwd: %d keys per sample (1..128 built)", kv_len);
  B200_REQUIRE(q_rows_per_batch % 128 == 0, B200_ERR_UNSUPPORTED,
               "cross_attention_bwd: query rows per sample %d must be a multiple of 128", q_rows_per_batch);
  B200_REQUIRE(batch <= 65535 && heads <= 65535, B200_ERR_UNSUPPORTED, "cross_attention_bwd: batch / heads exceed the grid");
  return B200_OK;
}

static size_t xattn_stats_bytes(int batch, int q_rows_per_batch, int heads) {
  return (static_cast<size_t>(2) * batch * heads * q_rows_per_batch * sizeof(float) + 255) / 256 * 256;
}

size_t cross_attention_bwd_workspace_bytes(int batch, int q_rows_per_batch, int kv_len, int heads, int head_dim) {
  if (xattn_bwd_check(batch, q_rows_per_batch, kv_len, heads, head_dim) != B200_OK) return 0;
  const size_t part = static_cast<size_t>(batch) * heads * xattn_chunks(q_rows_per_batch) * 128 * 2 * head_dim * sizeof(float);
  return xattn_stats_bytes(batch, q_rows_per_batch, heads) + part;
}

template <bool BF16, int HD>
static int xattn_bwd_launch(const XAttnBwd& p, int batch, uint16_t* dkv, int dkv_ld, int dkv_col0, cudaStream_t stream) {
  using G = AB<HD>;
  auto ka = xattn_bwd_dq_kernel<BF16, HD>;
  auto kb = xattn_bwd_dkv_kernel<BF16, HD>;
  const size_t smem_a = static_cast<size_t>(7) * G::TILE * 2 + 128 * sizeof(float);
  const size_t smem_b = static_cast<size_t>(8) * G::TILE * 2 + 256 * sizeof(float);
  B200_SET_SMEM_ONCE(ka, static_cast<int>(smem_a));
  B200_SET_SMEM_ONCE(kb, static_cast<int>(smem_b));
  ka<<<dim3(p.q_rows / 64, p.heads, batch), 128, smem_a, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  kb<<<dim3(p.chunks, p.heads, batch), (p.kv_len + 63) / 64 * 128, smem_b, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  const int D2 = 2 * p.heads * HD;
  xattn_bwd_reduce_kernel<BF16><<<dim3((D2 + 255) / 256, p.kv_len, batch), 256, 0, stream>>>(p.part, dkv, dkv_ld, dkv_col0, p.kv_len,
                                                                                           p.heads, HD, p.chunks);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_cross_attention_bwd(const CrossAttnBwdArgs& a, cudaStream_t stream) {
  B200_TRY(xattn_bwd_check(a.batch, a.q_rows_per_batch, a.kv_len, a.heads, a.head_dim));
  const int D = a.heads * a.head_dim;
  B200_REQUIRE(a.q_row_stride >= D && a.kv_row_stride >= 2 * D && a.q_row_stride % 8 == 0 && a.kv_row_stride % 8 == 0, B200_ERR_SHAPE,
               "cross_attention_bwd: bad q / kv row strides");
  B200_REQUIRE(a.dkv_col0 >= 0 && a.dkv_row_stride >= a.dkv_col0 + 2 * D, B200_ERR_SHAPE, "cross_attention_bwd: bad dkv column window");
  B200_REQUIRE(ALIGNED16(a.q) && ALIGNED16(a.kv) && ALIGNED16(a.o) && ALIGNED16(a.d_o) && ALIGNED16(a.dq) && ALIGNED16(a.workspace),
               B200_ERR_ALIGN, "cross_attention_bwd: q / kv / o / do / dq / workspace must be 16-byte aligned");
  B200_REQUIRE(a.dkv != nullptr, B200_ERR_SHAPE, "cross_attention_bwd: dkv missing");
  const size_t need = cross_attention_bwd_workspace_bytes(a.batch, a.q_rows_per_batch, a.kv_len, a.heads, a.head_dim);
  B200_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= need, B200_ERR_WORKSPACE,
               "cross_attention_bwd: workspace too small: need %zu bytes, got %zu", need, a.workspace_bytes);
  XAttnBwd p{};
  p.q = static_cast<const uint16_t*>(a.q);
  p.kv = static_cast<const uint16_t*>(a.kv);
  p.key_bias = a.key_bias;
  p.o = static_cast<const uint16_t*>(a.o);
  p.d_o = static_cast<const uint16_t*>(a.d_o);
  p.dq = static_cast<uint16_t*>(a.dq);
  const size_t nstat = static_cast<size_t>(a.batch) * a.heads * a.q_rows_per_batch;
  p.lse = static_cast<float*>(a.workspace);
  p.delta = p.lse + nstat;
  p.part = reinterpret_cast<float*>(static_cast<uint8_t*>(a.workspace) + xattn_stats_bytes(a.batch, a.q_rows_per_batch, a.heads));
  p.q_rows = a.q_rows_per_batch;
  p.kv_len = a.kv_len;
  p.q_ld = a.q_row_stride;
  p.kv_ld = a.kv_row_stride;
  p.heads = a.heads;
  p.chunks = xattn_chunks(a.q_rows_per_batch);
  p.scale_log2 = kXLog2e / sqrtf(static_cast<float>(a.head_dim));
  uint16_t* dkv = static_cast<uint16_t*>(a.dkv);
  if (a.head_dim == 72) {
    if (a.bf16) return xattn_bwd_launch<true, 72>(p, a.batch, dkv, a.dkv_row_stride, a.dkv_col0, stream);
    return xattn_bwd_launch<false, 72>(p, a.batch, dkv, a.dkv_row_stride, a.dkv_col0, stream);
  }
  if (a.bf16) return xattn_bwd_launch<true, 64>(p, a.batch, dkv, a.dkv_row_stride, a.dkv_col0, stream);
  return xattn_bwd_launch<false, 64>(p, a.batch, dkv, a.dkv_row_stride, a.dkv_col0, stream);
}

int launch_ada_outer(const float* dmod, long long dmod_bs, const void* sc16, float* dW, int batch, int NA, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(batch > 0 && batch <= 8 && NA > 0 && dim > 0 && dim % 4 == 0, B200_ERR_SHAPE, "ada_outer: batch <= 8, dim %% 4 == 0");
  B200_REQUIRE(ALIGNED16(dW), B200_ERR_ALIGN, "ada_outer: dW must be 16-byte aligned");
  const size_t smem = static_cast<size_t>(batch) * dim * sizeof(float);
  B200_REQUIRE(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "ada_outer: batch * dim too large for the staging buffer");
  const int blocks = NA < 132 * 8 ? NA : 132 * 8;
  if (bf16) ada_outer_kernel<true><<<blocks, 256, smem, stream>>>(dmod, dmod_bs, static_cast<const uint16_t*>(sc16), dW, batch, NA, dim);
  else ada_outer_kernel<false><<<blocks, 256, smem, stream>>>(dmod, dmod_bs, static_cast<const uint16_t*>(sc16), dW, batch, NA, dim);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_ada_dsc(const float* dmod, long long dmod_bs, const void* w16, float* dsc, int batch, int NA, int dim, int bf16, cudaStream_t stream) {
  B200_REQUIRE(batch > 0 && batch <= 8 && NA > 0 && dim > 0 && dim % 2 == 0, B200_ERR_SHAPE, "ada_dsc: batch <= 8, dim even");
  B200_CHECK_CUDA(cudaMemsetAsync(dsc, 0, sizeof(float) * batch * dim, stream));
  const int slab = 128;
  const int blocks = (NA + slab - 1) / slab;
  if (bf16) ada_dsc_kernel<true><<<blocks, 256, 0, stream>>>(dmod, dmod_bs, static_cast<const uint16_t*>(w16), dsc, batch, NA, dim, slab);
  else ada_dsc_kernel<false><<<blocks, 256, 0, stream>>>(dmod, dmod_bs, static_cast<const uint16_t*>(w16), dsc, batch, NA, dim, slab);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

}  // namespace b200
