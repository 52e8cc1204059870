// AutoencoderKL.decode (diffusers 0.24.0 `Decoder`, called at reference sample/sample.py:114, sample_ddp.py:167,
// pipeline_latte.py:758,771) as a chain of TMA implicit-GEMM convolutions on the wgmma GEMM kernel plus the
// memory-bound passes between them.  Activations are NHWC 16-bit so a pixel's channels are the GEMM K dimension.
//   3x3 conv          -> launch_gemm in conv mode: 9 taps x (Cin/64) k-blocks, the A tile of a tap is the output tile's
//                        pixel patch shifted by (dx, dy), borders zero-filled by TMA; bias (+ shortcut) in the epilogue
//   GroupNorm(32)+SiLU -> gn_stats (fp32 partial sums of x - pivot, fp64 combine) + gn_apply (one read, one write)
//   nearest 2x upsample, 1x1 convs (plain GEMM), mid-block attention (three GEMMs + a row softmax), tiny first/last layers.
// PARITY UNPINNED: diffusers is not available offline; the CPU truth is oracle/vae_oracle.py's restatement.
#include "common.h"
#include "ptx.cuh"

namespace b200 {
namespace {


// ---------------------------------------------------------------------------------- GroupNorm statistics
// x: [n_img, hw, C] 16-bit.  One block handles `rows_per_block` pixels of one image; thread t owns 8 channels
// (c8 = t % (C/8)); per-group partial (sum, sumsq) are reduced in smem and added to part[img][group][2] (fp32 atomics:
// <= a few hundred adds per slot).  The sums are of x - pivot, pivot = the group's first value in the image (gn_pivot):
// with |mean| >> std, E[x^2] - mean^2 of the raw values cancels most of the fp32 bits of the variance (at mean = 64 std
// over 65536 pixels the fp16 outputs were off by up to 7 roundings); the shifted sums keep them, and a constant group
// sums to exactly zero.
template <bool BF16>
__device__ __forceinline__ float gn_pivot(const uint16_t* x, int img, int hw, int C, int group, int cpg) {
  return unpack2<BF16>(static_cast<uint32_t>(x[static_cast<size_t>(img) * hw * C + group * cpg])).x;
}

template <bool BF16>
__global__ void __launch_bounds__(256) gn_stats_kernel(const uint16_t* __restrict__ x, float* __restrict__ part, int hw, int C,
                                                       int groups, int rows_per_block) {
  extern __shared__ float s_acc[];  // [groups][2]
  const int img = blockIdx.y;
  const int c8n = C / 8;
  const int cpg = C / groups;           // channels per group (multiple of 8 or a divisor of 8)
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  const int c8 = threadIdx.x % c8n;
  const int rlane = threadIdx.x / c8n;
  const int rstep = blockDim.x / c8n;
  const int row0 = blockIdx.x * rows_per_block;
  // pivots of this thread's channels 0-3 and 4-7 (two groups when cpg == 4)
  const float p_lo = gn_pivot<BF16>(x, img, hw, C, (c8 * 8) / cpg, cpg);
  const float p_hi = cpg == 4 ? gn_pivot<BF16>(x, img, hw, C, (c8 * 8) / cpg + 1, cpg) : p_lo;
  float s = 0.f, q = 0.f;
  float s2 = 0.f, q2 = 0.f;             // second group when 8 channels straddle two groups (cpg == 4)
  for (int r = row0 + rlane; r < row0 + rows_per_block && r < hw; r += rstep) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + (static_cast<size_t>(img) * hw + r) * C + c8 * 8);
    float2 a = unpack2<BF16>(v.x), b = unpack2<BF16>(v.y), c = unpack2<BF16>(v.z), d = unpack2<BF16>(v.w);
    a.x -= p_lo; a.y -= p_lo; b.x -= p_lo; b.y -= p_lo;
    c.x -= p_hi; c.y -= p_hi; d.x -= p_hi; d.y -= p_hi;
    if (cpg >= 8) {
      s += (a.x + a.y) + (b.x + b.y) + (c.x + c.y) + (d.x + d.y);
      q += (a.x * a.x + a.y * a.y) + (b.x * b.x + b.y * b.y) + (c.x * c.x + c.y * c.y) + (d.x * d.x + d.y * d.y);
    } else {  // cpg == 4
      s += (a.x + a.y) + (b.x + b.y);
      q += (a.x * a.x + a.y * a.y) + (b.x * b.x + b.y * b.y);
      s2 += (c.x + c.y) + (d.x + d.y);
      q2 += (c.x * c.x + c.y * c.y) + (d.x * d.x + d.y * d.y);
    }
  }
  if (cpg >= 8) {
    const int g = (c8 * 8) / cpg;
    atomicAdd(&s_acc[g * 2], s);
    atomicAdd(&s_acc[g * 2 + 1], q);
  } else {
    const int g = (c8 * 8) / cpg;
    atomicAdd(&s_acc[g * 2], s);
    atomicAdd(&s_acc[g * 2 + 1], q);
    atomicAdd(&s_acc[(g + 1) * 2], s2);
    atomicAdd(&s_acc[(g + 1) * 2 + 1], q2);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) atomicAdd(&part[static_cast<size_t>(img) * groups * 2 + i], s_acc[i]);
}

// (sum, sumsq) of x - pivot -> (mean, rstd), combined in fp64 once per (image, group)
template <bool BF16>
__global__ void gn_finalize_kernel(float* __restrict__ part, const uint16_t* __restrict__ x, int n_slots, int groups, int hw, int C,
                                   double cnt, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_slots) return;
  const double m = static_cast<double>(part[2 * i]) / cnt;     // mean - pivot
  const double var = static_cast<double>(part[2 * i + 1]) / cnt - m * m;
  part[2 * i] = static_cast<float>(gn_pivot<BF16>(x, i / groups, hw, C, i % groups, C / groups) + m);
  part[2 * i + 1] = rsqrtf(static_cast<float>(var > 0.0 ? var : 0.0) + eps);
}

// y = silu?((x - mean) * rstd * gamma + beta), 16-bit in/out, NHWC.  Same thread geometry as gn_stats (block = 256 pixels
// of ONE image, thread = 8 fixed channels), so everything that depends on (image, channel) -- the two statistics, gamma,
// beta -- is folded into 8 (a, b) pairs ONCE per thread and the per-element work is one FMA + SiLU on one MUFU op
// (x * sigmoid(x) = x * (0.5 tanh(x / 2) + 0.5)).  (r02 ncu of the first form, which divided by runtime divisors and
// re-read the statistics for every element: 335 us for 536 MB = 1.6 TB/s, 18 % of HBM, at the 256x256x128 layers.)
template <bool BF16>
__global__ void __launch_bounds__(256) gn_apply_kernel(const uint16_t* __restrict__ x, const float* __restrict__ part,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       uint16_t* __restrict__ y, int hw, int C, int groups, int rows_per_block,
                                                       int do_silu) {
  const int img = blockIdx.y;
  const int c8n = C / 8;
  const int cpg = C / groups;
  const int c8 = threadIdx.x % c8n;
  const int rlane = threadIdx.x / c8n;
  const int rstep = blockDim.x / c8n;
  float ka[8], kb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = c8 * 8 + j;
    const float2 st = __ldg(reinterpret_cast<const float2*>(part) + static_cast<size_t>(img) * groups + ch / cpg);   // (mean, rstd)
    ka[j] = st.y * __ldg(gamma + ch);
    kb[j] = fmaf(-st.x, ka[j], __ldg(beta + ch));
  }
  const int row0 = blockIdx.x * rows_per_block;
  for (int r = row0 + rlane; r < row0 + rows_per_block && r < hw; r += rstep) {
    const size_t idx = (static_cast<size_t>(img) * hw + r) * c8n + c8;
    const uint4 v = reinterpret_cast<const uint4*>(x)[idx];
    float f[8];
    {
      const float2 a = unpack2<BF16>(v.x), b = unpack2<BF16>(v.y), c = unpack2<BF16>(v.z), d = unpack2<BF16>(v.w);
      f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float o = fmaf(f[j], ka[j], kb[j]);
      if (do_silu) {
        float t;
        asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * o));
        f[j] = o * fmaf(0.5f, t, 0.5f);
      } else {
        f[j] = o;
      }
    }
    reinterpret_cast<uint4*>(y)[idx] = make_uint4(pack2<BF16>(f[0], f[1]), pack2<BF16>(f[2], f[3]), pack2<BF16>(f[4], f[5]), pack2<BF16>(f[6], f[7]));
  }
}

// nearest-neighbour 2x upsample, NHWC 16-bit (diffusers Upsample2D: F.interpolate(scale_factor=2, mode="nearest"))
__global__ void __launch_bounds__(256) upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int n_img, int h, int w, int c8n) {
  const long long total = static_cast<long long>(n_img) * (2 * h) * (2 * w) * c8n;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % c8n);
    long long p = i / c8n;
    const int ox = static_cast<int>(p % (2 * w)); p /= (2 * w);
    const int oy = static_cast<int>(p % (2 * h));
    const int img = static_cast<int>(p / (2 * h));
    y[i] = x[((static_cast<long long>(img) * h + oy / 2) * w + ox / 2) * c8n + c];
  }
}

// post_quant_conv (1x1, C->C) then conv_in (3x3, C->Cout, zero padding) on the fp32 NCHW latent -> NHWC 16-bit.
// K = 9*C is tiny (36): CUDA cores.  One block = 8 output pixels x all Cout.
template <bool BF16>
__global__ void __launch_bounds__(256) conv_in_kernel(const float* __restrict__ z, const float* __restrict__ pq_w, const float* __restrict__ pq_b,
                                                      const float* __restrict__ w, const float* __restrict__ b, uint16_t* __restrict__ y,
                                                      int n_img, int C, int h, int wd, int Cout, int use_pq) {
  __shared__ float patch[8][9 * 8];  // up to C = 8 latent channels
  const int K = 9 * C;
  const long long pix0 = static_cast<long long>(blockIdx.x) * 8;
  const long long total = static_cast<long long>(n_img) * h * wd;
  for (int i = threadIdx.x; i < 8 * K; i += blockDim.x) {
    const int pl = i / K, k = i % K;
    const int c = k / 9, tap = k % 9;
    const long long pix = pix0 + pl;
    float v = 0.f;
    if (pix < total) {
      const int x0 = static_cast<int>(pix % wd), y0 = static_cast<int>((pix / wd) % h), img = static_cast<int>(pix / (static_cast<long long>(wd) * h));
      const int xx = x0 + tap % 3 - 1, yy = y0 + tap / 3 - 1;
      if (xx >= 0 && xx < wd && yy >= 0 && yy < h) {
        if (use_pq) {
          v = pq_b[c];
          for (int m = 0; m < C; ++m) v = fmaf(pq_w[c * C + m], z[((static_cast<long long>(img) * C + m) * h + yy) * wd + xx], v);
        } else {
          v = z[((static_cast<long long>(img) * C + c) * h + yy) * wd + xx];
        }
      }
    }
    patch[pl][k] = v;
  }
  __syncthreads();
  for (int o = threadIdx.x; o < Cout; o += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int pl = 0; pl < 8; ++pl) acc[pl] = b[o];
    for (int k = 0; k < K; ++k) {
      const float wv = __ldg(w + static_cast<size_t>(o) * K + k);  // [Cout][C][3][3] flattened: k = c*9 + tap
#pragma unroll
      for (int pl = 0; pl < 8; ++pl) acc[pl] = fmaf(wv, patch[pl][k], acc[pl]);
    }
#pragma unroll
    for (int pl = 0; pl < 8; ++pl) {
      const long long pix = pix0 + pl;
      if (pix < total) {
        const uint32_t pk = pack2<BF16>(acc[pl], 0.f);
        y[pix * Cout + o] = static_cast<uint16_t>(pk & 0xffff);
      }
    }
  }
}

// softmax over rows of an fp32 [rows, n] score matrix scaled by `scale`, 16-bit output (mid-block attention, 1 head)
template <bool BF16>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, uint16_t* __restrict__ p, int rows, int n, float scale) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* r = s + static_cast<size_t>(warp) * n;
  float mx = -INFINITY;
  for (int i = lane; i < n; i += 32) mx = fmaxf(mx, r[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int i = lane; i < n; i += 32) sum += __expf((r[i] - mx) * scale);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  for (int i = lane * 2; i < n; i += 64) {
    const float a = __expf((r[i] - mx) * scale) * inv, b = __expf((r[i + 1] - mx) * scale) * inv;
    *reinterpret_cast<uint32_t*>(p + static_cast<size_t>(warp) * n + i) = pack2<BF16>(a, b);
  }
}

// [pixels, cpad] 16-bit NHWC (first `c` channels valid) -> [n_img, c, h, w] fp32
template <bool BF16>
__global__ void __launch_bounds__(256) to_nchw_kernel(const uint16_t* __restrict__ x, float* __restrict__ y, int n_img, int c, int cpad, int hw) {
  const long long total = static_cast<long long>(n_img) * c * hw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pix = static_cast<int>(i % hw);
    const int ch = static_cast<int>((i / hw) % c);
    const int img = static_cast<int>(i / (static_cast<long long>(hw) * c));
    const uint16_t v = x[(static_cast<size_t>(img) * hw + pix) * cpad + ch];
    y[i] = unpack2<BF16>(static_cast<uint32_t>(v)).x;
  }
}

// time_conv_out: Conv3d(C, C, (3,1,1), padding (1,0,0)) over the frames of one clip, fp32 NCHW in/out
__global__ void __launch_bounds__(256) time_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                                        float* __restrict__ y, int frames, int c, int hw) {
  const long long total = static_cast<long long>(frames) * c * hw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pix = static_cast<int>(i % hw);
    const int co = static_cast<int>((i / hw) % c);
    const int f = static_cast<int>(i / (static_cast<long long>(hw) * c));
    float acc = b[co];
    for (int ci = 0; ci < c; ++ci)
#pragma unroll
      for (int kt = 0; kt < 3; ++kt) {
        const int ff = f + kt - 1;
        if (ff >= 0 && ff < frames) acc = fmaf(w[(co * c + ci) * 3 + kt], x[(static_cast<long long>(ff) * c + ci) * hw + pix], acc);
      }
    y[i] = acc;
  }
}

// Encoder downsampling (diffusers Downsample2D: pad (0,1,0,1) then Conv2d 3x3 stride 2) as a stride-1 convolution: the input
// [n, H, W, C] is regrouped into its four pixel phases, out[n, y, x, (py*2+px)*C + c] = in[n, 2y+py, 2x+px, c]; input pixel
// (2y+dy, 2x+dx), dy,dx in 0..2, is then phase (dy&1, dx&1) at offset (dy>>1, dx>>1), i.e. a 2x2-tap convolution over 4C
// channels whose (phase 1, offset 1) weights are zero (host packer), and the bottom / right zero padding is the TMA box
// running past the edge.  One 16-byte chunk (8 channels) per thread.
__global__ void __launch_bounds__(256) space_to_depth_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int n_img, int h, int w, int c8n) {
  const int ho = h / 2, wo = w / 2;
  const long long total = static_cast<long long>(n_img) * ho * wo * 4 * c8n;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % c8n);
    const int ph = static_cast<int>((i / c8n) % 4);
    const long long p = i / (4LL * c8n);
    const int ox = static_cast<int>(p % wo), oy = static_cast<int>((p / wo) % ho);
    const int img = static_cast<int>(p / (static_cast<long long>(wo) * ho));
    y[i] = x[((static_cast<long long>(img) * h + 2 * oy + (ph >> 1)) * w + 2 * ox + (ph & 1)) * c8n + c];
  }
}

// conv_out result [pixels, 32] 16-bit NHWC (first M = 2 * latent channels valid) -> quant_conv (1x1, M -> M, fp32, optional)
// -> moments [n_img, M, h, w] fp32 (mean channels first, then log-variance: DiagonalGaussianDistribution's chunk(2, dim=1))
template <bool BF16>
__global__ void __launch_bounds__(256) moments_kernel(const uint16_t* __restrict__ x, const float* __restrict__ qw, const float* __restrict__ qb,
                                                      float* __restrict__ out, int n_img, int M, int hw) {
  const long long total = static_cast<long long>(n_img) * hw;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = j < M ? unpack2<BF16>(static_cast<uint32_t>(x[p * 32 + j])).x : 0.f;
    const int img = static_cast<int>(p / hw), pix = static_cast<int>(p % hw);
    for (int o = 0; o < M; ++o) {
      float acc = v[o];
      if (qw != nullptr) {
        acc = qb[o];
        for (int j = 0; j < M; ++j) acc = fmaf(qw[o * M + j], v[j], acc);
      }
      out[(static_cast<long long>(img) * M + o) * hw + pix] = acc;
    }
  }
}

inline int grid_for(long long n, int cap = 132 * 16) {
  long long b = (n + 255) / 256;
  return static_cast<int>(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace

int launch_gn(const void* x, float* part, const float* gamma, const float* beta, void* y, int n_img, int hw, int C, int groups,
              float eps, int do_silu, int bf16, cudaStream_t stream) {
  B200_REQUIRE(C % 8 == 0 && C % groups == 0 && ((C / groups) % 8 == 0 || (C / groups) == 4), B200_ERR_UNSUPPORTED,
               "group norm: C=%d groups=%d unsupported", C, groups);
  B200_REQUIRE(256 % (C / 8) == 0 || (C / 8) % 256 == 0 || C / 8 <= 256, B200_ERR_UNSUPPORTED, "group norm: C=%d", C);
  B200_REQUIRE(C / 8 <= 256 && 256 % (C / 8) == 0, B200_ERR_UNSUPPORTED, "group norm: C/8 = %d must divide 256", C / 8);
  B200_CHECK_CUDA(cudaMemsetAsync(part, 0, static_cast<size_t>(n_img) * groups * 2 * sizeof(float), stream));
  const int rows_per_block = 256;
  dim3 grid((hw + rows_per_block - 1) / rows_per_block, n_img);
  const size_t smem = static_cast<size_t>(groups) * 2 * sizeof(float);
  const int slots = n_img * groups;
  const double cnt = static_cast<double>(hw) * (C / groups);
  if (bf16) {
    gn_stats_kernel<true><<<grid, 256, smem, stream>>>(static_cast<const uint16_t*>(x), part, hw, C, groups, rows_per_block);
    gn_finalize_kernel<true><<<(slots + 127) / 128, 128, 0, stream>>>(part, static_cast<const uint16_t*>(x), slots, groups, hw, C, cnt, eps);
    gn_apply_kernel<true><<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), part, gamma, beta, static_cast<uint16_t*>(y), hw, C, groups, rows_per_block, do_silu);
  } else {
    gn_stats_kernel<false><<<grid, 256, smem, stream>>>(static_cast<const uint16_t*>(x), part, hw, C, groups, rows_per_block);
    gn_finalize_kernel<false><<<(slots + 127) / 128, 128, 0, stream>>>(part, static_cast<const uint16_t*>(x), slots, groups, hw, C, cnt, eps);
    gn_apply_kernel<false><<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), part, gamma, beta, static_cast<uint16_t*>(y), hw, C, groups, rows_per_block, do_silu);
  }
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_upsample2x(const void* x, void* y, int n_img, int h, int w, int C, cudaStream_t stream) {
  B200_REQUIRE(C % 8 == 0, B200_ERR_SHAPE, "upsample: C=%d must be a multiple of 8", C);
  const long long total = static_cast<long long>(n_img) * 4 * h * w * (C / 8);
  upsample2x_kernel<<<grid_for(total), 256, 0, stream>>>(static_cast<const uint4*>(x), static_cast<uint4*>(y), n_img, h, w, C / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_conv_in(const float* z, const float* pq_w, const float* pq_b, const float* w, const float* b, void* y, int n_img, int C,
                   int h, int wd, int Cout, int bf16, cudaStream_t stream) {
  B200_REQUIRE(C <= 8, B200_ERR_UNSUPPORTED, "conv_in: %d latent channels (<= 8 built)", C);
  const long long total = static_cast<long long>(n_img) * h * wd;
  const int blocks = static_cast<int>((total + 7) / 8);
  if (bf16) conv_in_kernel<true><<<blocks, 256, 0, stream>>>(z, pq_w, pq_b, w, b, static_cast<uint16_t*>(y), n_img, C, h, wd, Cout, pq_w != nullptr);
  else conv_in_kernel<false><<<blocks, 256, 0, stream>>>(z, pq_w, pq_b, w, b, static_cast<uint16_t*>(y), n_img, C, h, wd, Cout, pq_w != nullptr);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_softmax_rows(const float* s, void* p, int rows, int n, float scale, int bf16, cudaStream_t stream) {
  B200_REQUIRE(n % 2 == 0, B200_ERR_SHAPE, "softmax: n=%d must be even", n);
  const int blocks = (rows * 32 + 255) / 256;
  if (bf16) softmax_rows_kernel<true><<<blocks, 256, 0, stream>>>(s, static_cast<uint16_t*>(p), rows, n, scale);
  else softmax_rows_kernel<false><<<blocks, 256, 0, stream>>>(s, static_cast<uint16_t*>(p), rows, n, scale);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_time_conv(const float* x, const float* w, const float* b, float* y, int frames, int c, int hw, cudaStream_t stream) {
  const long long total = static_cast<long long>(frames) * c * hw;
  time_conv_kernel<<<grid_for(total), 256, 0, stream>>>(x, w, b, y, frames, c, hw);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_to_nchw(const void* x, float* y, int n_img, int c, int cpad, int hw, int bf16, cudaStream_t stream) {
  const long long total = static_cast<long long>(n_img) * c * hw;
  if (bf16) to_nchw_kernel<true><<<grid_for(total), 256, 0, stream>>>(static_cast<const uint16_t*>(x), y, n_img, c, cpad, hw);
  else to_nchw_kernel<false><<<grid_for(total), 256, 0, stream>>>(static_cast<const uint16_t*>(x), y, n_img, c, cpad, hw);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}


int launch_space_to_depth(const void* x, void* y, int n_img, int h, int w, int C, cudaStream_t stream) {
  B200_REQUIRE(C % 8 == 0 && h % 2 == 0 && w % 2 == 0, B200_ERR_SHAPE, "space_to_depth: C %% 8, even h and w required");
  const long long total = static_cast<long long>(n_img) * (h / 2) * (w / 2) * 4 * (C / 8);
  space_to_depth_kernel<<<grid_for(total), 256, 0, stream>>>(static_cast<const uint4*>(x), static_cast<uint4*>(y), n_img, h, w, C / 8);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

int launch_moments(const void* x, const float* qw, const float* qb, float* out, int n_img, int M, int hw, int bf16, cudaStream_t stream) {
  B200_REQUIRE(M > 0 && M <= 8, B200_ERR_UNSUPPORTED, "moments: %d channels (<= 8 built)", M);
  const long long total = static_cast<long long>(n_img) * hw;
  if (bf16) moments_kernel<true><<<grid_for(total), 256, 0, stream>>>(static_cast<const uint16_t*>(x), qw, qb, out, n_img, M, hw);
  else moments_kernel<false><<<grid_for(total), 256, 0, stream>>>(static_cast<const uint16_t*>(x), qw, qb, out, n_img, M, hw);
  B200_CHECK_CUDA(cudaGetLastError());
  return B200_OK;
}

// ====================================================================================================== decode
namespace {

inline size_t up1k(size_t v) { return (v + 1023) / 1024 * 1024; }

struct VaeWs {
  uint8_t* buf[4];     // activation ping-pong, each n_img * (8h*8w) * cmax_at_res... sized for the largest tensor
  uint8_t* q; uint8_t* k; uint8_t* vt; uint8_t* p16; float* scores; float* ones; float* part;
  size_t bytes;
};

size_t largest_activation(const B200VaeDecoder* d, int n_img, int h, int w) {
  size_t best = 0;
  int c = d->up_channels[0];
  size_t pix = static_cast<size_t>(n_img) * h * w;
  best = pix * c * 2;
  for (int b = 0; b < d->n_up; ++b) {
    const int co = d->up_channels[b];
    const size_t here = pix * static_cast<size_t>(c > co ? c : co) * 2;
    if (here > best) best = here;
    c = co;
    if (b + 1 < d->n_up) {
      pix *= 4;
      if (pix * c * 2 > best) best = pix * c * 2;
    }
  }
  const size_t outpad = pix * 32 * 2;
  return best > outpad ? best : outpad;
}

void vae_carve(const B200VaeDecoder* d, int n_img, int h, int w, void* base, VaeWs* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += up1k(bytes);
    return p;
  };
  const size_t act = largest_activation(d, n_img, h, w);
  for (int i = 0; i < 4; ++i) ws->buf[i] = take(act);
  const size_t hw = static_cast<size_t>(h) * w, C0 = d->up_channels[0];
  ws->q = take(static_cast<size_t>(n_img) * hw * C0 * 2);
  ws->k = take(static_cast<size_t>(n_img) * hw * C0 * 2);
  ws->vt = take(C0 * hw * 2);
  ws->p16 = take(hw * hw * 2);
  ws->scores = reinterpret_cast<float*>(take(hw * hw * 4));
  ws->ones = reinterpret_cast<float*>(take(hw * 4));
  ws->part = reinterpret_cast<float*>(take(static_cast<size_t>(n_img) * d->groups * 2 * 4));
  ws->bytes = off;
}

int vae_ok(const B200VaeDecoder* d, int n_img, int h, int w) {
  B200_REQUIRE(d && n_img > 0 && h > 0 && w > 0, B200_ERR_SHAPE, "vae: bad arguments");
  B200_REQUIRE(d->n_up >= 1 && d->n_up <= 4 && d->layers_per_block == 2, B200_ERR_UNSUPPORTED, "vae: topology not built (n_up %d, layers %d)", d->n_up, d->layers_per_block);
  B200_REQUIRE(d->latent_channels <= 8 && d->out_channels <= 32, B200_ERR_UNSUPPORTED, "vae: channels");
  for (int b = 0; b < d->n_up; ++b) B200_REQUIRE(d->up_channels[b] % 64 == 0, B200_ERR_UNSUPPORTED, "vae: channels %d not a multiple of 64", d->up_channels[b]);
  B200_REQUIRE((h * w) % 128 == 0 && (w >= 128 ? w % 128 == 0 : 128 % w == 0) && h % (w >= 128 ? 1 : 128 / w) == 0, B200_ERR_UNSUPPORTED,
               "vae: %dx%d latent cannot be tiled by 128-pixel patches", h, w);
  B200_REQUIRE(d->dtype == B200_FP16 || d->dtype == B200_BF16, B200_ERR_DTYPE, "vae: dtype");
  return B200_OK;
}

struct VaeCtx {
  const B200VaeDecoder* d;
  VaeWs ws;
  int groups;
  float eps, temporal_eps;
  int n_img, bf16;
  int frames;     // > 0: temporal decoder, the n_img frames form n_img / frames clips
  cudaStream_t stream;
};

int conv3x3(VaeCtx& c, const void* x, const void* w16, const float* bias, void* y, int h, int w, int cin, int cout, const void* add16) {
  GemmArgs a{};
  a.A = x; a.W = w16; a.bias = bias; a.M = c.n_img * h * w; a.N = cout; a.K = 9 * cin; a.bf16 = c.bf16;
  a.epilogue = add16 ? B200_EPI_BIAS_ADD16 : B200_EPI_BIAS; a.out16 = y; a.add16 = add16;
  a.conv_taps = 9; a.conv_n = c.n_img; a.conv_h = h; a.conv_w = w; a.conv_c = cin;
  for (int t = 0; t < 9; ++t) { a.conv_dx[t] = t % 3 - 1; a.conv_dy[t] = t / 3 - 1; a.conv_dz[t] = 0; }
  return launch_gemm(a, c.stream);
}

// Conv3d (3,1,1), padding (1,0,0): 3 taps along the frame index of ONE clip (the image coordinate of the TMA box)
int conv_t3(VaeCtx& c, const void* x, const void* w16, const float* bias, void* y, int h, int w, int ch, const void* add16) {
  GemmArgs a{};
  a.A = x; a.W = w16; a.bias = bias; a.M = c.n_img * h * w; a.N = ch; a.K = 3 * ch; a.bf16 = c.bf16;
  a.epilogue = add16 ? B200_EPI_BIAS_ADD16 : B200_EPI_BIAS; a.out16 = y; a.add16 = add16;
  a.conv_taps = 3; a.conv_n = c.n_img; a.conv_h = h; a.conv_w = w; a.conv_c = ch;
  for (int t = 0; t < 9; ++t) { a.conv_dx[t] = 0; a.conv_dy[t] = 0; a.conv_dz[t] = t < 3 ? t - 1 : 0; }
  return launch_gemm(a, c.stream);
}

// Downsample2D (pad (0,1,0,1), Conv2d 3x3 stride 2) on an h x w input: space_to_depth into `s2d` [n_img, h/2, w/2, 4 cin], then
// the 2x2-tap implicit GEMM over 4 cin channels; w16 is [cout][tap = oy*2+ox][phase = py*2+px][cin] (host packer)
int conv_down2(VaeCtx& c, const void* x, void* s2d, const void* w16, const float* bias, void* y, int h, int w, int cin, int cout) {
  B200_TRY(launch_space_to_depth(x, s2d, c.n_img, h, w, cin, c.stream));
  const int ho = h / 2, wo = w / 2;
  GemmArgs a{};
  a.A = s2d; a.W = w16; a.bias = bias; a.M = c.n_img * ho * wo; a.N = cout; a.K = 4 * 4 * cin; a.bf16 = c.bf16;
  a.epilogue = B200_EPI_BIAS; a.out16 = y;
  a.conv_taps = 4; a.conv_n = c.n_img; a.conv_h = ho; a.conv_w = wo; a.conv_c = 4 * cin;
  for (int t = 0; t < 9; ++t) { a.conv_dx[t] = t < 4 ? (t & 1) : 0; a.conv_dy[t] = t < 4 ? (t >> 1) : 0; a.conv_dz[t] = 0; }
  return launch_gemm(a, c.stream);
}

int gemm16(VaeCtx& c, const void* A, const void* W, const float* bias, int M, int N, int K, void* y, const void* add16) {
  GemmArgs a{};
  a.A = A; a.W = W; a.bias = bias; a.M = M; a.N = N; a.K = K; a.bf16 = c.bf16;
  a.epilogue = add16 ? B200_EPI_BIAS_ADD16 : B200_EPI_BIAS; a.out16 = y; a.add16 = add16;
  return launch_gemm(a, c.stream);
}

// x in buf[xi]; returns index of the buffer holding the block output
int resnet(VaeCtx& c, const B200VaeResnet& r, int xi, int h, int w, int* out_idx) {
  int free_[3], nf = 0;
  for (int i = 0; i < 4; ++i) if (i != xi) free_[nf++] = i;
  uint8_t* x = c.ws.buf[xi];
  uint8_t* t1 = c.ws.buf[free_[0]];
  uint8_t* t2 = c.ws.buf[free_[1]];
  uint8_t* sc = c.ws.buf[free_[2]];
  const int hw = h * w;
  B200_TRY(launch_gn(x, c.ws.part, r.gn1_g, r.gn1_b, t1, c.n_img, hw, r.cin, c.groups, c.eps, 1, c.bf16, c.stream));
  B200_TRY(conv3x3(c, t1, r.conv1_w16, r.conv1_b, t2, h, w, r.cin, r.cout, nullptr));
  B200_TRY(launch_gn(t2, c.ws.part, r.gn2_g, r.gn2_b, t1, c.n_img, hw, r.cout, c.groups, c.eps, 1, c.bf16, c.stream));
  const void* shortcut = x;
  if (r.short_w16) {
    B200_TRY(gemm16(c, x, r.short_w16, r.short_b, c.n_img * hw, r.cout, r.cin, sc, nullptr));
    shortcut = sc;
  }
  B200_TRY(conv3x3(c, t1, r.conv2_w16, r.conv2_b, t2, h, w, r.cout, r.cout, shortcut));
  *out_idx = free_[1];
  if (r.t_conv1_w16 && c.frames > 0) {
    // TemporalResnetBlock on x_s = t2 (GroupNorm statistics over ALL frames of the clip), blended by the AlphaBlender:
    //   out = x_s + (1 - alpha) * conv2(silu(gn2(conv1(silu(gn1(x_s))))))   -- (1 - alpha) is folded into conv2 by the packer
    const int clips = c.n_img / c.frames;
    uint8_t* xs = t2;
    uint8_t* u1 = t1;
    uint8_t* u2 = x;     // the block input is dead by now
    B200_TRY(launch_gn(xs, c.ws.part, r.t_gn1_g, r.t_gn1_b, u1, clips, c.frames * hw, r.cout, c.groups, c.temporal_eps, 1, c.bf16, c.stream));
    B200_TRY(conv_t3(c, u1, r.t_conv1_w16, r.t_conv1_b, u2, h, w, r.cout, nullptr));
    B200_TRY(launch_gn(u2, c.ws.part, r.t_gn2_g, r.t_gn2_b, u1, clips, c.frames * hw, r.cout, c.groups, c.temporal_eps, 1, c.bf16, c.stream));
    B200_TRY(conv_t3(c, u1, r.t_conv2_w16, r.t_conv2_b, u2, h, w, r.cout, xs));
    *out_idx = xi;
  }
  return B200_OK;
}

// mid-block attention (1 head over the h*w positions of each image): x + to_out(softmax(q k^T / sqrt(C)) v), GroupNorm first
struct MidAttn {
  const float* gn_g; const float* gn_b;
  const void* q_w16; const float* q_b; const void* k_w16; const float* k_b;
  const void* v_w16;                    // v bias folded into o_b by the packer
  const void* o_w16; const float* o_b;
};
int mid_attention(VaeCtx& c, const MidAttn& a, int C0, int xi, int h, int w, int* out_idx) {
  const int hw = h * w, n_img = c.n_img;
  cudaStream_t stream = c.stream;
  int fr[3], nf = 0;
  for (int i = 0; i < 4; ++i) if (i != xi) fr[nf++] = i;
  uint8_t* x = c.ws.buf[xi];
  uint8_t* xg = c.ws.buf[fr[0]];
  uint8_t* o = c.ws.buf[fr[1]];
  B200_TRY(launch_gn(x, c.ws.part, a.gn_g, a.gn_b, xg, n_img, hw, C0, c.groups, c.eps, 0, c.bf16, stream));
  B200_TRY(gemm16(c, xg, a.q_w16, a.q_b, n_img * hw, C0, C0, c.ws.q, nullptr));
  B200_TRY(gemm16(c, xg, a.k_w16, a.k_b, n_img * hw, C0, C0, c.ws.k, nullptr));
  B200_TRY(launch_fill(c.ws.ones, 1.0f, hw, stream));
  const float scale = 1.0f / sqrtf(static_cast<float>(C0));
  for (int f = 0; f < n_img; ++f) {
    const size_t off = static_cast<size_t>(f) * hw * C0 * 2;
    // V^T [C0, hw] = Wv [C0, C0] . xg_f^T  (bias of v is folded into the output projection bias by the packer)
    B200_TRY(gemm16(c, a.v_w16, xg + off, nullptr, C0, hw, C0, c.ws.vt, nullptr));
    // fp32 scores = q_f k_f^T through the residual epilogue on a zeroed buffer (gate = 1)
    B200_CHECK_CUDA(cudaMemsetAsync(c.ws.scores, 0, static_cast<size_t>(hw) * hw * 4, stream));
    GemmArgs sc{};
    sc.A = c.ws.q + off; sc.W = c.ws.k + off; sc.M = hw; sc.N = hw; sc.K = C0; sc.bf16 = c.bf16; sc.epilogue = B200_EPI_GATE_RESIDUAL;
    sc.resid = c.ws.scores; sc.gate = c.ws.ones; sc.gate_batch_stride = 0; sc.rows_per_batch = hw;
    B200_TRY(launch_gemm(sc, stream));
    B200_TRY(launch_softmax_rows(c.ws.scores, c.ws.p16, hw, hw, scale, c.bf16, stream));
    B200_TRY(gemm16(c, c.ws.p16, c.ws.vt, nullptr, hw, C0, hw, o + off, nullptr));
  }
  B200_TRY(gemm16(c, o, a.o_w16, a.o_b, n_img * hw, C0, C0, xg, x));   // + residual
  *out_idx = fr[0];
  return B200_OK;
}

int vae_decode(const B200VaeDecoder* d, const float* z, int n_img, int h, int w, int num_frames, float* out, void* workspace,
               size_t workspace_bytes, cudaStream_t stream) {
  B200_TRY(vae_ok(d, n_img, h, w));
  B200_REQUIRE(num_frames == 0 || num_frames == n_img, B200_ERR_UNSUPPORTED,
               "vae: temporal decode takes ONE clip per call (n_img %d != num_frames %d); decode clips one by one", n_img, num_frames);
  B200_REQUIRE(z && out && workspace && (reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, B200_ERR_ALIGN, "vae: bad pointers");
  B200_TRY(check_arch());
  VaeCtx c{};
  c.d = d; c.n_img = n_img; c.bf16 = d->dtype == B200_BF16; c.stream = stream; c.frames = num_frames;
  c.groups = d->groups; c.eps = d->eps; c.temporal_eps = d->temporal_eps;
  vae_carve(d, n_img, h, w, workspace, &c.ws);
  B200_REQUIRE(c.ws.bytes <= workspace_bytes, B200_ERR_WORKSPACE, "vae: workspace too small: need %zu bytes, got %zu", c.ws.bytes, workspace_bytes);
  const int C0 = d->up_channels[0];
  const int hw = h * w;

  // post_quant_conv + conv_in
  int xi = 0;
  B200_TRY(launch_conv_in(z, d->pq_w, d->pq_b, d->conv_in_w, d->conv_in_b, c.ws.buf[xi], n_img, d->latent_channels, h, w, C0, c.bf16, stream));
  // mid block: resnet, single-head attention over the h*w positions, resnet
  B200_TRY(resnet(c, d->mid[0], xi, h, w, &xi));
  {
    const MidAttn at{d->attn_gn_g, d->attn_gn_b, d->attn_q_w16, d->attn_q_b, d->attn_k_w16, d->attn_k_b, d->attn_v_w16, d->attn_o_w16, d->attn_o_b};
    B200_TRY(mid_attention(c, at, C0, xi, h, w, &xi));
  }
  B200_TRY(resnet(c, d->mid[1], xi, h, w, &xi));

  // up blocks
  int ch = h, cw = w;
  for (int b = 0; b < d->n_up; ++b) {
    for (int r = 0; r < 3; ++r) B200_TRY(resnet(c, d->up[b * 3 + r], xi, ch, cw, &xi));
    if (b + 1 < d->n_up) {
      const int co = d->up_channels[b];
      int fr[3], nf = 0;
      for (int i = 0; i < 4; ++i) if (i != xi) fr[nf++] = i;
      B200_TRY(launch_upsample2x(c.ws.buf[xi], c.ws.buf[fr[0]], n_img, ch, cw, co, stream));
      ch *= 2; cw *= 2;
      B200_TRY(conv3x3(c, c.ws.buf[fr[0]], d->ups_w16[b], d->ups_b[b], c.ws.buf[fr[1]], ch, cw, co, co, nullptr));
      xi = fr[1];
    }
  }
  // conv_norm_out + SiLU + conv_out (Cout padded to 32) -> NCHW fp32
  {
    const int cl = d->up_channels[d->n_up - 1];
    int fr[3], nf = 0;
    for (int i = 0; i < 4; ++i) if (i != xi) fr[nf++] = i;
    B200_TRY(launch_gn(c.ws.buf[xi], c.ws.part, d->norm_out_g, d->norm_out_b, c.ws.buf[fr[0]], n_img, ch * cw, cl, d->groups, d->eps, 1, c.bf16, stream));
    B200_TRY(conv3x3(c, c.ws.buf[fr[0]], d->conv_out_w16, d->conv_out_b, c.ws.buf[fr[1]], ch, cw, cl, 32, nullptr));
    if (num_frames > 0 && d->time_conv_w) {
      float* tmp = reinterpret_cast<float*>(c.ws.buf[fr[2]]);
      B200_TRY(launch_to_nchw(c.ws.buf[fr[1]], tmp, n_img, d->out_channels, 32, ch * cw, c.bf16, stream));
      B200_TRY(launch_time_conv(tmp, d->time_conv_w, d->time_conv_b, out, n_img, d->out_channels, ch * cw, stream));
    } else {
      B200_TRY(launch_to_nchw(c.ws.buf[fr[1]], out, n_img, d->out_channels, 32, ch * cw, c.bf16, stream));
    }
  }
  return B200_OK;
}

// ====================================================================================================== encode
// AutoencoderKL.encode (train.py:206-211: vae.encode(x).latent_dist): Encoder = conv_in, n_down DownEncoderBlock2D (2 resnets,
// stride-2 conv except the last), mid block (resnet, attention, resnet), GroupNorm + SiLU, conv_out -> quant_conv -> moments.
int enc_ok(const B200VaeEncoder* e, int n_img, int h, int w) {
  B200_REQUIRE(e && n_img > 0 && h > 0 && w > 0, B200_ERR_SHAPE, "vae encode: bad arguments");
  B200_REQUIRE(e->n_down >= 1 && e->n_down <= 4 && e->in_channels <= 8 && e->latent_channels >= 1 && e->latent_channels <= 4,
               B200_ERR_UNSUPPORTED, "vae encode: topology not built (n_down %d, in %d, latent %d)", e->n_down, e->in_channels, e->latent_channels);
  for (int b = 0; b < e->n_down; ++b) B200_REQUIRE(e->down_channels[b] % 64 == 0, B200_ERR_UNSUPPORTED, "vae encode: channels %d not a multiple of 64", e->down_channels[b]);
  const int f = 1 << (e->n_down - 1);
  B200_REQUIRE(h % f == 0 && w % f == 0, B200_ERR_SHAPE, "vae encode: %dx%d not divisible by %d", h, w, f);
  for (int b = 0, ch = h, cw = w; b < e->n_down; ++b, ch /= 2, cw /= 2)
    B200_REQUIRE((ch * cw) % 128 == 0 && (cw >= 128 ? cw % 128 == 0 : 128 % cw == 0) && ch % (cw >= 128 ? 1 : 128 / cw) == 0, B200_ERR_UNSUPPORTED,
                 "vae encode: the %dx%d feature map cannot be tiled by 128-pixel patches", ch, cw);
  B200_REQUIRE(e->dtype == B200_FP16 || e->dtype == B200_BF16, B200_ERR_DTYPE, "vae encode: dtype");
  return B200_OK;
}

void enc_carve(const B200VaeEncoder* e, int n_img, int h, int w, void* base, VaeWs* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += up1k(bytes);
    return p;
  };
  size_t act = 0;
  for (int b = 0, ch = h, cw = w, cin = e->down_channels[0]; b < e->n_down; ++b, ch /= 2, cw /= 2) {
    const int co = e->down_channels[b];
    const size_t here = static_cast<size_t>(n_img) * ch * cw * static_cast<size_t>(cin > co ? cin : co) * 2;
    if (here > act) act = here;
    cin = co;
  }
  for (int i = 0; i < 4; ++i) ws->buf[i] = take(act);
  const int f = 1 << (e->n_down - 1);
  const size_t hw = static_cast<size_t>(h / f) * (w / f), C0 = e->down_channels[e->n_down - 1];
  ws->q = take(static_cast<size_t>(n_img) * hw * C0 * 2);
  ws->k = take(static_cast<size_t>(n_img) * hw * C0 * 2);
  ws->vt = take(C0 * hw * 2);
  ws->p16 = take(hw * hw * 2);
  ws->scores = reinterpret_cast<float*>(take(hw * hw * 4));
  ws->ones = reinterpret_cast<float*>(take(hw * 4));
  ws->part = reinterpret_cast<float*>(take(static_cast<size_t>(n_img) * e->groups * 2 * 4));
  ws->bytes = off;
}

int vae_encode(const B200VaeEncoder* e, const float* x, int n_img, int h, int w, float* moments, void* workspace, size_t workspace_bytes,
               cudaStream_t stream) {
  B200_TRY(enc_ok(e, n_img, h, w));
  B200_REQUIRE(x && moments && workspace && (reinterpret_cast<uintptr_t>(workspace) & 1023) == 0, B200_ERR_ALIGN, "vae encode: bad pointers");
  B200_TRY(check_arch());
  VaeCtx c{};
  c.d = nullptr; c.n_img = n_img; c.bf16 = e->dtype == B200_BF16; c.stream = stream; c.frames = 0;
  c.groups = e->groups; c.eps = e->eps; c.temporal_eps = e->eps;
  enc_carve(e, n_img, h, w, workspace, &c.ws);
  B200_REQUIRE(c.ws.bytes <= workspace_bytes, B200_ERR_WORKSPACE, "vae encode: workspace too small: need %zu bytes, got %zu", c.ws.bytes, workspace_bytes);
  int xi = 0, ch = h, cw = w;
  B200_TRY(launch_conv_in(x, nullptr, nullptr, e->conv_in_w, e->conv_in_b, c.ws.buf[xi], n_img, e->in_channels, h, w, e->down_channels[0], c.bf16, stream));
  for (int b = 0; b < e->n_down; ++b) {
    for (int r = 0; r < 2; ++r) B200_TRY(resnet(c, e->down[b * 2 + r], xi, ch, cw, &xi));
    if (b + 1 < e->n_down) {
      const int co = e->down_channels[b];
      int fr[3], nf = 0;
      for (int i = 0; i < 4; ++i) if (i != xi) fr[nf++] = i;
      B200_TRY(conv_down2(c, c.ws.buf[xi], c.ws.buf[fr[0]], e->down_w16[b], e->down_b[b], c.ws.buf[fr[1]], ch, cw, co, co));
      ch /= 2; cw /= 2;
      xi = fr[1];
    }
  }
  const int C0 = e->down_channels[e->n_down - 1];
  B200_TRY(resnet(c, e->mid[0], xi, ch, cw, &xi));
  {
    const MidAttn at{e->attn_gn_g, e->attn_gn_b, e->attn_q_w16, e->attn_q_b, e->attn_k_w16, e->attn_k_b, e->attn_v_w16, e->attn_o_w16, e->attn_o_b};
    B200_TRY(mid_attention(c, at, C0, xi, ch, cw, &xi));
  }
  B200_TRY(resnet(c, e->mid[1], xi, ch, cw, &xi));
  {
    int fr[3], nf = 0;
    for (int i = 0; i < 4; ++i) if (i != xi) fr[nf++] = i;
    B200_TRY(launch_gn(c.ws.buf[xi], c.ws.part, e->norm_out_g, e->norm_out_b, c.ws.buf[fr[0]], n_img, ch * cw, C0, e->groups, e->eps, 1, c.bf16, stream));
    B200_TRY(conv3x3(c, c.ws.buf[fr[0]], e->conv_out_w16, e->conv_out_b, c.ws.buf[fr[1]], ch, cw, C0, 32, nullptr));
    B200_TRY(launch_moments(c.ws.buf[fr[1]], e->quant_w, e->quant_b, moments, n_img, 2 * e->latent_channels, ch * cw, c.bf16, stream));
  }
  return B200_OK;
}

// ====================================================================================================== single layers
// The C-ABI entry points below run one layer of the decoder / encoder through the same internal functions, so each can be
// compared with its torch op in isolation.
int mid_attn_ok(int n_img, int h, int w, int C, int groups) {
  B200_REQUIRE(n_img > 0 && h > 0 && w > 0 && C > 0 && groups > 0, B200_ERR_SHAPE, "vae attention: bad arguments");
  B200_REQUIRE(C % 64 == 0 && C % groups == 0 && (h * w) % 64 == 0, B200_ERR_UNSUPPORTED,
               "vae attention: C=%d must be a multiple of 64 and of groups=%d, h*w=%d a multiple of 64", C, groups, h * w);
  return B200_OK;
}

// buf[0] = x (read only), buf[1] = the caller's output (also the GroupNorm result until the last GEMM), buf[2] = attention
// output; then the scratch of mid_attention exactly as vae_carve lays it out
void mid_attn_carve(int n_img, int hw, int C, int groups, void* base, VaeWs* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? static_cast<uint8_t*>(base) + off : nullptr;
    off += up1k(bytes);
    return p;
  };
  const size_t act = static_cast<size_t>(n_img) * hw * C * 2;
  ws->buf[2] = take(act);
  ws->q = take(act);
  ws->k = take(act);
  ws->vt = take(static_cast<size_t>(C) * hw * 2);
  ws->p16 = take(static_cast<size_t>(hw) * hw * 2);
  ws->scores = reinterpret_cast<float*>(take(static_cast<size_t>(hw) * hw * 4));
  ws->ones = reinterpret_cast<float*>(take(static_cast<size_t>(hw) * 4));
  ws->part = reinterpret_cast<float*>(take(static_cast<size_t>(n_img) * groups * 2 * 4));
  ws->bytes = off;
}

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace b200

extern "C" {

B200_API size_t b200_vae_workspace_bytes(const B200VaeDecoder* d, int n_img, int h, int w) {
  if (b200::vae_ok(d, n_img, h, w) != B200_OK) return 0;
  b200::VaeWs ws;
  b200::vae_carve(d, n_img, h, w, nullptr, &ws);
  return ws.bytes;
}

B200_API int b200_vae_decode(const B200VaeDecoder* d, const float* z, int n_img, int h, int w, float* out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  return b200::vae_decode(d, z, n_img, h, w, 0, out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

B200_API size_t b200_vae_encode_workspace_bytes(const B200VaeEncoder* e, int n_img, int h, int w) {
  if (b200::enc_ok(e, n_img, h, w) != B200_OK) return 0;
  b200::VaeWs ws;
  b200::enc_carve(e, n_img, h, w, nullptr, &ws);
  return ws.bytes;
}

B200_API int b200_vae_encode(const B200VaeEncoder* e, const float* x, int n_img, int h, int w, float* moments, void* workspace,
                             size_t workspace_bytes, void* stream) {
  return b200::vae_encode(e, x, n_img, h, w, moments, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

B200_API int b200_vae_decode_temporal(const B200VaeDecoder* d, const float* z, int n_img, int h, int w, int num_frames, float* out,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(num_frames > 0, B200_ERR_SHAPE, "vae: num_frames must be positive");
  return b200::vae_decode(d, z, n_img, h, w, num_frames, out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

B200_API int b200_vae_conv(const void* x, const void* w16, const float* bias, const void* add16, void* out16, void* scratch, int n_img,
                           int h, int w, int cin, int cout, int kind, int dtype, void* stream) {
  using namespace b200;
  B200_REQUIRE(n_img > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, B200_ERR_SHAPE, "vae conv: bad shape");
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "vae conv: dtype %d", dtype);
  B200_REQUIRE(kind == B200_VAE_CONV3X3 || kind == B200_VAE_CONV_T3 || kind == B200_VAE_CONV_DOWN2, B200_ERR_UNSUPPORTED,
               "vae conv: unknown kind %d", kind);
  B200_REQUIRE(cin % 64 == 0, B200_ERR_UNSUPPORTED, "vae conv: cin=%d must be a multiple of 64", cin);
  B200_REQUIRE(kind != B200_VAE_CONV_T3 || cin == cout, B200_ERR_UNSUPPORTED, "vae conv: the temporal conv maps C -> C (cin %d, cout %d)", cin, cout);
  B200_REQUIRE(kind != B200_VAE_CONV_DOWN2 || (add16 == nullptr && h % 2 == 0 && w % 2 == 0), B200_ERR_UNSUPPORTED,
               "vae conv: the stride-2 conv takes an even-sized input and no shortcut");
  B200_REQUIRE(x && w16 && out16 && al16(x) && al16(out16) && (kind != B200_VAE_CONV_DOWN2 || (scratch && al16(scratch))), B200_ERR_ALIGN,
               "vae conv: x, out16 (and the stride-2 scratch) must be 16-byte aligned");
  B200_TRY(check_arch());
  VaeCtx c{};
  c.n_img = n_img; c.bf16 = dtype == B200_BF16; c.stream = static_cast<cudaStream_t>(stream);
  if (kind == B200_VAE_CONV3X3) return conv3x3(c, x, w16, bias, out16, h, w, cin, cout, add16);
  if (kind == B200_VAE_CONV_T3) return conv_t3(c, x, w16, bias, out16, h, w, cin, add16);
  return conv_down2(c, x, scratch, w16, bias, out16, h, w, cin, cout);
}

B200_API int b200_group_norm(const void* x, void* y, const float* gamma, const float* beta, float* part, int n_img, int hw, int C,
                             int groups, float eps, int silu, int dtype, void* stream) {
  using namespace b200;
  B200_REQUIRE(n_img > 0 && n_img <= 65535 && hw > 0 && C > 0 && groups > 0, B200_ERR_SHAPE, "group norm: bad shape");
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "group norm: dtype %d", dtype);
  B200_REQUIRE(x && y && gamma && beta && part && al16(x) && al16(y) && (reinterpret_cast<uintptr_t>(part) & 7) == 0, B200_ERR_ALIGN,
               "group norm: x and y must be 16-byte aligned, part 8-byte aligned");
  B200_TRY(check_arch());
  return launch_gn(x, part, gamma, beta, y, n_img, hw, C, groups, eps, silu, dtype == B200_BF16, static_cast<cudaStream_t>(stream));
}

B200_API size_t b200_vae_mid_attention_workspace_bytes(int n_img, int h, int w, int C, int groups) {
  if (b200::mid_attn_ok(n_img, h, w, C, groups) != B200_OK) return 0;
  b200::VaeWs ws;
  b200::mid_attn_carve(n_img, h * w, C, groups, nullptr, &ws);
  return ws.bytes;
}

B200_API int b200_vae_mid_attention(const void* x, void* out, const float* gn_g, const float* gn_b, const void* q_w16, const float* q_b,
                                    const void* k_w16, const float* k_b, const void* v_w16, const void* o_w16, const float* o_b, int n_img,
                                    int h, int w, int C, int groups, float eps, int dtype, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  using namespace b200;
  B200_TRY(mid_attn_ok(n_img, h, w, C, groups));
  B200_REQUIRE(dtype == B200_FP16 || dtype == B200_BF16, B200_ERR_DTYPE, "vae attention: dtype %d", dtype);
  B200_REQUIRE(x && out && gn_g && gn_b && q_w16 && k_w16 && v_w16 && o_w16 && al16(x) && al16(out) && workspace &&
                   (reinterpret_cast<uintptr_t>(workspace) & 1023) == 0,
               B200_ERR_ALIGN, "vae attention: x and out must be 16-byte aligned, workspace 1024-byte aligned");
  B200_TRY(check_arch());
  VaeCtx c{};
  c.n_img = n_img; c.bf16 = dtype == B200_BF16; c.stream = static_cast<cudaStream_t>(stream);
  c.groups = groups; c.eps = eps; c.temporal_eps = eps;
  mid_attn_carve(n_img, h * w, C, groups, workspace, &c.ws);
  B200_REQUIRE(c.ws.bytes <= workspace_bytes, B200_ERR_WORKSPACE, "vae attention: workspace too small: need %zu bytes, got %zu",
               c.ws.bytes, workspace_bytes);
  c.ws.buf[0] = static_cast<uint8_t*>(const_cast<void*>(x));
  c.ws.buf[1] = static_cast<uint8_t*>(out);
  c.ws.buf[3] = nullptr;
  const MidAttn at{gn_g, gn_b, q_w16, q_b, k_w16, k_b, v_w16, o_w16, o_b};
  int out_idx;   // with the input in buf[0] the result lands in buf[1] = out
  return mid_attention(c, at, C, 0, h, w, &out_idx);
}

}  // extern "C"
