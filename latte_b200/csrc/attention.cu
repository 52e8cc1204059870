// Fused spatial / temporal / cross attention on wgmma:  out = softmax(q k^T * scale (+ bias)) v  per head.
//
// Replaces the 'math' branch of Attention.forward between its two Linears (reference models/latte.py:50-70:
// reshape/permute/.contiguous(), q@k^T, *scale, softmax, @v, transpose/reshape) AND the two einops
// rearranges that regroup tokens between spatial and temporal blocks (latte.py:355,368).  The hidden state and
// the qkv buffer stay in ONE layout, rows = (b, f, n); the regrouping is done by the TMA box that fetches a tile:
//   spatial  (temporal=0): a tile is 128 consecutive tokens of one frame; keys = the frame's N tokens, fetched in
//            chunks of 128 rows.  3-D map {hd, 3H, T}; Q box {64|16, 1, 128}, K/V box {64|16, 1, 128}.
//            N < 128: 128/N whole sequences are packed per tile with a block-diagonal mask (r/N == c/N).
//   temporal (temporal=1): a tile is G = floor(128/F) neighbouring tokens x all F frames, fetched with a 4-D map
//            {hd, 3H, N, B*F} and box {64|16, 1, G, F} -> tile row r = f*G + g < G*F <= 128; the G sequences are
//            masked block-diagonally (c < G*F and r % G == c % G).  Wasted tensor FLOPs (x G) are cheap; HBM traffic
//            is minimal: every q/k/v element is read once, every output written once, no transpose pass.
//            When G does not divide N the last group of a sequence is partial: TMA zero-fills its missing tokens on
//            load and clips them on store.  When G*F < 128, K/V rows [G*F, 128) are never loaded; the V rows are
//            zeroed (P = 0 times stale NaN bits would be NaN), the K rows are removed by the mask select.
//            F a power of two (G*F = 128) keeps the original xor mask (MODE_TEMPORAL); any other F in [1, 128] runs
//            MODE_TEMPORAL_ANY.
//   cross    (text conditioning, T5): queries of one sample against its <= 128 text keys, with an optional additive
//            bias per key (mask) and per (head, query row, key) (T5's relative position bias).
// head_dim 72 / 80 are not multiples of the K = 16 granule of the second product: the first 64 dims use 128B-swizzled
// tiles, dims [64,80) a second 32B-swizzled tile whose out-of-range columns TMA zero-fills.
//
// CTA = one 128-row query tile of one head, 256 threads = two warpgroups of 64 query rows each (wgmma M = 64).
//   S = Q K^T        wgmma 64 x 128 per warpgroup, both operands K-major in shared memory, fp32 in registers
//   online softmax   in registers (exp2 domain); a row's running max / sum live in the 4 threads that hold the row
//   O += P V         wgmma 64 x 64 (+ 64 x 16 head_dim tail) with P as the register A operand and V MN-major in smem
// K/V chunks are double-buffered: thread 0 refills a stage once both warpgroups have released it.  The output is
// staged dense [128][hd] over the (dead) Q tile and leaves through one TMA bulk store whose box regroups the rows
// exactly like the loads.
#include <cstdlib>
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 128;            // keys per K/V stage

enum { MODE_FULL = 0, MODE_PACKED = 1, MODE_TEMPORAL = 2, MODE_CROSS = 3, MODE_TEMPORAL_ANY = 4 };

struct AttnDev {
  int heads;
  int hd;
  int tokens;       // N
  int frames;       // F
  int group;        // PACKED: N (tokens per sequence); TEMPORAL: G = 128 / F  (power of two); TEMPORAL_ANY: floor(128 / F)
  int gshift;       // log2(group)  (PACKED, TEMPORAL)
  int k_head0, v_head0;  // index of head 0 of K / V in the (hd, heads-like, rows) view of the K/V buffer
  int kv_rows_per_batch; // CROSS: rows of the K/V buffer per sample
  int q_rows_per_batch;  // CROSS: query rows per sample (F * N)
  int chunks;       // key chunks of 128 per tile: FULL N / 128, otherwise 1
  int tiles_per_seq;  // FULL: N / 128; TEMPORAL: N / G; TEMPORAL_ANY: ceil(N / G)
  float scale_log2; // score scale * log2(e)
  const float* key_bias;  // CROSS: additive bias on the scores, fp32 [batch][128] (natural-log units, e.g. 0 / -10000), or nullptr
  const float* pos_bias;  // CROSS: additive bias fp32 [heads][128][128] per (head, query row, key), or nullptr
  int kv_valid;           // CROSS: number of valid keys per sample (<= kv_rows_per_batch)
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool TAIL>
struct AttnSmem {
  static constexpr int Q_MAIN = 0, Q_TAIL = 128 * 128;
  static constexpr int Q_BYTES = 128 * 128 + (TAIL ? 128 * 32 : 0);     // also the [128][hd] output staging tile
  static constexpr int K_MAIN = 0, K_TAIL = kChunk * 128;
  static constexpr int V_MAIN = K_TAIL + (TAIL ? kChunk * 32 : 0);
  static constexpr int V_TAIL = V_MAIN + kChunk * 128;
  static constexpr int KV_BYTES = V_TAIL + (TAIL ? kChunk * 32 : 0);
  static constexpr int STAGE0 = Q_BYTES;
  static constexpr int BARS = STAGE0 + 2 * KV_BYTES;
  static constexpr int TOTAL = BARS + 64 + 1024;
  static_assert(Q_BYTES % 1024 == 0 && KV_BYTES % 1024 == 0 && V_MAIN % 1024 == 0, "128B-swizzled tiles need 1 KiB alignment");
};

template <bool BF16, bool TAIL, int MODE>
__global__ void __launch_bounds__(kThreads, 1)
attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmQt,
            const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmKVt,
            const __grid_constant__ CUtensorMap tmO, const AttnDev p) {
  using L = AttnSmem<TAIL>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BARS);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;    // [2]
  uint64_t* kv_empty = bars + 3;   // [2]

  constexpr bool kTemporal = MODE == MODE_TEMPORAL || MODE == MODE_TEMPORAL_ANY;
  const int head = blockIdx.y, tile = blockIdx.x;
  // TMA coordinates of the tile: query rows (c2, c3), first key row kv2
  int c2, c3 = 0, kv2;
  if constexpr (kTemporal) {
    c2 = (tile % p.tiles_per_seq) * p.group;        // first token of the group
    c3 = (tile / p.tiles_per_seq) * p.frames;       // first (b, f) image
    kv2 = c2;
  } else if constexpr (MODE == MODE_FULL) {
    kv2 = (tile / p.tiles_per_seq) * p.tokens;
    c2 = kv2 + (tile % p.tiles_per_seq) * 128;
  } else if constexpr (MODE == MODE_CROSS) {
    c2 = tile * 128;
    c3 = c2 / p.q_rows_per_batch;                   // sample index (key-bias row)
    kv2 = c3 * p.kv_rows_per_batch;
  } else {
    c2 = kv2 = tile * 128;
  }
  const int nchunks = MODE == MODE_FULL ? p.chunks : 1;
  // rows of a Q / K / V tile that TMA writes (out-of-bounds elements it zero-fills count towards the transaction bytes)
  const int tile_rows = MODE == MODE_TEMPORAL_ANY ? p.group * p.frames : 128;
  const uint32_t q_bytes = MODE == MODE_TEMPORAL_ANY ? tile_rows * (128u + (TAIL ? 32u : 0u)) : uint32_t(L::Q_BYTES);
  const uint32_t kv_bytes = MODE == MODE_TEMPORAL_ANY ? 2u * q_bytes : uint32_t(L::KV_BYTES);

  auto load_kv = [&](int j) {
    uint8_t* st = smem + L::STAGE0 + (j & 1) * L::KV_BYTES;
    uint64_t* bar = kv_full + (j & 1);
    mbar_arrive_expect_tx(bar, kv_bytes);
    if constexpr (kTemporal) {
      tma_load_4d(st + L::K_MAIN, &tmKV, bar, 0, p.k_head0 + head, kv2, c3);
      tma_load_4d(st + L::V_MAIN, &tmKV, bar, 0, p.v_head0 + head, kv2, c3);
      if constexpr (TAIL) {
        tma_load_4d(st + L::K_TAIL, &tmKVt, bar, 64, p.k_head0 + head, kv2, c3);
        tma_load_4d(st + L::V_TAIL, &tmKVt, bar, 64, p.v_head0 + head, kv2, c3);
      }
    } else {
      const int row = kv2 + j * kChunk;
      tma_load_3d(st + L::K_MAIN, &tmKV, bar, 0, p.k_head0 + head, row);
      tma_load_3d(st + L::V_MAIN, &tmKV, bar, 0, p.v_head0 + head, row);
      if constexpr (TAIL) {
        tma_load_3d(st + L::K_TAIL, &tmKVt, bar, 64, p.k_head0 + head, row);
        tma_load_3d(st + L::V_TAIL, &tmKVt, bar, 64, p.v_head0 + head, row);
      }
    }
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    tma_prefetch_desc(&tmO);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(kv_full + i, 1);
      mbar_init(kv_empty + i, kThreads);
    }
    fence_mbar_init();
  }
  if constexpr (MODE == MODE_TEMPORAL_ANY) {
    // V rows [tile_rows, 128) of the (only) stage are never loaded; zero them so that P = 0 multiplies zeros, not stale
    // bits.  Whole rows: a row stays a row under both the 128B and the 32B swizzle.  TMA writes rows [0, tile_rows) only.
    uint8_t* st = smem + L::STAGE0;
    const int main_chunks = (128 - tile_rows) * 8, n = main_chunks + (TAIL ? (128 - tile_rows) * 2 : 0);
    for (int i = threadIdx.x; i < n; i += kThreads) {
      uint8_t* dst = i < main_chunks ? st + L::V_MAIN + tile_rows * 128 + i * 16 : st + L::V_TAIL + tile_rows * 32 + (i - main_chunks) * 16;
      *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async_smem();     // the zeros are read by wgmma (async proxy) after the barrier below
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();   // qkv (written by the preceding GEMM) is visible from here
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(q_full, q_bytes);
    if constexpr (kTemporal) {
      tma_load_4d(smem + L::Q_MAIN, &tmQ, q_full, 0, head, c2, c3);
      if constexpr (TAIL) tma_load_4d(smem + L::Q_TAIL, &tmQt, q_full, 64, head, c2, c3);
    } else {
      tma_load_3d(smem + L::Q_MAIN, &tmQ, q_full, 0, head, c2);
      if constexpr (TAIL) tma_load_3d(smem + L::Q_TAIL, &tmQt, q_full, 64, head, c2);
    }
    load_kv(0);
    if (nchunks > 1) load_kv(1);
  }

  const int wg = threadIdx.x >> 7;
  const int te = threadIdx.x & 127;
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, cq = lane & 3;
  const int rA = wg * 64 + (te >> 5) * 16 + g;    // tile rows of this thread: rA and rA + 8
  const int rows[2] = {rA, rA + 8};
  // TEMPORAL_ANY: bit 2*j8 + e of kmask[h] says whether key column c = 8*j8 + 2*cq + e is valid for row rows[h]
  // (c < G*F and c % G == rows[h] % G).  Residues are stepped by 8 % G per j8 instead of divided per score.
  uint32_t kmask[2] = {0u, 0u};
  if constexpr (MODE == MODE_TEMPORAL_ANY) {
    const int G = p.group, step = 8 % G;
    const int rres[2] = {rows[0] % G, rows[1] % G};
    int cres[2] = {(2 * cq) % G, (2 * cq + 1) % G};
#pragma unroll
    for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool in_tile = 8 * j8 + 2 * cq + e < tile_rows;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          kmask[h] |= (in_tile && cres[e] == rres[h]) ? 1u << (2 * j8 + e) : 0u;
        cres[e] += step;
        cres[e] -= cres[e] >= G ? G : 0;
      }
    }
  }

  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32], ot[8];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ot[i] = 0.f;

  const uint32_t q_base = smem_u32(smem);
  const uint64_t dq = gmma_desc(q_base + L::Q_MAIN + wg * 64 * 128, 16, 1024, GMMA_LAYOUT_SW128);
  const uint64_t dqt = gmma_desc(q_base + L::Q_TAIL + wg * 64 * 32, 16, 256, GMMA_LAYOUT_SW32);
  const float* prow[2] = {nullptr, nullptr};       // CROSS: (head, query row)'s 128 relative-position biases
  const float* kbias = nullptr;                   // CROSS: this sample's 128 key biases
  if constexpr (MODE == MODE_CROSS) {
    if (p.pos_bias)
      for (int h = 0; h < 2; ++h) prow[h] = p.pos_bias + (static_cast<size_t>(head) * 128 + rows[h]) * 128;
    if (p.key_bias) kbias = p.key_bias + static_cast<size_t>(c3) * 128;
  }
  constexpr float kLog2e = 1.4426950408889634f;

  mbar_wait(q_full, 0);
  for (int j = 0; j < nchunks; ++j) {
    const int sidx = j & 1;
    const uint32_t st = q_base + L::STAGE0 + sidx * L::KV_BYTES;
    mbar_wait(kv_full + sidx, (j >> 1) & 1);

    // ---- S = Q K^T (64 x 128 per warpgroup)
    float s[64];
    wgmma_fence();
    {
      const uint64_t dk = gmma_desc(st + L::K_MAIN, 16, 1024, GMMA_LAYOUT_SW128);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        WgmmaSS<128, 0, 0, BF16>::mma(s, gmma_desc_advance(dq, k * 32), gmma_desc_advance(dk, k * 32), k > 0 ? 1u : 0u);
      if constexpr (TAIL)
        WgmmaSS<128, 0, 0, BF16>::mma(s, dqt, gmma_desc(st + L::K_TAIL, 16, 256, GMMA_LAYOUT_SW32), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- online softmax (exp2 domain): element (h, j8, e) is row rows[h], key column 8*j8 + 2*cq + e of the chunk
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rows[h];
      float mx = -INFINITY;
#pragma unroll
      for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j8 + 2 * cq + e;
          float x = s[4 * j8 + 2 * h + e] * p.scale_log2;
          bool valid = true;
          if constexpr (MODE == MODE_PACKED) valid = (r >> p.gshift) == (c >> p.gshift);
          if constexpr (MODE == MODE_TEMPORAL) valid = ((r ^ c) & ((1 << p.gshift) - 1)) == 0;
          if constexpr (MODE == MODE_TEMPORAL_ANY) valid = (kmask[h] >> (2 * j8 + e)) & 1u;
          if constexpr (MODE == MODE_CROSS) {
            valid = c < p.kv_valid;
            if (kbias) x = fmaf(__ldg(kbias + c), kLog2e, x);
            if (prow[h]) x = fmaf(__ldg(prow[h] + c), kLog2e, x);
          }
          x = valid ? x : -INFINITY;
          s[4 * j8 + 2 * h + e] = x;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);
      const float shift = m_new == -INFINITY ? 0.f : m_new;   // a row with no valid key yet keeps everything at zero
      alpha[h] = ex2(m[h] - shift);
      m[h] = m_new;
      float part[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j8 = 0; j8 < 16; ++j8) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = ex2(s[4 * j8 + 2 * h + e] - shift);
          s[4 * j8 + 2 * h + e] = v;
          part[(j8 & 1) * 2 + e] += v;
        }
      }
      l[h] = fmaf(l[h], alpha[h], (part[0] + part[1]) + (part[2] + part[3]));
    }
#pragma unroll
    for (int j8 = 0; j8 < 8; ++j8) {
      o[4 * j8 + 0] *= alpha[0]; o[4 * j8 + 1] *= alpha[0];
      o[4 * j8 + 2] *= alpha[1]; o[4 * j8 + 3] *= alpha[1];
    }
#pragma unroll
    for (int j8 = 0; j8 < 2; ++j8) {
      ot[4 * j8 + 0] *= alpha[0]; ot[4 * j8 + 1] *= alpha[0];
      ot[4 * j8 + 2] *= alpha[1]; ot[4 * j8 + 3] *= alpha[1];
    }

    // ---- O += P V: P (16-bit) as the register A operand, k-step kk = keys [16kk, 16kk + 16)
    wgmma_fence();
    {
      const uint64_t dv = gmma_desc(st + L::V_MAIN, 8192, 1024, GMMA_LAYOUT_SW128);
      const uint64_t dvt = gmma_desc(st + L::V_TAIL, 512, 256, GMMA_LAYOUT_SW32);
#pragma unroll
      for (int kk = 0; kk < kChunk / 16; ++kk) {
        uint32_t a[4];
        a[0] = pack2<BF16>(s[8 * kk + 0], s[8 * kk + 1]);
        a[1] = pack2<BF16>(s[8 * kk + 2], s[8 * kk + 3]);
        a[2] = pack2<BF16>(s[8 * kk + 4], s[8 * kk + 5]);
        a[3] = pack2<BF16>(s[8 * kk + 6], s[8 * kk + 7]);
        WgmmaRS<64, 1, BF16>::mma(o, a, gmma_desc_advance(dv, kk * 16 * 128), 1u);
        if constexpr (TAIL) WgmmaRS<16, 1, BF16>::mma(ot, a, gmma_desc_advance(dvt, kk * 16 * 32), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(ot);
    mbar_arrive(kv_empty + sidx);
    if (threadIdx.x == 0 && j + 2 < nchunks) {
      mbar_wait(kv_empty + sidx, (j >> 1) & 1);   // both warpgroups are done with this stage
      load_kv(j + 2);
    }
  }

  // ---- epilogue: O / l -> 16-bit -> dense [128][hd] staging tile over Q (dead once both warpgroups' S are done)
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float t = l[h];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    inv[h] = 1.0f / t;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  uint8_t* stage_out = smem;
  const int row_bytes = p.hd * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint8_t* drow = stage_out + rows[h] * row_bytes;
#pragma unroll
    for (int j8 = 0; j8 < 8; ++j8)
      *reinterpret_cast<uint32_t*>(drow + (8 * j8 + 2 * cq) * 2) =
          pack2<BF16>(o[4 * j8 + 2 * h] * inv[h], o[4 * j8 + 2 * h + 1] * inv[h]);
    if constexpr (TAIL) {
#pragma unroll
      for (int j8 = 0; j8 < 2; ++j8) {
        const int col = 64 + 8 * j8 + 2 * cq;
        if (col < p.hd)
          *reinterpret_cast<uint32_t*>(drow + col * 2) = pack2<BF16>(ot[4 * j8 + 2 * h] * inv[h], ot[4 * j8 + 2 * h + 1] * inv[h]);
      }
    }
  }
  fence_proxy_async_smem();       // the staging tile is read by the TMA engine
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (threadIdx.x == 0) {
    if constexpr (kTemporal) tma_store_4d(&tmO, stage_out, 0, head, c2, c3);
    else tma_store_3d(&tmO, stage_out, 0, head, c2);
    tma_store_commit();
    tma_store_wait_all<0>();
  }
}

template <bool BF16, bool TAIL, int MODE>
int launch_mode(const CUtensorMap* m, const AttnDev& p, dim3 grid, cudaStream_t stream) {
  auto kern = attn_kernel<BF16, TAIL, MODE>;
  constexpr int smem_bytes = AttnSmem<TAIL>::TOTAL;
  B200_SET_SMEM_ONCE(kern, smem_bytes);
  B200_CHECK_CUDA(launch_pdl(kern, grid, dim3(kThreads), static_cast<size_t>(smem_bytes), stream, m[0], m[1], m[2], m[3], m[4], p));
  return B200_OK;
}

template <bool BF16, bool TAIL>
int launch_tail(int mode, const CUtensorMap* m, const AttnDev& p, dim3 grid, cudaStream_t s) {
  switch (mode) {
    case MODE_FULL: return launch_mode<BF16, TAIL, MODE_FULL>(m, p, grid, s);
    case MODE_PACKED: return launch_mode<BF16, TAIL, MODE_PACKED>(m, p, grid, s);
    case MODE_CROSS: return launch_mode<BF16, TAIL, MODE_CROSS>(m, p, grid, s);
    case MODE_TEMPORAL_ANY: return launch_mode<BF16, TAIL, MODE_TEMPORAL_ANY>(m, p, grid, s);
    default: return launch_mode<BF16, TAIL, MODE_TEMPORAL>(m, p, grid, s);
  }
}

int launch_any(int mode, int bf16, bool tail, const CUtensorMap* m, const AttnDev& p, dim3 grid, cudaStream_t s) {
  if (bf16) return tail ? launch_tail<true, true>(mode, m, p, grid, s) : launch_tail<true, false>(mode, m, p, grid, s);
  return tail ? launch_tail<false, true>(mode, m, p, grid, s) : launch_tail<false, false>(mode, m, p, grid, s);
}

}  // namespace

bool attention_spatial_len_ok(int tokens) {
  return tokens > 0 && (tokens >= 128 ? tokens == 128 || tokens % 256 == 0 : 128 % tokens == 0);
}

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  B200_REQUIRE(a.batch > 0 && a.frames > 0 && a.tokens > 0 && a.heads > 0, B200_ERR_SHAPE, "attention: bad shape");
  B200_REQUIRE(a.head_dim == 64 || a.head_dim == 72 || a.head_dim == 80, B200_ERR_UNSUPPORTED,
               "attention: head_dim %d unsupported (64, 72, 80)", a.head_dim);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(a.qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 15) == 0,
               B200_ERR_ALIGN, "attention: qkv/out must be 16-byte aligned");
  B200_TRY(check_arch());
  const int H = a.heads, hd = a.head_dim, D = H * hd;
  const long long T = static_cast<long long>(a.batch) * a.frames * a.tokens;
  const bool tail = hd > 64;

  AttnDev p{};
  p.heads = H;
  p.hd = hd;
  p.tokens = a.tokens;
  p.frames = a.frames;
  p.scale_log2 = (1.0f / sqrtf(static_cast<float>(hd))) * 1.4426950408889634f;
  p.group = 1;
  p.gshift = 0;
  p.k_head0 = H;
  p.v_head0 = 2 * H;
  p.chunks = 1;
  auto ilog2 = [](int v) { int s = 0; while ((1 << s) < v) ++s; return s; };

  CUtensorMap maps[5];
  int mode;
  dim3 grid;
  if (!a.temporal) {
    if (a.tokens >= 128) {
      B200_REQUIRE(attention_spatial_len_ok(a.tokens), B200_ERR_UNSUPPORTED,
                   "attention: spatial sequence length %d unsupported (<=64 power of two, 128, multiples of 256)", a.tokens);
      mode = MODE_FULL;
      p.chunks = a.tokens / kChunk;
      p.tiles_per_seq = a.tokens / 128;
      grid = dim3(static_cast<unsigned>(a.batch * a.frames * p.tiles_per_seq), H);
    } else {
      B200_REQUIRE(attention_spatial_len_ok(a.tokens), B200_ERR_UNSUPPORTED, "attention: spatial sequence length %d must divide 128", a.tokens);
      mode = MODE_PACKED;
      p.group = a.tokens;
      p.gshift = ilog2(a.tokens);
      p.tiles_per_seq = 1;
      grid = dim3(static_cast<unsigned>((T + 127) / 128), H);
    }
    const uint64_t dims[3] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(3 * H), static_cast<uint64_t>(T)};
    const uint64_t str[2] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(3 * D) * 2};
    const uint32_t box[3] = {64, 1, 128}, boxt[3] = {16, 1, 128};
    B200_TRY(make_tmap_16bit(&maps[0], a.qkv, 3, dims, str, box, TMAP_SW_128));
    maps[2] = maps[0];
    if (tail) {
      B200_TRY(make_tmap_16bit(&maps[1], a.qkv, 3, dims, str, boxt, TMAP_SW_32));
      maps[3] = maps[1];
    } else {
      maps[1] = maps[0];
      maps[3] = maps[0];
    }
    {   // output tile store: dense [128][hd] rows of the staging tile -> rows (b, f, n) of out, columns of this head
      const uint64_t odims[3] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(H), static_cast<uint64_t>(T)};
      const uint64_t ostr[2] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(D) * 2};
      const uint32_t obox[3] = {static_cast<uint32_t>(hd), 1, 128};
      B200_TRY(make_tmap_16bit(&maps[4], a.out, 3, odims, ostr, obox, TMAP_SW_NONE));
    }
  } else {
    const int F = a.frames;
    B200_REQUIRE(F >= 1 && F <= 128, B200_ERR_UNSUPPORTED, "attention: temporal length %d unsupported (1..128)", F);
    const int G = 128 / F;
    // G * F == 128 exactly when F is a power of two: the full tile keeps the xor mask and compile-time byte counts
    mode = G * F == 128 ? MODE_TEMPORAL : MODE_TEMPORAL_ANY;
    p.group = G;
    p.gshift = ilog2(G);
    p.tiles_per_seq = (a.tokens + G - 1) / G;
    grid = dim3(static_cast<unsigned>(a.batch * p.tiles_per_seq), H);
    const uint64_t dims[4] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(3 * H), static_cast<uint64_t>(a.tokens),
                              static_cast<uint64_t>(a.batch) * F};
    const uint64_t str[3] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(3 * D) * 2,
                             static_cast<uint64_t>(3 * D) * 2 * a.tokens};
    const uint32_t box[4] = {64, 1, static_cast<uint32_t>(G), static_cast<uint32_t>(F)};
    const uint32_t boxt[4] = {16, 1, static_cast<uint32_t>(G), static_cast<uint32_t>(F)};
    B200_TRY(make_tmap_16bit(&maps[0], a.qkv, 4, dims, str, box, TMAP_SW_128));
    maps[2] = maps[0];
    if (tail) {
      B200_TRY(make_tmap_16bit(&maps[1], a.qkv, 4, dims, str, boxt, TMAP_SW_32));
      maps[3] = maps[1];
    } else {
      maps[1] = maps[0];
      maps[3] = maps[0];
    }
    {   // output store with the same (token group) x (frames) box as the loads: tile row f*G + g -> out row (b*F + f)*N + n0 + g
      const uint64_t odims[4] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(H), static_cast<uint64_t>(a.tokens),
                                 static_cast<uint64_t>(a.batch) * F};
      const uint64_t ostr[3] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(D) * 2, static_cast<uint64_t>(D) * 2 * a.tokens};
      const uint32_t obox[4] = {static_cast<uint32_t>(hd), 1, static_cast<uint32_t>(G), static_cast<uint32_t>(F)};
      B200_TRY(make_tmap_16bit(&maps[4], a.out, 4, odims, ostr, obox, TMAP_SW_NONE));
    }
  }
  return launch_any(mode, a.bf16, tail, maps, p, grid, stream);
}

int launch_cross_attention(const CrossAttnArgs& a, cudaStream_t stream) {
  B200_REQUIRE(a.batch > 0 && a.q_rows_per_batch > 0 && a.heads > 0, B200_ERR_SHAPE, "cross attention: bad shape");
  B200_REQUIRE(a.head_dim == 64 || a.head_dim == 72 || a.head_dim == 80, B200_ERR_UNSUPPORTED,
               "cross attention: head_dim %d unsupported (64, 72, 80)", a.head_dim);
  B200_REQUIRE(a.kv_len >= 1 && a.kv_len <= 128, B200_ERR_UNSUPPORTED, "cross attention: %d keys per sample (1..128 built)", a.kv_len);
  B200_REQUIRE(a.q_rows_per_batch % 128 == 0, B200_ERR_UNSUPPORTED, "cross attention: query rows per sample %d must be a multiple of 128",
               a.q_rows_per_batch);
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.kv) | reinterpret_cast<uintptr_t>(a.out)) & 15) == 0,
               B200_ERR_ALIGN, "cross attention: q/kv/out must be 16-byte aligned");
  B200_TRY(check_arch());
  const int H = a.heads, hd = a.head_dim, D = H * hd;
  const long long T = static_cast<long long>(a.batch) * a.q_rows_per_batch;
  const long long R = static_cast<long long>(a.batch) * (a.kv_batch_rows > 0 ? a.kv_batch_rows : a.kv_len);
  const bool tail = hd > 64;
  AttnDev p{};
  p.heads = H; p.hd = hd;
  p.tokens = a.q_rows_per_batch; p.frames = 1; p.group = 1; p.gshift = 0; p.chunks = 1; p.tiles_per_seq = 1;
  p.scale_log2 = (a.scale > 0.f ? a.scale : 1.0f / sqrtf(static_cast<float>(hd))) * 1.4426950408889634f;
  p.k_head0 = 0; p.v_head0 = H; p.q_rows_per_batch = a.q_rows_per_batch;
  p.kv_rows_per_batch = a.kv_batch_rows > 0 ? a.kv_batch_rows : a.kv_len;
  p.kv_valid = a.kv_len;
  B200_REQUIRE(p.kv_rows_per_batch >= a.kv_len, B200_ERR_SHAPE, "cross attention: kv_batch_rows %d < kv_len %d", a.kv_batch_rows, a.kv_len);
  B200_REQUIRE(!a.pos_bias || (a.q_rows_per_batch == 128 && (reinterpret_cast<uintptr_t>(a.pos_bias) & 15) == 0), B200_ERR_UNSUPPORTED,
               "cross attention: pos_bias needs 128 query rows per sample (one tile) and 16-byte alignment");
  p.pos_bias = a.pos_bias;
  B200_REQUIRE(!a.key_bias || (reinterpret_cast<uintptr_t>(a.key_bias) & 15) == 0, B200_ERR_ALIGN, "cross attention: key_bias must be 16-byte aligned");
  p.key_bias = a.key_bias;
  CUtensorMap maps[5];
  const uint64_t qdims[3] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(H), static_cast<uint64_t>(T)};
  const uint64_t qstr[2] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(a.q_row_stride) * 2};
  const uint64_t kdims[3] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(2 * H), static_cast<uint64_t>(R)};
  const uint64_t kstr[2] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(a.kv_row_stride) * 2};
  const uint32_t box[3] = {64, 1, 128}, boxt[3] = {16, 1, 128};
  B200_REQUIRE(a.q_row_stride >= D && a.kv_row_stride >= 2 * D && a.q_row_stride % 8 == 0 && a.kv_row_stride % 8 == 0, B200_ERR_SHAPE, "cross attention: bad row strides");
  B200_TRY(make_tmap_16bit(&maps[0], a.q, 3, qdims, qstr, box, TMAP_SW_128));
  B200_TRY(make_tmap_16bit(&maps[2], a.kv, 3, kdims, kstr, box, TMAP_SW_128));
  if (tail) {
    B200_TRY(make_tmap_16bit(&maps[1], a.q, 3, qdims, qstr, boxt, TMAP_SW_32));
    B200_TRY(make_tmap_16bit(&maps[3], a.kv, 3, kdims, kstr, boxt, TMAP_SW_32));
  } else {
    maps[1] = maps[0];
    maps[3] = maps[2];
  }
  {
    const uint64_t odims[3] = {static_cast<uint64_t>(hd), static_cast<uint64_t>(H), static_cast<uint64_t>(T)};
    const uint64_t ostr[2] = {static_cast<uint64_t>(hd) * 2, static_cast<uint64_t>(D) * 2};
    const uint32_t obox[3] = {static_cast<uint32_t>(hd), 1, 128};
    B200_TRY(make_tmap_16bit(&maps[4], a.out, 3, odims, ostr, obox, TMAP_SW_NONE));
  }
  const dim3 grid(static_cast<unsigned>(T / 128), H);
  return launch_any(MODE_CROSS, a.bf16, tail, maps, p, grid, stream);
}

}  // namespace b200
