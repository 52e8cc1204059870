// wgmma GEMM with fused epilogues: out = epi(A[M,K] @ W[N,K]^T + bias)
//
// Replaces the nn.Linear calls inside a Latte TransformerBlock (reference models/latte.py:50 qkv, :75 proj,
// timm Mlp fc1/fc2 reached from :171,:180) together with the elementwise work that follows them:
//   EPI_BIAS           qkv projection               -> 16-bit [M,N]
//   EPI_BIAS_GELU      fc1 + GELU(tanh)             -> 16-bit [M,N]            (latte.py:169)
//   EPI_GATE_RESIDUAL  proj / fc2 + adaLN gate + residual add, fp32 residual stream in place
//                      (latte.py:179-180), optionally + temp_embed rows        (latte.py:357-358)
//
// Hopper structure: CTAs run as PAIRS (cluster of 2).  A pair owns a 256 x BN pair-tile: each CTA multiplies its own 128 A
// rows, and each fetches only HALF of the W tile and multicasts it into both CTAs' shared memory (TMA .multicast::cluster),
// so every W byte crosses L2 -> SM once per pair.
// 384 threads, warp-specialized; setmaxnreg moves registers from the producer (40 per thread) to the consumers (232):
//   warpgroup 0     the TMA producer, one thread: A tile 128x64 and the W half (BN/2)x64 (128B-swizzled) per pipeline
//                   stage; a stage is full when this CTA's A bytes and BOTH W halves have landed on its "full" barrier.
//                   It waits only on "empty" and keeps every stage in flight, through the consumers' epilogues.
//   warpgroups 1-2  the consumers: wgmma (64 x BN x 16, fp32 accumulators in registers), one 64-row half of the tile each,
//                   then the epilogue; they wait only on "full", and a stage is released with one arrival per warpgroup
//                   on the "empty" barriers of BOTH CTAs (the peer's next multicast writes into it)
//
// Epilogue: the consumers never write global memory themselves.  Each warpgroup moves its 64 rows of the tile, one column
// chunk at a time, into one of its two 64-row x 128-byte staging buffers (128B-swizzled, the layout of a SW128 tensor map),
// and one thread hands the chunk to TMA; the warpgroup goes straight on to the next chunk and then the next tile's MMAs
// while the bytes drain.  TMA clips rows past M and columns past N.
//   16-bit outputs:  64-column chunks, stmatrix into the buffer, cp.async.bulk.tensor store
//   residual:        32-column fp32 chunks of the increment gate * (acc + bias) (+ row_add); x is never loaded: a
//                    cp.reduce.async.bulk.tensor .add folds the chunk into the fp32 residual stream in L2, once per GEMM --
//                    or, for the stream-K tiles of the last waves, once per K segment in k order (TileSched below).
#include <cstdio>
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

#include <cstdlib>

namespace b200 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 16-bit = one 128-byte swizzle row
constexpr int kThreads = 384;   // warpgroup 0: TMA producer; warpgroups 1-2: MMA + epilogue
// per-thread registers after setmaxnreg.  The kernel is compiled for 65536 / 384 -> 168; the producer's release pays for
// the consumers' raise exactly: 128 * (168 - 40) = 256 * (232 - 168), and (40 + 2 * 232) * 128 = 64,512 fit the SM's 65,536.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

// epilogue staging buffer: 64 rows x 128 bytes (32 fp32 or 64 16-bit columns), two per consumer warpgroup
constexpr int kEpiBufBytes = 64 * 128;

template <int BN, int EPI>
struct Cfg {
  static constexpr int BLOCK_N = BN;
  static constexpr bool RESID = EPI == B200_EPI_GATE_RESIDUAL;
  static constexpr bool TWO_OUT = EPI == B200_EPI_BIAS_GELU_BOTH;   // out16 and out16b
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;                       // the whole W tile (both CTAs' halves)
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_BYTES = 2 * 2 * kEpiBufBytes;            // 2 consumer warpgroups x 2 buffers = 32 KiB
  static constexpr int BAR_BYTES = 256;
  static constexpr int STAGES_FIT = (232448 - EPI_BYTES - BAR_BYTES - 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;   // BN 256: 4, 192: 4, 128: 6
  static constexpr int EPI_OFF = STAGES * STAGE_BYTES;             // 1 KiB aligned: the buffers keep the swizzle phase
  static constexpr int BAR_OFF = EPI_OFF + EPI_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + BAR_BYTES + 1024;    // +1024: manual 1 KiB alignment of the base
  static_assert(STAGE_BYTES % 1024 == 0, "stage must keep 1 KiB alignment");
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
  static_assert(2 * STAGES <= BAR_BYTES / 8, "barrier area too small");
  static_assert(BN % 64 == 0, "the 16-bit epilogue works in 64-column chunks");
};

struct GemmDev {
  int M, N, K;
  int num_m, num_n;
  const float* bias;
  void* out16;
  const float* gate;
  long long gate_bs;
  int rows_per_batch;
  const float* row_add;
  int row_add_div, row_add_period;
  const uint16_t* add16;
  uint16_t* out16b;    // EPI_BIAS_GELU_BOTH: second output, gelu(out16)
  // implicit-GEMM convolution: see GemmArgs
  int conv_taps, conv_cblk, conv_h, conv_w, conv_bw, conv_bh;
  int conv_dx[9], conv_dy[9], conv_dz[9];
  float* resid; // EPI_GATE_RESIDUAL: [M, N] fp32 residual stream, updated in place
  int streamk;  // residual epilogue only: split the last partial wave of tiles along K across all pairs (see TileSched)
  // stream-K ordering flags (caller's workspace), one per (streamed tile, CTA rank, epilogue warpgroup): "k-blocks of the
  // tile already added into x".  All zero between launches: the segment that completes a tile resets its flag, so the
  // protocol holds no host-side state and a captured CUDA graph replays it unchanged.
  unsigned long long* sk_flags;
};

__device__ __forceinline__ void flag_release(unsigned long long* f, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(f), "l"(v) : "memory");
}
__device__ __forceinline__ void flag_wait(const unsigned long long* f, unsigned long long want) {
  const long long t0 = clock64();
  while (true) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
    if (v == want) return;
    if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s: a protocol bug must not hang the GPU (no printf: see mbar_wait)
    __nanosleep(64);
  }
}

// Work schedule of one CTA pair.  Data-parallel part: pair k owns tiles k, k + P, ... for the `full_waves` complete waves.
// Stream-K part (residual epilogue only, where partial sums can be reduce-added into x): the tiles of the last, partial
// wave (and of the full wave before it) are flattened into (tile, k-block) units and every pair takes an equal contiguous share, so no SM idles while a
// few pairs finish a whole extra tile.  A segment is (tile, [kb0, kb1)); bias / row_add go with the segment that has kb0 = 0.
// The partial sums of a tile are added into x in k order (a global flag per tile carries "k-blocks added so far"; the
// epilogue of a kb0 > 0 segment waits for flag == kb0), so the result is bit-reproducible although several pairs add to it.
struct TileSched {
  int pair, P, num_tiles, num_kb, full_waves, wave;
  long long u, u_end;
  __host__ __device__ TileSched(int pair_, int P_, int num_tiles_, int num_kb_, bool streamk)
      : pair(pair_), P(P_), num_tiles(num_tiles_), num_kb(num_kb_), wave(0) {
    if (streamk) {
      // stream the partial wave TOGETHER WITH the last full wave: every pair's share is then at least one tile long, so
      // a tile is cut at most once (two segments) and the ordered adds never form a chain of waiting pairs
      full_waves = num_tiles / P;
      if (full_waves > 0) --full_waves;
      const long long units = static_cast<long long>(num_tiles - full_waves * P) * num_kb;
      u = units * pair / P;
      u_end = units * (pair + 1) / P;
    } else {
      full_waves = (num_tiles + P - 1) / P;
      u = u_end = 0;
    }
  }
  __host__ __device__ bool next(int& tile, int& kb0, int& kb1) {
    if (wave < full_waves) {
      tile = wave * P + pair;
      ++wave;
      kb0 = 0;
      kb1 = num_kb;
      return tile < num_tiles;     // only the last data-parallel wave can run past the end
    }
    if (u >= u_end) return false;
    // streamed share, walked from its END: the segment that starts a tile (kb0 = 0) is done first and the one that
    // continues a tile begun by the previous pair (kb0 > 0) last, by which time that pair's part has long been added
    const int t = static_cast<int>((u_end - 1) / num_kb);
    const long long t0 = static_cast<long long>(t) * num_kb;
    kb1 = static_cast<int>(u_end - t0);
    kb0 = u > t0 ? static_cast<int>(u - t0) : 0;
    tile = full_waves * P + t;
    u_end = t0 + kb0;
    return true;
  }
};

// the residual epilogue's increment gate * (acc + bias) (+ row_add), added to x by the caller; rounded step by step (no FMA
// contraction) so that every path through the epilogue produces the same bits
__device__ __forceinline__ float resid_delta(float acc, float b, float gt, float ra, bool has_ra) {
  const float dv = __fmul_rn(gt, __fadd_rn(acc, b));
  return has_ra ? __fadd_rn(dv, ra) : dv;
}

// named barrier of consumer warpgroup wg (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void epi_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5 x (1 + tanh(u)),  u = sqrt(2/pi) (x + 0.044715 x^3).  ONE MUFU op per element (tanh.approx, rel. error 2^-11,
  // the same size as the 16-bit rounding of the result) instead of ex2 + rcp: the 16/clk/SM MUFU pipe is the fc1
  // epilogue's narrowest resource.
  const float u = 0.7978845608028654f * fmaf(0.044715f * x * x, x, x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}

// ----------------------------------------------------------------------------- the pieces both GEMM kernels are made of
// gemm_kernel and fp8_linear_kernel share the structure described at the top of this file through the code below: the
// prologue, the pair-tile geometry, the TMA producer loop, the consumers' stage bookkeeping and the 16-bit output
// epilogue.  What each kernel loads per stage, how it multiplies a k-block and how it computes an output value are its own.

// One CTA's operand pipeline in the Cfg layout: STAGES slots, each with a "full" and an "empty" barrier.
template <class C>
struct Pipeline {
  uint8_t* smem;     // dynamic shared memory, 1 KiB aligned: the 128B swizzle's period
  uint64_t* full;    // this CTA's expect_tx arrival; the bytes of A and of both W halves complete it
  uint64_t* empty;   // one arrival per consumer warpgroup of BOTH CTAs (each W half lands in both)
  __device__ __forceinline__ uint8_t* slot(int stage) const { return smem + stage * C::STAGE_BYTES; }
};

// Thread 0 prefetches the tensor maps and initialises the barriers.  The cluster barrier has both CTAs' barriers
// initialised before any multicast / remote arrival can target them; then the next kernel may begin its prologue as SMs
// drain (PDL).
template <class C, class... Maps>
__device__ __forceinline__ Pipeline<C> gemm_prologue(const Maps*... maps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  const Pipeline<C> pl{smem, bars, bars + C::STAGES};
  if (threadIdx.x == 0) {
    (tma_prefetch_desc(maps), ...);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&pl.full[i], 1);
      mbar_init(&pl.empty[i], 4);
    }
    fence_mbar_init();
  }
  cluster_sync_all();
  pdl_launch_dependents();
  return pl;
}

// Pair-tile geometry: cluster k owns pair-tiles k, k + #clusters, ... (TileSched); a pair-tile is two M-adjacent 128-row
// tiles of one BN-wide column, and this CTA takes row-tile m_blk = 2 * pair_m + rank (it may lie past M: zero-filled
// loads, clipped stores).  Each CTA fetches half of the W tile, rows w_row0 .. w_row0 + BN/2, and multicasts it to both.
template <int BN>
struct PairTiles {
  const GemmDev& p;
  uint32_t rank;
  int num_tiles, my_pair, num_pairs;
  __device__ __forceinline__ explicit PairTiles(const GemmDev& p_)
      : p(p_), rank(cluster_ctarank()), num_tiles((p_.num_m + 1) / 2 * p_.num_n), my_pair(blockIdx.x >> 1),
        num_pairs(gridDim.x >> 1) {}
  __device__ __forceinline__ TileSched sched(int num_kb, bool streamk) const {
    return TileSched(my_pair, num_pairs, num_tiles, num_kb, streamk);
  }
  __device__ __forceinline__ int m_blk(int tile) const { return 2 * (tile / p.num_n) + static_cast<int>(rank); }
  __device__ __forceinline__ int n0(int tile) const { return (tile % p.num_n) * BN; }
  __device__ __forceinline__ int w_row0(int tile) const { return n0(tile) + static_cast<int>(rank) * (BN / 2); }
};

// The TMA producer: warpgroup 0 hands its registers to the consumers, and one thread walks this CTA's k-block sequence.
// Load q goes to slot q % STAGES; it is issued as soon as the slot's previous contents (load q - STAGES) have been released
// by both consumer warpgroups of both CTAs, so all STAGES slots stay in flight, across tile boundaries and through the
// consumers' epilogues.  The producer waits on nothing but `empty`.  load(slot, bar, m_blk, w_row0, kb) issues k-block
// kb's TMA loads into the slot: this CTA's A tile and its W half, multicast; together they complete STAGE_BYTES on `bar`.
template <class C, class Load>
__device__ __forceinline__ void produce(const Pipeline<C>& pl, const PairTiles<C::BLOCK_N>& pt, int num_kb, bool streamk,
                                        Load load) {
  setmaxnreg_dec<kProducerRegs>();
  if (threadIdx.x == 0) {
    pdl_wait();                             // operands: visible from here
    TileSched sched = pt.sched(num_kb, streamk);
    int stage = 0;
    uint32_t phase = 0;
    int tile, kb0, kb1;
    while (sched.next(tile, kb0, kb1)) {
      const int m_blk = pt.m_blk(tile), w_row0 = pt.w_row0(tile);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&pl.empty[stage], phase ^ 1);  // both CTAs' consumer warpgroups are done with the slot
        mbar_arrive_expect_tx(&pl.full[stage], C::STAGE_BYTES);
        load(pl.slot(stage), &pl.full[stage], m_blk, w_row0, kb);
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
    }
  }
  __syncwarp();                             // warp 0 reconverges before the cluster barrier
}

// A consumer thread: warpgroups 1-2, one 64-row half of the tile each, after raising their register budget.
// Accumulator fragment: thread (w4, g, cq) holds rows lr0 = 16*w4 + g and lr0 + 8 of its warpgroup's 64, columns
// 8j + 2cq + {0,1}: acc[4j + 2h + {0,1}] for row lr0 + 8h.
// Stages: wait() returns the next one's shared address once it is full.  After wgmma_wait<1>, release_prev() frees the
// slot of the k-block before in both CTAs (the peer's next multicast writes into it); after the tile's wgmma_wait<0>,
// release_last() frees the tile's last slot.
// Staging buffers: warpgroup wg owns epi buffers 2 wg and 2 wg + 1; chunk i of its output uses buffer i % 2 (ep counts).
template <class C>
struct Consumer {
  Pipeline<C> pl;
  int wg, te, lane, w4, g, cq, lr0;
  uint32_t empty_peer;
  uint8_t* epi;
  int stage = 0, prev = -1, ep = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ Consumer(const Pipeline<C>& pl_, uint32_t rank, int wg_) : pl(pl_), wg(wg_) {
    setmaxnreg_inc<kConsumerRegs>();
    pdl_wait();                               // bias / scales / side inputs / residual stream: visible from here
    lane = threadIdx.x & 31;
    te = threadIdx.x & 127;
    w4 = te >> 5, g = lane >> 2, cq = lane & 3;
    lr0 = w4 * 16 + g;
    empty_peer = mapa_u32(&pl.empty[0], rank ^ 1u);
    epi = pl.smem + C::EPI_OFF;
  }
  __device__ __forceinline__ uint32_t wait() {
    mbar_wait(&pl.full[stage], phase);
    return smem_u32(pl.slot(stage));
  }
  __device__ __forceinline__ void release_prev() {
    if (prev >= 0 && te == 0) {
      mbar_arrive(&pl.empty[prev]);
      mbar_arrive_cluster(empty_peer + prev * 8);
    }
    prev = stage;
    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
  }
  __device__ __forceinline__ void release_last() {
    if (te == 0) {
      mbar_arrive(&pl.empty[prev]);
      mbar_arrive_cluster(empty_peer + prev * 8);
    }
    prev = -1;
  }

  // The 16-bit output epilogue: out16 (and out16b with TWO_OUT, in both buffers per chunk) in 64-column chunks.
  // vals(j, col, col_ok, v, vb) packs the two 16-bit values of column group j (matrix columns col, col + 1) for rows
  // lr0 and lr0 + 8 into v[0], v[1] (and vb[0], vb[1]), each rounded exactly as a direct store would round it; stmatrix
  // writes them into the swizzled buffer: an 8x8 matrix is 8 rows x one 16-byte unit, the rows in 8 different bank groups.
  template <class Vals>
  __device__ __forceinline__ void store16(const CUtensorMap* tmC, const CUtensorMap* tmC2, int m0w, int n0, int N, Vals vals) {
    constexpr bool TWO = C::TWO_OUT;
    const int mi = lane >> 3;                               // the matrix whose row this lane addresses
    const int lrow = w4 * 16 + (lane & 7) + 8 * (mi & 1);
#pragma unroll
    for (int c = 0; c < C::BLOCK_N / 64; ++c) {
      if (n0 + 64 * c >= N) break;           // N % 32 == 0: the last chunk may be half inside N; TMA clips the rest
      uint8_t* buf = epi + (2 * wg + (TWO ? 0 : (ep & 1))) * kEpiBufBytes;
      const uint32_t row_addr = smem_u32(buf) + lrow * 128;
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {       // column groups j = 8c + 2jp + q, q = 0, 1: matrix 2q + h holds rows lr0 + 8h
        uint32_t v[4], vb[4];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int j = 8 * c + 2 * jp + q, col = n0 + 8 * j + 2 * cq;
          vals(j, col, col < N, v + 2 * q, vb + 2 * q);
        }
        // this lane's row holds column group 2jp + (mi >> 1) in 16-byte unit (2jp + (mi >> 1)) ^ (lrow % 8)
        const uint32_t unit = ((2 * jp + (mi >> 1)) ^ (lane & 7)) << 4;
        stmatrix_x4(row_addr + unit, v[0], v[1], v[2], v[3]);
        if constexpr (TWO) stmatrix_x4(row_addr + kEpiBufBytes + unit, vb[0], vb[1], vb[2], vb[3]);
      }
      fence_proxy_async_smem();              // the writes above -> visible to TMA
      epi_bar(wg);
      if (te == 0) {
        tma_store_2d(tmC, buf, n0 + 64 * c, m0w);
        if constexpr (TWO) tma_store_2d(tmC2, buf + kEpiBufBytes, n0 + 64 * c, m0w);
        tma_store_commit();
        // TWO rewrites both buffers every chunk; otherwise the previous chunk has been read out of the other buffer ...
        if constexpr (TWO) tma_store_wait_read<0>(); else tma_store_wait_read<1>();
      }
      epi_bar(wg);                           // ... which may now be rewritten
      ++ep;
    }
  }

  // every store / reduce-add of this warpgroup has been performed before the CTA retires, so the writes are complete with
  // the grid, as a PDL-launched successor's griddepcontrol.wait expects
  __device__ __forceinline__ void finish() const {
    if (te == 0) tma_store_wait_all<0>();
  }
};

// MN: operand layout.  Bit 0: A is stored [K, M]; bit 1: W is stored [K, N] (the contraction dimension is the ROW index):
// such an operand is fetched as 64-wide MN blocks x 64 k-rows and multiplied through an MN-major wgmma descriptor.
// wgrad uses 3 (dW = dY^T X), dgrad 2 (dX = dY W with W in its [out, in] layout), everything else 0.  A compile-time
// layout keeps one straight-line wgmma sequence per k-block: a run-time choice between four makes ptxas join them with
// an injected empty wgmma group, which turns wgmma_wait<1> into a full drain.
template <int BN, int EPI, bool BF16, int MN>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2, const GemmDev p) {
  // tmC: the output, fp32 resid [M, N] (box 32 x 64) or 16-bit out16 [M, N] (box 64 x 64); tmC2: out16b (GELU_BOTH only)
  using C = Cfg<BN, EPI>;
  constexpr int TA = MN & 1, TB = MN >> 1;
  static_assert(MN == 0 || MN == 2 || MN == 3, "operand layouts: 0 forward, 2 dgrad, 3 wgrad");
  const int warp = threadIdx.x >> 5;
  const Pipeline<C> pl = C::TWO_OUT ? gemm_prologue<C>(&tmA, &tmB, &tmC, &tmC2) : gemm_prologue<C>(&tmA, &tmB, &tmC);
  const PairTiles<BN> pt(p);
  const int num_kb = p.K / BK;
  const bool streamk = C::RESID && p.streamk != 0;

  if (warp < 4) {
    produce(pl, pt, num_kb, streamk, [&](uint8_t* sa, uint64_t* bar, int m_blk, int w_row0, int kb) {
      if (MN == 0 && p.conv_taps > 0) {
        // implicit GEMM: this k-block is channels [cb*64, +64) of filter tap `tap`; the A tile is the tile's
        // conv_bh x conv_bw pixel patch shifted by the tap offset (borders zero-filled by TMA)
        const int tap = kb / p.conv_cblk, cb = kb % p.conv_cblk;
        const int pix0 = m_blk * BM;
        const int hw = p.conv_h * p.conv_w;
        const int img = pix0 / hw, rem = pix0 % hw;
        tma_load_4d(sa, &tmA, bar, cb * BK, rem % p.conv_w + p.conv_dx[tap], rem / p.conv_w + p.conv_dy[tap],
                    img + p.conv_dz[tap]);
      } else if constexpr (TA) {
        // operand stored [K][MN]: one box = 64 MN elements (a 128-byte swizzle row) x 64 k-rows = 8 KiB, the canonical
        // MN-major SW128 block; blocks past the live rows are zero-filled by TMA and still count their bytes
#pragma unroll
        for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * 8192, &tmA, bar, m_blk * BM + j * 64, kb * BK);
      } else {
        tma_load_2d(sa, &tmA, bar, kb * BK, m_blk * BM);
      }
      if constexpr (TB) {
        constexpr int per_cta = BN / 128;    // 64-column blocks of W this CTA fetches
#pragma unroll
        for (int j = 0; j < per_cta; ++j)
          tma_load_2d_mcast(sa + C::A_BYTES + (pt.rank * per_cta + j) * 8192, &tmB, bar, w_row0 + j * 64, kb * BK, 0x3);
      } else {
        tma_load_2d_mcast(sa + C::A_BYTES + pt.rank * (C::B_BYTES / 2), &tmB, bar, kb * BK, w_row0, 0x3);
      }
    });
  } else {
    Consumer<C> cs(pl, pt.rank, (warp >> 2) - 1);
    float acc[BN / 2];
    TileSched sched = pt.sched(num_kb, streamk);
    int tile, kb0, kb1;
    while (sched.next(tile, kb0, kb1)) {
      const int m0 = pt.m_blk(tile) * BM, n0 = pt.n0(tile);
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t sa = cs.wait(), sb = sa + C::A_BYTES;
        wgmma_fence();
        // K-major: 8-row groups 1024 B apart, a k-step of 16 elements = 32 B inside the swizzle row.  MN-major: 64-wide
        // blocks 8192 B apart (leading offset), 8-k-row groups 1024 B apart, a k-step of 16 k-rows = 2048 B.
        const uint64_t da = gmma_desc(sa + cs.wg * 8192, TA ? 8192 : 16, 1024, GMMA_LAYOUT_SW128);
        const uint64_t db = gmma_desc(sb, TB ? 8192 : 16, 1024, GMMA_LAYOUT_SW128);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          WgmmaSS<BN, TA, TB, BF16>::mma(acc, gmma_desc_advance(da, k * (TA ? 2048 : 32)),
                                         gmma_desc_advance(db, k * (TB ? 2048 : 32)), (kb != kb0 || k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                      // the previous k-block's MMAs have read their slot
        cs.release_prev();
      }
      wgmma_wait<0>();
      reg_fence(acc);
      cs.release_last();

      const int m0w = m0 + cs.wg * 64;        // this warpgroup's first row
      if constexpr (C::RESID) {
        // x += gate * (acc + bias) (+ row_add) without ever loading x: the increment goes to a staging buffer in 32-column
        // chunks and TMA adds each chunk into x in L2.  Every element receives one add per GEMM -- or, for stream-K tiles,
        // one per segment in k order (the flag of the tile's rows of this warpgroup) -- so results are deterministic.
        const bool first_seg = kb0 == 0;       // bias and row_add are added once per output element
        const bool partial = kb0 > 0 || kb1 < num_kb;
        unsigned long long* flag = nullptr;
        if (partial) flag = p.sk_flags + (static_cast<size_t>(tile - sched.full_waves * pt.num_pairs) * 2 + pt.rank) * 2 + cs.wg;
        bool ordered = kb0 == 0;               // issuing thread: may this segment add into x yet?
        const float* bias = (p.bias && first_seg) ? p.bias : nullptr;
        const float* gate_row[2];
        const float* add_row[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // a row past M computes an increment from a clamped row, and the reduce-add clips it
          const int row = m0w + cs.lr0 + 8 * h < p.M ? m0w + cs.lr0 + 8 * h : p.M - 1;
          gate_row[h] = p.gate + static_cast<long long>(row / p.rows_per_batch) * p.gate_bs;
          add_row[h] = (p.row_add && first_seg) ? p.row_add + static_cast<size_t>((row / p.row_add_div) % p.row_add_period) * p.N : nullptr;
        }
#pragma unroll
        for (int c = 0; c < BN / 32; ++c) {
          if (n0 + 32 * c >= p.N) break;       // N % 32 == 0: a chunk lies wholly inside N or wholly past it
          uint8_t* buf = cs.epi + (2 * cs.wg + (cs.ep & 1)) * kEpiBufBytes;
          const uint32_t buf_addr = smem_u32(buf);
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * c + jj, col = n0 + 8 * j + 2 * cs.cq;
            const float2 b2 = bias ? __ldg(reinterpret_cast<const float2*>(bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float2 gt = __ldg(reinterpret_cast<const float2*>(gate_row[h] + col));
              const float2 ra = add_row[h] ? __ldg(reinterpret_cast<const float2*>(add_row[h] + col)) : make_float2(0.f, 0.f);
              const float d0 = resid_delta(acc[4 * j + 2 * h], b2.x, gt.x, ra.x, add_row[h] != nullptr);
              const float d1 = resid_delta(acc[4 * j + 2 * h + 1], b2.y, gt.y, ra.y, add_row[h] != nullptr);
              // buffer row lr0 + 8h is 128 bytes; its 16-byte units are XOR-swizzled by the row % 8 (= g), as SW128 TMA reads them
              st_shared_f2(buf_addr + (cs.lr0 + 8 * h) * 128 + (((2 * jj + (cs.cq >> 1)) ^ cs.g) << 4) + 8 * (cs.cq & 1), d0, d1);
            }
          }
          fence_proxy_async_smem();            // the writes above -> visible to TMA
          epi_bar(cs.wg);
          if (cs.te == 0) {
            if (!ordered) {
              // continuing segment: acquire the previous segment's release (it follows that segment's completed adds) ...
              flag_wait(flag, static_cast<unsigned long long>(kb0));
              fence_proxy_async_global();      // ... and order our reduce-adds (async proxy) after the acquire
              if (kb1 == num_kb) flag_release(flag, 0ull);   // nobody else waits on it; left zero for the next launch
              ordered = true;
            }
            tma_reduce_add_2d(&tmC, buf, n0 + 32 * c, m0w);
            tma_store_commit();
            tma_store_wait_read<1>();          // the previous chunk has been read out of the other buffer ...
          }
          epi_bar(cs.wg);                      // ... which may now be rewritten
          ++cs.ep;
        }
        if (partial && kb1 < num_kb && cs.te == 0) {
          tma_store_wait_all<0>();             // this segment's adds have been performed in x ...
          fence_proxy_async_global();          // ... and are ordered before the generic-proxy release:
          flag_release(flag, static_cast<unsigned long long>(kb1));   // the next segment may add
        }
      } else {
        cs.store16(&tmC, &tmC2, m0w, n0, p.N, [&](int j, int col, bool col_ok, uint32_t* v, uint32_t* vb) {
          const float2 b2 = (p.bias && col_ok) ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            if (p.bias) { f0 += b2.x; f1 += b2.y; }
            if constexpr (EPI == B200_EPI_BIAS_GELU) { f0 = gelu_tanh(f0); f1 = gelu_tanh(f1); }
            uint32_t val = pack2<BF16>(f0, f1);
            if constexpr (EPI == B200_EPI_BIAS_ADD16 || EPI == B200_EPI_BIAS_MUL16) {
              const int row = m0w + cs.lr0 + 8 * h;
              const uint32_t side = (row < p.M && col_ok)
                  ? __ldg(reinterpret_cast<const uint32_t*>(p.add16) + (static_cast<size_t>(row) * p.N + col) / 2) : 0u;
              const float2 a = unpack2<BF16>(val), r = unpack2<BF16>(side);
              // + shortcut, both already rounded to 16 bits like the reference
              if constexpr (EPI == B200_EPI_BIAS_ADD16) val = pack2<BF16>(a.x + r.x, a.y + r.y);
              // gated feed-forward: (h wi_1^T) * gelu(h wi_0^T), the second factor read back in 16 bits
              if constexpr (EPI == B200_EPI_BIAS_MUL16) val = pack2<BF16>(a.x * r.x, a.y * r.y);
            }
            if constexpr (C::TWO_OUT) {      // training, fc1: keep the pre-activation u (out16) AND write gelu(u) (out16b)
              const float2 a = unpack2<BF16>(val);
              vb[h] = pack2<BF16>(gelu_tanh(a.x), gelu_tanh(a.y));
            }
            v[h] = val;
          }
        });
      }
    }
    cs.finish();
  }

  cluster_sync_all();   // the peer may still multicast into our smem / arrive on our barriers until it is done too
}

// the kernel's four tensor maps: operands A and W, output (resid or out16) and second output (out16b)
struct GemmMaps { CUtensorMap a, b, c, c2; };

template <int BN, int EPI, bool BF16, int MN>
int launch_one(const GemmMaps& tm, const GemmDev& p, int grid, cudaStream_t stream) {
  using C = Cfg<BN, EPI>;
  auto kern = gemm_kernel<BN, EPI, BF16, MN>;
  B200_SET_SMEM_ONCE(kern, C::SMEM_BYTES);
  B200_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), C::SMEM_BYTES, stream, tm.a, tm.b, tm.c, tm.c2, p));
  return B200_OK;
}

// Only the (epilogue, operand layout) pairs that callers launch are instantiated: every epilogue with K-major operands,
// dgrad's bias with W stored [K, N], and wgrad's unit-gate accumulation with both operands transposed (transposed
// operands take 128- or 256-wide tiles only).
template <int BN, bool BF16>
int launch_epi(int epi, int mn, const GemmMaps& tm, const GemmDev& p, int grid, cudaStream_t s) {
  if (mn == 0) {
    switch (epi) {
      case B200_EPI_BIAS: return launch_one<BN, B200_EPI_BIAS, BF16, 0>(tm, p, grid, s);
      case B200_EPI_BIAS_GELU: return launch_one<BN, B200_EPI_BIAS_GELU, BF16, 0>(tm, p, grid, s);
      case B200_EPI_GATE_RESIDUAL: return launch_one<BN, B200_EPI_GATE_RESIDUAL, BF16, 0>(tm, p, grid, s);
      case B200_EPI_BIAS_ADD16: return launch_one<BN, B200_EPI_BIAS_ADD16, BF16, 0>(tm, p, grid, s);
      case B200_EPI_BIAS_MUL16: return launch_one<BN, B200_EPI_BIAS_MUL16, BF16, 0>(tm, p, grid, s);
      case B200_EPI_BIAS_GELU_BOTH: return launch_one<BN, B200_EPI_BIAS_GELU_BOTH, BF16, 0>(tm, p, grid, s);
    }
  }
  if constexpr (BN != 192) {
    if (mn == 2 && epi == B200_EPI_BIAS) return launch_one<BN, B200_EPI_BIAS, BF16, 2>(tm, p, grid, s);
    if (mn == 3 && epi == B200_EPI_GATE_RESIDUAL) return launch_one<BN, B200_EPI_GATE_RESIDUAL, BF16, 3>(tm, p, grid, s);
  }
  set_error("gemm: epilogue %d with operand layout %d and block_n %d is not built", epi, mn, BN);
  return B200_ERR_UNSUPPORTED;
}

template <int BN>
int launch_bn(int bf16, int epi, int mn, const GemmMaps& tm, const GemmDev& p, int grid, cudaStream_t s) {
  return bf16 ? launch_epi<BN, true>(epi, mn, tm, p, grid, s) : launch_epi<BN, false>(epi, mn, tm, p, grid, s);
}

constexpr int kStreamKMinKb = 32;          // K / 64 below which the split costs more than the idle tail it removes
constexpr int kSkFlags = B200_GEMM_SK_FLAGS;   // flags (u64) in the caller's buffer: 4 per streamed tile

int pick_block_n(int M, int N, int K, bool resid, int sms) {
  // minimise waves x per-tile time.  A tile's cost is modelled by the operand bytes a CTA receives per k-block, A plus
  // its multicast half of W: 128 + BN/2.
  // Where the last wave is streamed along K (residual epilogue, long K) there is no wave rounding.
  // Re-measured with the TMA epilogue on 132 SMs (DESIGN §6): this picks the fastest width for proj and fc1, and widths
  // 4-6 % slower than 192 for QKV and fc2.  No per-tile cost independent of the SM count picks 192 for QKV on 132 SMs
  // but keeps 256 on 148 (QKV at 256 / 192: 7 / 9 waves on 132 SMs, 7 / 8 on 148), and the 148-SM choices are kept as
  // tests/test_schedule.py states them, so the rule is unchanged.
  if (N <= 128) return 128;   // narrow outputs (e.g. the VAE's 3-channel conv_out padded to 32): smallest tile that covers N
  const bool sk = resid && K / BK >= kStreamKMinKb;
  const int cand[3] = {256, 192, 128};
  int best = 128;
  double best_cost = 1e300;
  for (int i = 0; i < 3; ++i) {
    const long long tiles = static_cast<long long>((M + BM - 1) / BM) * ((N + cand[i] - 1) / cand[i]);
    const double waves = (sk && tiles > sms) ? static_cast<double>(tiles) / sms : static_cast<double>((tiles + sms - 1) / sms);
    const double cost = waves * (128 + cand[i] / 2);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = cand[i]; }
  }
  return best;
}

// The scheduling decisions of one launch (shared by launch_gemm and the schedule dump the CPU tests read).  mn: the
// operand layout of gemm_kernel (0 K-major, 2 dgrad, 3 wgrad).
struct GemmPlan { int bn, pairs, pair_tiles, num_kb, streamk; };
GemmPlan plan_gemm(int M, int N, int K, bool resid, int block_n, int sms, int mn = 0) {
  GemmPlan g;
  g.bn = block_n;
  if (g.bn == 0) {
    g.bn = pick_block_n(M, N, K, resid, sms);
    if (mn != 0 && g.bn == 192) g.bn = (N % 256 == 0 || N > 1024) ? 256 : 128;   // W chunks are 64 wide per CTA: 128 or 256 only
    // weight gradients: 256-wide tiles for every output of at least 256 columns (the tiles are split along K anyway, so
    // the wider tile only halves the A traffic)
    if (mn == 3 && N >= 256) g.bn = 256;
  }
  const int num_m = (M + BM - 1) / BM, num_n = (N + g.bn - 1) / g.bn;
  g.pair_tiles = ((num_m + 1) / 2) * num_n;
  const int grid = 2 * g.pair_tiles < sms ? 2 * g.pair_tiles : (sms & ~1);   // whole clusters of 2
  g.pairs = grid / 2;
  g.num_kb = K / BK;
  g.streamk = (resid && g.pair_tiles > g.pairs && g.pair_tiles % g.pairs != 0 && g.num_kb >= kStreamKMinKb) ? 1 : 0;
  // weight gradients: a small output (fewer tiles than CTA pairs) under a very long contraction (K = tokens).  All tiles are
  // streamed: the (tile, k-block) units are cut into one equal share per pair, a tile's partial sums are reduce-added in k
  // order through the same flags (a chain of waits only ever points from pair p+1 to pair p, and every pair is resident).
  if (mn == 3 && resid && g.pair_tiles <= sms / 2 && g.pair_tiles % (sms / 2) != 0 &&
      static_cast<long long>(g.pair_tiles) * g.num_kb >= static_cast<long long>(sms / 2) * kStreamKMinKb) {
    g.pairs = sms / 2;
    g.streamk = 1;
  }
  return g;
}

// GemmDev with the problem and its grid of BM x bn tiles set, every other field zero
GemmDev gemm_dev(int M, int N, int K, int bn) {
  GemmDev p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m = (M + BM - 1) / BM;
  p.num_n = (N + bn - 1) / bn;
  return p;
}

// a 16-bit [M, N] row-major output: one 64-row x 128-byte box (64 columns) per staging buffer; the callers' alignment
// checks and N % 32 == 0 give TMA its 16-byte base and row stride
int make_out16_map(CUtensorMap* m, void* out, int M, int N) {
  const uint64_t dims[2] = {static_cast<uint64_t>(N), static_cast<uint64_t>(M)};
  const uint64_t str[1] = {static_cast<uint64_t>(N) * 2};
  const uint32_t box[2] = {64, 64};
  return make_tmap_16bit(m, out, 2, dims, str, box, TMAP_SW_128);
}

// ---------------------------------------------------------------------------------------------------- FP8 (e4m3) GEMM
// out16 = epi(s_a[row] * s_w[col] * (A8 . W8^T) + bias) for QKV and fc1 of the sampling forward: A8 and s_a come from
// the e4m3 instance of ln_modulate (one scale per token), W8 and s_w from quantize_rows_e4m3 (one per output channel).
// It runs on the shared pieces above with K-major operands: prologue, pair tiles, TMA producer, stage bookkeeping and the
// 16-bit epilogue.  Its own are the k-block and the output value.  A 128-byte swizzle row holds 128 e4m3 elements, so
// one stage is one 128-wide k-block with the same bytes as a 16-bit stage, and a k-block is four m64nNk32 e4m3 wgmma whose
// descriptors advance 32 bytes each, as the 16-bit k16 steps do.  K need not be a multiple of 128: the last k-block's
// columns past K are zero-filled by TMA (which still counts the whole box toward the barrier's bytes).
// Accumulation: FP8 wgmma keeps fewer accumulator bits than fp32 (DESIGN.md §6, FP8 sampling path), so each k-block is
// summed in registers of its own -- alternately acc0 and acc1, the k-block's first wgmma overwriting -- and added into the
// fp32 total `sum` once the NEXT k-block's wgmma are in flight: the k-loop still waits with wgmma_wait<1>.  The three
// 64-float fragments fit the consumers' 232 registers at BN = 128 only, so that is the one tile width.
// Output value: ((sum * s_a[row]) * s_w[col]) + bias, each step rounded, then GELU for fc1.
constexpr int BN8 = 128;
constexpr int BK8 = 128;

template <int EPI, bool BF16>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
fp8_linear_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const GemmDev p, const float* __restrict__ a_scale,
                  const float* __restrict__ w_scale) {
  using C = Cfg<BN8, EPI>;
  static_assert(C::A_BYTES == BM * BK8 && C::B_BYTES == BN8 * BK8, "a stage holds one e4m3 k-block");
  static_assert(EPI == B200_EPI_BIAS || EPI == B200_EPI_BIAS_GELU, "16-bit output epilogues only");
  const int warp = threadIdx.x >> 5;
  const Pipeline<C> pl = gemm_prologue<C>(&tmA, &tmB, &tmC);
  const PairTiles<BN8> pt(p);
  const int num_kb = (p.K + BK8 - 1) / BK8;

  if (warp < 4) {
    produce(pl, pt, num_kb, false, [&](uint8_t* sa, uint64_t* bar, int m_blk, int w_row0, int kb) {
      tma_load_2d(sa, &tmA, bar, kb * BK8, m_blk * BM);
      tma_load_2d_mcast(sa + C::A_BYTES + pt.rank * (C::B_BYTES / 2), &tmB, bar, kb * BK8, w_row0, 0x3);
    });
  } else {
    Consumer<C> cs(pl, pt.rank, (warp >> 2) - 1);
    float acc0[BN8 / 2], acc1[BN8 / 2], sum[BN8 / 2];
    // one k-block into `cur`; once the previous k-block's wgmma have completed, its slot is released and its partial sum
    // `done` is added into `sum`
    auto kblock = [&](float (&cur)[BN8 / 2], float (&done)[BN8 / 2]) {
      const uint32_t sa = cs.wait(), sb = sa + C::A_BYTES;
      wgmma_fence();
      const uint64_t da = gmma_desc(sa + cs.wg * 8192, 16, 1024, GMMA_LAYOUT_SW128);
      const uint64_t db = gmma_desc(sb, 16, 1024, GMMA_LAYOUT_SW128);
#pragma unroll
      for (int k = 0; k < BK8 / 32; ++k)
        WgmmaE4M3<BN8>::mma(cur, gmma_desc_advance(da, k * 32), gmma_desc_advance(db, k * 32), k ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      reg_fence(done);
      cs.release_prev();
#pragma unroll
      for (int i = 0; i < BN8 / 2; ++i) sum[i] += done[i];
    };
    auto drain = [&](float (&cur)[BN8 / 2]) {
      wgmma_wait<0>();
      reg_fence(cur);
      cs.release_last();
#pragma unroll
      for (int i = 0; i < BN8 / 2; ++i) sum[i] += cur[i];
    };
    TileSched sched = pt.sched(num_kb, false);
    int tile, kb0, kb1;
    while (sched.next(tile, kb0, kb1)) {
      const int m0 = pt.m_blk(tile) * BM, n0 = pt.n0(tile);
#pragma unroll
      for (int i = 0; i < BN8 / 2; ++i) { sum[i] = 0.f; acc1[i] = 0.f; }
      for (int kb = kb0;;) {                  // k-blocks alternate between acc0 and acc1 (acc1 = 0 before the first)
        kblock(acc0, acc1);
        if (++kb == kb1) { drain(acc0); break; }
        kblock(acc1, acc0);
        if (++kb == kb1) { drain(acc1); break; }
      }

      const int m0w = m0 + cs.wg * 64;
      float sa_row[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0w + cs.lr0 + 8 * h;
        sa_row[h] = row < p.M ? __ldg(a_scale + row) : 0.f;   // rows past M are clipped by the TMA store
      }
      cs.store16(&tmC, nullptr, m0w, n0, p.N, [&](int j, int col, bool col_ok, uint32_t* v, uint32_t*) {
        const float2 b2 = (p.bias && col_ok) ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
        const float2 s2 = col_ok ? __ldg(reinterpret_cast<const float2*>(w_scale + col)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f0 = __fadd_rn(__fmul_rn(__fmul_rn(sum[4 * j + 2 * h], sa_row[h]), s2.x), b2.x);
          float f1 = __fadd_rn(__fmul_rn(__fmul_rn(sum[4 * j + 2 * h + 1], sa_row[h]), s2.y), b2.y);
          if constexpr (EPI == B200_EPI_BIAS_GELU) { f0 = gelu_tanh(f0); f1 = gelu_tanh(f1); }
          v[h] = pack2<BF16>(f0, f1);
        }
      });
    }
    cs.finish();
  }

  cluster_sync_all();
}

template <int EPI, bool BF16>
int launch_e4m3(const GemmMaps& tm, const GemmDev& p, const float* a_scale, const float* w_scale, int grid, cudaStream_t stream) {
  using C = Cfg<BN8, EPI>;
  auto kern = fp8_linear_kernel<EPI, BF16>;
  B200_SET_SMEM_ONCE(kern, C::SMEM_BYTES);
  B200_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), C::SMEM_BYTES, stream, tm.a, tm.b, tm.c, p, a_scale, w_scale));
  return B200_OK;
}

}  // namespace

int gemm_schedule(int M, int N, int K, int epilogue, int block_n, int sms, int* bn_out, int* pairs_out, int* streamk_out,
                  int* segments, int max_segments, int wgrad) {
  B200_REQUIRE(M > 0 && N > 0 && K > 0 && K % BK == 0 && sms >= 2, B200_ERR_SHAPE, "gemm_schedule: bad arguments");
  B200_REQUIRE(block_n == 0 || block_n == 128 || block_n == 192 || block_n == 256, B200_ERR_UNSUPPORTED, "gemm_schedule: block_n %d", block_n);
  // wgrad: the schedule launch_gemm gives a weight gradient (both operands transposed)
  const GemmPlan g = plan_gemm(M, N, K, epilogue == B200_EPI_GATE_RESIDUAL, block_n, sms, wgrad ? 3 : 0);
  if (bn_out) *bn_out = g.bn;
  if (pairs_out) *pairs_out = g.pairs;
  if (streamk_out) *streamk_out = g.streamk;
  int n = 0;
  for (int pair = 0; pair < g.pairs; ++pair) {
    TileSched sched(pair, g.pairs, g.pair_tiles, g.num_kb, g.streamk != 0);
    int tile, kb0, kb1;
    while (sched.next(tile, kb0, kb1)) {       // in the order the pair executes them
      if (segments && n < max_segments) {
        segments[4 * n + 0] = pair; segments[4 * n + 1] = tile; segments[4 * n + 2] = kb0; segments[4 * n + 3] = kb1;
      }
      ++n;
    }
  }
  return n;
}

int launch_gemm(const GemmArgs& a, cudaStream_t stream) {
  B200_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, B200_ERR_SHAPE, "gemm: bad shape M=%d N=%d K=%d", a.M, a.N, a.K);
  B200_REQUIRE(a.K % BK == 0, B200_ERR_SHAPE, "gemm: K=%d must be a multiple of %d", a.K, BK);
  B200_REQUIRE(a.N % 32 == 0, B200_ERR_SHAPE, "gemm: N=%d must be a multiple of 32", a.N);
  B200_REQUIRE(a.epilogue == B200_EPI_BIAS || a.epilogue == B200_EPI_BIAS_GELU || a.epilogue == B200_EPI_GATE_RESIDUAL ||
                   a.epilogue == B200_EPI_BIAS_ADD16 || a.epilogue == B200_EPI_BIAS_MUL16 || a.epilogue == B200_EPI_BIAS_GELU_BOTH,
               B200_ERR_UNSUPPORTED, "gemm: unknown epilogue %d", a.epilogue);
  B200_REQUIRE((a.epilogue != B200_EPI_BIAS_ADD16 && a.epilogue != B200_EPI_BIAS_MUL16) ||
                   (a.add16 && (reinterpret_cast<uintptr_t>(a.add16) & 15) == 0), B200_ERR_ALIGN, "gemm: add16 tensor missing or unaligned");
  B200_REQUIRE(a.epilogue != B200_EPI_BIAS_GELU_BOTH || (a.out16b && (reinterpret_cast<uintptr_t>(a.out16b) & 15) == 0), B200_ERR_ALIGN,
               "gemm: second output missing or unaligned");
  B200_REQUIRE(a.epilogue != B200_EPI_BIAS_GELU_BOTH || a.N % 8 == 0, B200_ERR_SHAPE, "gemm: N %% 8");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(a.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.W) & 15) == 0,
               B200_ERR_ALIGN, "gemm: A and W must be 16-byte aligned");
  const bool resid = a.epilogue == B200_EPI_GATE_RESIDUAL;
  if (resid) {
    B200_REQUIRE(a.resid && a.gate && a.rows_per_batch > 0, B200_ERR_SHAPE, "gemm: gated-residual epilogue needs resid, gate, rows_per_batch");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(a.resid) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.gate) & 15) == 0 &&
                     (a.gate_batch_stride % 4) == 0,
                 B200_ERR_ALIGN, "gemm: resid/gate must be 16-byte aligned");
    B200_REQUIRE(!a.row_add || (reinterpret_cast<uintptr_t>(a.row_add) & 15) == 0, B200_ERR_ALIGN, "gemm: row_add must be 16-byte aligned");
  } else {
    B200_REQUIRE(a.out16 && (reinterpret_cast<uintptr_t>(a.out16) & 15) == 0, B200_ERR_ALIGN, "gemm: out16 must be 16-byte aligned");
  }
  B200_REQUIRE(!a.bias || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0, B200_ERR_ALIGN, "gemm: bias must be 16-byte aligned");
  B200_TRY(check_arch());
  int sms = 0;
  B200_TRY(device_sm_count(&sms));

  B200_REQUIRE(a.block_n == 0 || a.block_n == 128 || a.block_n == 192 || a.block_n == 256, B200_ERR_UNSUPPORTED,
               "gemm: block_n must be 128, 192 or 256 (got %d)", a.block_n);
  if (a.mn_major) {
    B200_REQUIRE((a.mn_major == 2 || a.mn_major == 3) && a.conv_taps == 0 && (!(a.mn_major & 1) || a.M % 8 == 0) &&
                     (!(a.mn_major & 2) || a.N % 128 == 0) && (a.block_n == 0 || a.block_n == 128 || a.block_n == 256),
                 B200_ERR_UNSUPPORTED, "gemm (transposed operands): mn_major 2 or 3, M %% 8 == 0, N %% 128 == 0, block_n 128 or 256 (M=%d N=%d)",
                 a.M, a.N);
  }
  const GemmPlan plan = plan_gemm(a.M, a.N, a.K, resid, a.block_n, sms, a.mn_major);
  const int bn = plan.bn;

  GemmMaps tm;
  CUtensorMap& tmA = tm.a;
  CUtensorMap& tmB = tm.b;
  int conv_bw = 0, conv_bh = 0;
  {
    if (a.conv_taps > 0) {
      B200_REQUIRE(a.conv_taps <= 9 && a.conv_c % BK == 0 && a.K == a.conv_taps * a.conv_c &&
                       a.M == a.conv_n * a.conv_h * a.conv_w,
                   B200_ERR_SHAPE, "conv: inconsistent geometry (taps %d, C %d, K %d, M %d)", a.conv_taps, a.conv_c, a.K, a.M);
      conv_bw = a.conv_w >= BM ? BM : a.conv_w;
      conv_bh = BM / conv_bw;
      B200_REQUIRE(BM % conv_bw == 0 && a.conv_w % conv_bw == 0 && a.conv_h % conv_bh == 0, B200_ERR_UNSUPPORTED,
                   "conv: %dx%d feature map cannot be tiled by 128-pixel patches", a.conv_h, a.conv_w);
      const uint64_t dimsA[4] = {static_cast<uint64_t>(a.conv_c), static_cast<uint64_t>(a.conv_w), static_cast<uint64_t>(a.conv_h),
                                 static_cast<uint64_t>(a.conv_n)};
      const uint64_t strA[3] = {static_cast<uint64_t>(a.conv_c) * 2, static_cast<uint64_t>(a.conv_c) * 2 * a.conv_w,
                                static_cast<uint64_t>(a.conv_c) * 2 * a.conv_w * a.conv_h};
      const uint32_t boxA[4] = {BK, static_cast<uint32_t>(conv_bw), static_cast<uint32_t>(conv_bh), 1};
      B200_TRY(make_tmap_16bit(&tmA, a.A, 4, dimsA, strA, boxA, TMAP_SW_128));
    } else if (a.mn_major & 1) {
      const uint64_t dimsA[2] = {static_cast<uint64_t>(a.M), static_cast<uint64_t>(a.K)};      // stored [K][M]
      const uint64_t strA[1] = {static_cast<uint64_t>(a.M) * 2};
      const uint32_t boxA[2] = {64, BK};
      B200_TRY(make_tmap_16bit(&tmA, a.A, 2, dimsA, strA, boxA, TMAP_SW_128));
    } else {
      const uint64_t dimsA[2] = {static_cast<uint64_t>(a.K), static_cast<uint64_t>(a.M)};
      const uint64_t strA[1] = {static_cast<uint64_t>(a.K) * 2};
      const uint32_t boxA[2] = {BK, BM};
      B200_TRY(make_tmap_16bit(&tmA, a.A, 2, dimsA, strA, boxA, TMAP_SW_128));
    }
    if (a.mn_major & 2) {
      const uint64_t dimsB[2] = {static_cast<uint64_t>(a.N), static_cast<uint64_t>(a.K)};      // stored [K][N]
      const uint64_t strB[1] = {static_cast<uint64_t>(a.N) * 2};
      const uint32_t boxB[2] = {64, BK};
      B200_TRY(make_tmap_16bit(&tmB, a.W, 2, dimsB, strB, boxB, TMAP_SW_128));
    } else {
      const uint64_t dimsB[2] = {static_cast<uint64_t>(a.K), static_cast<uint64_t>(a.N)};
      const uint64_t strB[1] = {static_cast<uint64_t>(a.K) * 2};
      const uint32_t boxB[2] = {BK, static_cast<uint32_t>(bn / 2)};   // each CTA of the pair fetches half and multicasts it
      B200_TRY(make_tmap_16bit(&tmB, a.W, 2, dimsB, strB, boxB, TMAP_SW_128));
    }
    // the output, [M, N] row-major: one 64-row x 128-byte box per staging buffer (32 fp32 or 64 16-bit columns)
    if (resid) {
      const uint64_t dimsC[2] = {static_cast<uint64_t>(a.N), static_cast<uint64_t>(a.M)};
      const uint64_t strC[1] = {static_cast<uint64_t>(a.N) * 4};
      const uint32_t boxC[2] = {32, 64};
      B200_TRY(make_tmap(&tm.c, a.resid, 4, 2, dimsC, strC, boxC, TMAP_SW_128));
      tm.c2 = tm.c;
    } else {
      B200_TRY(make_out16_map(&tm.c, a.out16, a.M, a.N));
      if (a.epilogue == B200_EPI_BIAS_GELU_BOTH) B200_TRY(make_out16_map(&tm.c2, a.out16b, a.M, a.N));
      else tm.c2 = tm.c;
    }
  }
  GemmDev p = gemm_dev(a.M, a.N, a.K, bn);
  p.bias = a.bias;
  p.out16 = a.out16;
  p.gate = a.gate;
  p.gate_bs = a.gate_batch_stride;
  p.rows_per_batch = a.rows_per_batch > 0 ? a.rows_per_batch : 1;
  p.row_add = a.row_add;
  p.row_add_div = a.row_add_div > 0 ? a.row_add_div : 1;
  p.row_add_period = a.row_add_period > 0 ? a.row_add_period : 1;
  p.add16 = static_cast<const uint16_t*>(a.add16);
  p.out16b = static_cast<uint16_t*>(a.out16b);
  p.conv_taps = a.conv_taps;
  p.conv_cblk = a.conv_taps > 0 ? a.conv_c / BK : 0;
  p.conv_h = a.conv_h; p.conv_w = a.conv_w; p.conv_bw = conv_bw; p.conv_bh = conv_bh;
  for (int i = 0; i < 9; ++i) { p.conv_dx[i] = a.conv_dx[i]; p.conv_dy[i] = a.conv_dy[i]; p.conv_dz[i] = a.conv_dz[i]; }
  p.resid = a.resid;
  const int pair_tiles = plan.pair_tiles;
  const int grid = 2 * plan.pairs;
  {
    // stream-K over the last waves: only where partial sums can be reduce-added (residual epilogue) and K is long enough
    // to be worth splitting (plan_gemm).
    const int pairs = plan.pairs;
    // the ordering flags live in the CALLER's buffer (zeroed once; every launch leaves it zeroed): without one the
    // schedule stays data-parallel
    const int streamed = pair_tiles % pairs + pairs;  // tiles of the partial wave and of the full wave before it
    p.streamk = (plan.streamk && a.sk_flags != nullptr && streamed * 4 <= kSkFlags) ? 1 : 0;
    p.sk_flags = p.streamk ? a.sk_flags : nullptr;
  }
  switch (bn) {
    case 128: return launch_bn<128>(a.bf16, a.epilogue, a.mn_major, tm, p, grid, stream);
    case 192: return launch_bn<192>(a.bf16, a.epilogue, a.mn_major, tm, p, grid, stream);
    default: return launch_bn<256>(a.bf16, a.epilogue, a.mn_major, tm, p, grid, stream);
  }
}

int launch_linear_e4m3(const void* A8, const float* a_scale, const void* W8, const float* w_scale, const float* bias, int M, int N,
                       int K, int bf16, int epilogue, void* out16, cudaStream_t stream) {
  B200_REQUIRE(M > 0 && N > 0 && K > 0, B200_ERR_SHAPE, "gemm e4m3: bad shape M=%d N=%d K=%d", M, N, K);
  B200_REQUIRE(K % 16 == 0, B200_ERR_UNSUPPORTED, "gemm e4m3: K=%d: rows must be a multiple of 16 bytes", K);
  B200_REQUIRE(N % 32 == 0, B200_ERR_SHAPE, "gemm e4m3: N=%d must be a multiple of 32", N);
  B200_REQUIRE(epilogue == B200_EPI_BIAS || epilogue == B200_EPI_BIAS_GELU, B200_ERR_UNSUPPORTED,
               "gemm e4m3: epilogue %d not built (bias and bias+GELU only)", epilogue);
  B200_REQUIRE(((reinterpret_cast<uintptr_t>(A8) | reinterpret_cast<uintptr_t>(W8) | reinterpret_cast<uintptr_t>(out16) |
                 reinterpret_cast<uintptr_t>(bias)) & 15) == 0 && A8 && W8 && out16,
               B200_ERR_ALIGN, "gemm e4m3: A, W, out16 (and bias) must be 16-byte aligned");
  B200_REQUIRE(a_scale && w_scale && (reinterpret_cast<uintptr_t>(a_scale) & 3) == 0 && (reinterpret_cast<uintptr_t>(w_scale) & 7) == 0,
               B200_ERR_ALIGN, "gemm e4m3: a_scale (4-byte) and w_scale (8-byte aligned) are required");
  B200_TRY(check_arch());
  int sms = 0;
  B200_TRY(device_sm_count(&sms));
  const GemmPlan plan = plan_gemm(M, N, K, false, BN8, sms);
  GemmMaps tm;
  {
    const uint64_t dimsA[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    const uint64_t strA[1] = {static_cast<uint64_t>(K)};
    const uint32_t boxA[2] = {BK8, BM};
    B200_TRY(make_tmap(&tm.a, A8, 1, 2, dimsA, strA, boxA, TMAP_SW_128));
    const uint64_t dimsB[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    const uint32_t boxB[2] = {BK8, BN8 / 2};
    B200_TRY(make_tmap(&tm.b, W8, 1, 2, dimsB, strA, boxB, TMAP_SW_128));
    B200_TRY(make_out16_map(&tm.c, out16, M, N));
  }
  GemmDev p = gemm_dev(M, N, K, BN8);
  p.bias = bias;
  p.out16 = out16;
  p.rows_per_batch = 1;
  const int grid = 2 * plan.pairs;
  if (epilogue == B200_EPI_BIAS)
    return bf16 ? launch_e4m3<B200_EPI_BIAS, true>(tm, p, a_scale, w_scale, grid, stream)
                : launch_e4m3<B200_EPI_BIAS, false>(tm, p, a_scale, w_scale, grid, stream);
  return bf16 ? launch_e4m3<B200_EPI_BIAS_GELU, true>(tm, p, a_scale, w_scale, grid, stream)
              : launch_e4m3<B200_EPI_BIAS_GELU, false>(tm, p, a_scale, w_scale, grid, stream);
}

}  // namespace b200
