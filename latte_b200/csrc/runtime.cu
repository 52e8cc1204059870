// Host-side runtime pieces: thread-local error text, TMA tensor-map encoding, device queries.
#include "common.h"

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace b200 {

namespace {
thread_local char g_err[512] = {0};
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// cuTensorMapEncodeTiled is a driver-API symbol. The library must load on machines without libcuda
// (the CPU-only build/test container), so it is resolved at first use through the runtime.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, TmapSwizzle sw) {
  return make_tmap(out, base, 2, rank, dims, strides_bytes, box, sw);
}

// ---- descriptor cache.  A denoising step re-issues the same ~20 distinct (pointer, shape, box) combinations hundreds of
// times (203 launches, 2-4 maps each); a map is a pure function of its arguments, so encoded maps are kept per thread
// keyed by those arguments.  Bounded: the table is dropped when it grows past kTmapCacheMax entries.
namespace {
struct TmapKey {
  uint64_t base;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  uint32_t rank_elem_sw;
  bool operator==(const TmapKey& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) { h ^= w[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); }
    return static_cast<size_t>(h);
  }
};
static_assert(sizeof(TmapKey) % 8 == 0, "TmapKey is hashed as 64-bit words");
constexpr size_t kTmapCacheMax = 4096;
int encode_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, TmapSwizzle sw);
}  // namespace

int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, TmapSwizzle sw) {
  B200_REQUIRE(rank >= 2 && rank <= 5, B200_ERR_SHAPE, "tensor map rank %d unsupported", rank);
  thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey k;
  std::memset(&k, 0, sizeof(k));
  k.base = reinterpret_cast<uint64_t>(base);
  for (int i = 0; i < rank; ++i) { k.dims[i] = dims[i]; k.box[i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) k.strides[i] = strides_bytes[i];
  k.rank_elem_sw = static_cast<uint32_t>(rank) | (static_cast<uint32_t>(elem_bytes) << 8) | (static_cast<uint32_t>(sw) << 16);
  auto it = cache.find(k);
  if (it != cache.end()) {
    *out = it->second;
    return B200_OK;
  }
  B200_TRY(encode_tmap(out, base, elem_bytes, rank, dims, strides_bytes, box, sw));
  if (cache.size() >= kTmapCacheMax) cache.clear();
  cache.emplace(k, *out);
  return B200_OK;
}

namespace {
int encode_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, TmapSwizzle sw) {
  EncodeTiledFn fn = get_encode_fn();
  B200_REQUIRE(fn != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeTiled not available from the CUDA driver");
  B200_REQUIRE(rank >= 2 && rank <= 5, B200_ERR_SHAPE, "tensor map rank %d unsupported", rank);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_bytes[i];
  CUtensorMapSwizzle s = CU_TENSOR_MAP_SWIZZLE_NONE;
  switch (sw) {
    case TMAP_SW_32: s = CU_TENSOR_MAP_SWIZZLE_32B; break;
    case TMAP_SW_64: s = CU_TENSOR_MAP_SWIZZLE_64B; break;
    case TMAP_SW_128: s = CU_TENSOR_MAP_SWIZZLE_128B; break;
    default: break;
  }
  // the bit pattern is moved, never interpreted, so one unsigned type per element size serves e4m3, fp16/bf16 and fp32
  B200_REQUIRE(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4, B200_ERR_DTYPE, "tensor map element size %d unsupported", elem_bytes);
  // 4-byte maps are typed FLOAT32 so that TMA reductions (cp.reduce ... .add) add floats
  const CUtensorMapDataType dt = elem_bytes == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                 : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                                   : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, s, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, B200_ERR_CUDA,
               "cuTensorMapEncodeTiled failed (CUresult %d; rank %d dims %llu,%llu box %u,%u base %p)", static_cast<int>(r),
               rank, static_cast<unsigned long long>(dims[0]), static_cast<unsigned long long>(dims[1]), box[0], box[1],
               base);
  return B200_OK;
}
}  // namespace

namespace {
struct DevInfo {
  int valid = 0, major = 0, minor = 0, sms = 0;
};
DevInfo g_dev[64];
std::mutex g_dev_mu;

int dev_info(DevInfo* out) {
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_REQUIRE(dev >= 0 && dev < 64, B200_ERR_CUDA, "device ordinal %d out of range", dev);
  std::lock_guard<std::mutex> lk(g_dev_mu);
  if (!g_dev[dev].valid) {
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&g_dev[dev].major, cudaDevAttrComputeCapabilityMajor, dev));
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&g_dev[dev].minor, cudaDevAttrComputeCapabilityMinor, dev));
    B200_CHECK_CUDA(cudaDeviceGetAttribute(&g_dev[dev].sms, cudaDevAttrMultiProcessorCount, dev));
    g_dev[dev].valid = 1;
  }
  *out = g_dev[dev];
  return B200_OK;
}
}  // namespace

int current_device(int* out) {
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_REQUIRE(dev >= 0 && dev < 64, B200_ERR_CUDA, "device ordinal %d out of range", dev);
  *out = dev;
  return B200_OK;
}

int device_sm_count(int* out) {
  DevInfo d;
  B200_TRY(dev_info(&d));
  *out = d.sms;
  return B200_OK;
}

int check_arch() {
  DevInfo d;
  B200_TRY(dev_info(&d));
  B200_REQUIRE(d.major == 9 && d.minor == 0, B200_ERR_ARCH, "latte_b200 kernels are sm_90a (Hopper) only; current device is sm_%d%d",
               d.major, d.minor);
  return B200_OK;
}

}  // namespace b200
