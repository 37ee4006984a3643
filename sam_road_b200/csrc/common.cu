// sam_road_b200 :: host-side common pieces: last-error slot, launch check and count, shared-memory opt-in,
// SM count, TMA descriptor encoding.
#include "common.cuh"
#include "ops.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <mutex>
#include <utility>

namespace srb {

static thread_local char g_last_error[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}
const char* get_last_error() { return g_last_error; }

static std::atomic<uint64_t> g_launches{0};
static void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
uint64_t launch_count(bool reset) {
  return reset ? g_launches.exchange(0) : g_launches.load();
}

int launched(const char* file, int line, const char* call) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s:%d: SRB_LAUNCH(%s) -> %s", file, line, call, cudaGetErrorString(e));
    return 1;
  }
  note_launch();
  return 0;
}

int allow_dynamic_smem(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> allowed;   // (device, kernel) -> bytes set
  int dev = 0;
  SRB_CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = allowed[{dev, kernel}];
  if (bytes <= have) return 0;
  SRB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
  have = bytes;
  return 0;
}

template <bool kPinned>
void Buffer<kPinned>::release() {
  if (p_) kPinned ? cudaFreeHost(p_) : cudaFree(p_);
  p_ = nullptr;
  cap_ = 0;
}

template <bool kPinned>
int Buffer<kPinned>::reserve(size_t bytes, const char* what) {
  if (bytes <= cap_) return 0;
  release();
  if ((kPinned ? cudaMallocHost(&p_, bytes) : cudaMalloc(&p_, bytes)) != cudaSuccess) {
    cudaGetLastError();   // a failed allocation must not fail the next call's launch check
    p_ = nullptr;
    set_last_error("%s: out of %s memory (%zu bytes)", what, kPinned ? "pinned host" : "device", bytes);
    return 1;
  }
  cap_ = bytes;
  return 0;
}

template class Buffer<false>;
template class Buffer<true>;

int open_device(int device) {
  int ndev = 0;
  SRB_CUDA_OK(cudaGetDeviceCount(&ndev));
  SRB_REQUIRE(ndev > 0, "no CUDA device: libsamroad_b200 has no CPU fallback");
  SRB_REQUIRE(device >= 0 && device < ndev, "device %d out of range (0..%d)", device, ndev - 1);
  SRB_CUDA_OK(cudaSetDevice(device));
  return 0;
}

int check_csr(const char* what, int32_t n, const int32_t* start, const int32_t* list) {
  SRB_REQUIRE(start[0] == 0, "%s: adjacency offsets must start at 0", what);
  for (int32_t i = 0; i < n; ++i)
    SRB_REQUIRE(start[i + 1] >= start[i], "%s: adjacency offsets decrease at %d", what, i);
  const int32_t m = start[n];
  SRB_REQUIRE(m == 0 || list != nullptr, "%s: null adjacency", what);
  for (int32_t e = 0; e < m; ++e)
    SRB_REQUIRE(list[e] >= 0 && list[e] < n, "%s: neighbour %d out of range", what, list[e]);
  return 0;
}

int device_sm_count() {
  static int cached[64] = {0};     // per device: a process may drive several GPUs
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;   // H100 SXM
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      return 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap_f16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                     uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled fn = get_encode_fn();
  SRB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15u) == 0, "TMA base %p not 16-byte aligned",
              base);
  SRB_REQUIRE((ld_elems * 2) % 16 == 0, "TMA row pitch %llu B not a multiple of 16",
              (unsigned long long)(ld_elems * 2));
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstr, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SRB_REQUIRE(r == CUDA_SUCCESS,
              "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box=%ux%u", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems,
              box_rows, box_cols);
  return 0;
}

int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                     uint32_t box_rows) {
  PFN_encodeTiled fn = get_encode_fn();
  SRB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15u) == 0, "TMA base %p not 16-byte aligned",
              base);
  SRB_REQUIRE((ld_elems * 4) % 16 == 0, "TMA row pitch %llu B not a multiple of 16",
              (unsigned long long)(ld_elems * 4));
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld_elems * 4};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SRB_REQUIRE(r == CUDA_SUCCESS,
              "cuTensorMapEncodeTiled(f32) failed (%d) rows=%llu cols=%llu ld=%llu box=%ux32", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows);
  return 0;
}

int make_tmap_f16_4d(CUtensorMap* out, const void* base, const uint64_t dims[4],
                     const uint64_t strides_elems[3], const uint32_t box[4]) {
  PFN_encodeTiled fn = get_encode_fn();
  SRB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15u) == 0, "TMA base %p not 16-byte aligned",
              base);
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides_elems[0] * 2, strides_elems[1] * 2, strides_elems[2] * 2};
  for (int i = 0; i < 3; ++i)
    SRB_REQUIRE(gstr[i] % 16 == 0, "TMA stride %d = %llu B not a multiple of 16", i,
                (unsigned long long)gstr[i]);
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gdim, gstr, bx,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SRB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(4D) failed (%d)", (int)r);
  return 0;
}

// fp32 4-D map without swizzle (dense smem box), strides in bytes
int make_tmap_f32_4d_dense(CUtensorMap* out, const void* base, const uint64_t dims[4],
                           const uint64_t strides_bytes[3], const uint32_t box[4]) {
  PFN_encodeTiled fn = get_encode_fn();
  SRB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  SRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15u) == 0, "TMA base %p not 16-byte aligned",
              base);
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  for (int i = 0; i < 3; ++i)
    SRB_REQUIRE(gstr[i] % 16 == 0, "TMA stride %d = %llu B not a multiple of 16", i,
                (unsigned long long)gstr[i]);
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), gdim, gstr, bx,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SRB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(4D f32) failed (%d)", (int)r);
  return 0;
}

// Stream memory operations (cuStreamWriteValue32 / cuStreamWaitValue32): flag writes and waits executed by the
// stream front end, no kernel and no SM involved -- the exchange step's barrier between ranks uses them on
// symmetric (peer-mapped) flag words so that nothing spins on an SM next to the persistent compute kernels.
typedef CUresult (*PFN_streamMemOp32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static PFN_streamMemOp32 get_memop_fn(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
    return reinterpret_cast<PFN_streamMemOp32>(p);
  return nullptr;
}
int stream_write_value32(void* addr, uint32_t value, cudaStream_t st) {
  static PFN_streamMemOp32 fn = get_memop_fn("cuStreamWriteValue32");
  SRB_REQUIRE(fn != nullptr, "cuStreamWriteValue32 driver entry point not available");
  const CUresult r = fn(reinterpret_cast<CUstream>(st), reinterpret_cast<CUdeviceptr>(addr), value, 0 /* default: ordered write */);
  SRB_REQUIRE(r == CUDA_SUCCESS, "cuStreamWriteValue32 failed (%d)", static_cast<int>(r));
  return 0;
}
int stream_wait_value32_geq(void* addr, uint32_t value, cudaStream_t st) {
  static PFN_streamMemOp32 fn = get_memop_fn("cuStreamWaitValue32");
  SRB_REQUIRE(fn != nullptr, "cuStreamWaitValue32 driver entry point not available");
  const CUresult r = fn(reinterpret_cast<CUstream>(st), reinterpret_cast<CUdeviceptr>(addr), value, CU_STREAM_WAIT_VALUE_GEQ);
  SRB_REQUIRE(r == CUDA_SUCCESS, "cuStreamWaitValue32 failed (%d)", static_cast<int>(r));
  return 0;
}

}  // namespace srb
