// sam_road_b200 :: common device/host helpers for sm_90a.
//
// Thin inline-PTX wrappers for the Hopper primitives the hot path uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors),
// plus small math helpers shared by the kernels.  Nothing here is a port of
// reference code: the reference (htcr/sam_road) ships no CUDA at all
// (SURVEY.md §2.2); these are the building blocks of the native path.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srb {

// ----------------------------------------------------------------------------------------------
// error plumbing (C-ABI never throws: every entry point returns an int and stores a message)
// ----------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define SRB_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::srb::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                  \
                            cudaGetErrorString(_e));                                       \
      return 1;                                                                            \
    }                                                                                      \
  } while (0)

#define SRB_REQUIRE(cond, ...)                                                             \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      ::srb::set_last_error(__VA_ARGS__);                                                  \
      return 2;                                                                            \
    }                                                                                      \
  } while (0)

// Return the status of a call that already set the error message, when it is not 0.
#define SRB_TRY(expr)                                                                      \
  do {                                                                                     \
    if (int _rc = (expr)) return _rc;                                                      \
  } while (0)

// ----------------------------------------------------------------------------------------------
// kernel launch: every kernel goes on a stream through SRB_LAUNCH
// ----------------------------------------------------------------------------------------------
// Reads the launch's error right away, so that a bad configuration is reported at its own call site and not
// by the next unrelated check, and counts one launch when it was enqueued (samroad_launch_count).  Returns 0,
// or 1 with "<file>:<line>: SRB_LAUNCH(<arguments>) -> <error>" set.
int launched(const char* file, int line, const char* call);

template <typename... Params, typename... Args>
int launch(const char* file, int line, const char* call, void (*kernel)(Params...), dim3 grid, dim3 block,
           size_t smem, cudaStream_t stream, Args&&... args) {
  kernel<<<grid, block, smem, stream>>>(static_cast<Args&&>(args)...);
  return launched(file, line, call);
}

// SRB_LAUNCH(kernel, grid, block, smem, stream, kernel arguments...) launches with <<<grid, block, smem, stream>>>
// and returns the error status from the calling function when the launch fails.  The kernel may be a template
// specialisation with commas in its argument list, or a pointer.
#define SRB_LAUNCH(...) SRB_TRY(::srb::launch(__FILE__, __LINE__, #__VA_ARGS__, __VA_ARGS__))

// Lets `kernel` take `bytes` of dynamic shared memory on the current device.  The attribute is only ever
// raised, once per size above what was set before for that kernel and device, so launchers may call it before
// every launch, from any host thread.
int allow_dynamic_smem(const void* kernel, size_t bytes);
template <typename... Params>
int allow_dynamic_smem(void (*kernel)(Params...), size_t bytes) {
  return allow_dynamic_smem(reinterpret_cast<const void*>(kernel), bytes);
}

// ----------------------------------------------------------------------------------------------
// resources: every handle owns its memory through these, so destructors free it
// ----------------------------------------------------------------------------------------------
// Move-only owner of one cudaMalloc (kPinned: cudaMallocHost) block.  reserve() replaces the block only
// when `bytes` exceeds the capacity and allocates exactly `bytes`; on failure it clears the runtime's last
// error, sets "<what>: out of device memory (<n> bytes)", leaves the buffer empty and returns 1.  It never
// synchronises: a caller whose queued work may still use the old block synchronises before calling it.
template <bool kPinned>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
  Buffer& operator=(Buffer&& o) noexcept {
    if (this != &o) {
      release();
      p_ = o.p_;
      cap_ = o.cap_;
      o.p_ = nullptr;
      o.cap_ = 0;
    }
    return *this;
  }
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  ~Buffer() { release(); }

  int reserve(size_t bytes, const char* what);
  void release();
  void* get() const { return p_; }
  template <typename T> T* as() const { return static_cast<T*>(p_); }
  size_t capacity() const { return cap_; }

 private:
  void* p_ = nullptr;
  size_t cap_ = 0;
};
using DeviceBuffer = Buffer<false>;
using PinnedBuffer = Buffer<true>;

__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Blocks of `per` elements that cover n elements: a grid size.
inline int blocks_for(long long n, int per) { return static_cast<int>((n + per - 1) / per); }

// Bump allocator over a workspace.  Each workspace has one function that takes its regions in order; called
// with a null base it only counts (bytes() is then the size to allocate, and what take() returns is an
// offset, not a pointer), called with the allocation it carves the same regions.  Every region starts at a
// multiple of `align` from the base.
class Layout {
 public:
  __host__ __device__ explicit Layout(void* base, size_t align = 256)
      : base_(reinterpret_cast<uintptr_t>(base)), align_(align) {}
  template <typename T>
  __host__ __device__ T* take(size_t count) {
    T* p = reinterpret_cast<T*>(base_ + off_);
    off_ += align_up(sizeof(T) * count, align_);
    return p;
  }
  __host__ __device__ size_t bytes() const { return off_; }

 private:
  uintptr_t base_;
  size_t align_;
  size_t off_ = 0;
};

// The shared start of every *_create: a device exists, `device` names one, and it becomes current.
int open_device(int device);

// CSR adjacency from outside: offsets start at 0 and never decrease, every neighbour is in [0, n), and the
// neighbour list is present when it is not empty.  Messages start with `what`.
int check_csr(const char* what, int32_t n, const int32_t* start, const int32_t* list);

// ----------------------------------------------------------------------------------------------
// small device helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Element-wise fp32x2 add / fma, each lane rounded as its scalar counterpart.
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// Fast erf-GELU for GEMM epilogues: gelu(x) = relu(x) - |x| * 0.5*erfc(|x|/sqrt2), with
// log2(0.5*erfc(a/sqrt2)) fitted by a degree-4 polynomial on [0, 5.6] (clamped beyond, where the term
// is < 1e-7).  4 FMA + 1 MUFU.EX2 + 3 ALU; max abs error 6.1e-6 (fit + error scan in DESIGN.md "GELU"):
// 1 % of the half-ulp of the fp16 value the result is rounded to at |gelu| ~ 1, and below the fp16
// half-ulp everywhere above |gelu| = 0.016.  Two elements at a time; the polynomial is evaluated in
// t = -min(|x|, 5.6) (odd coefficients negated).
__device__ __forceinline__ float2 gelu_erf_fast2(float2 x) {
  const float2 na = make_float2(fminf(x.x, -x.x), fminf(x.y, -x.y));
  const float2 t = make_float2(fmaxf(na.x, -5.6f), fmaxf(na.y, -5.6f));
  float2 l = ffma2(make_float2(0.0038648627f, 0.0038648627f), t, make_float2(0.044072032f, 0.044072032f));
  l = ffma2(l, t, make_float2(-0.46802717f, -0.46802717f));
  l = ffma2(l, t, make_float2(1.1473644f, 1.1473644f));
  l = ffma2(l, t, make_float2(-1.0004811f, -1.0004811f));
  float2 e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(l.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(l.y));
  return ffma2(na, e, make_float2(fmaxf(x.x, 0.0f), fmaxf(x.y, 0.0f)));
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) -- SASS: UTMALDG
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)),
      "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, const void* smem_src, int32_t c0,
                                             int32_t c1, int32_t c2, int32_t c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2),
               "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)),
      "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a) -- SASS: HGMMA
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle, rows of 64 fp16 (=128 B) as
// written by a 128B-swizzled TMA box.  8-row swizzle atoms are 1024 B apart (SBO); LBO is unused
// for swizzled K-major layouts.  Advancing 16 elements (32 B) along K inside the atom is +2 on the
// start-address field.
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);        // start address >> 4
  d |= static_cast<uint64_t>(1) << 16;                           // leading byte offset (unused)
  d |= static_cast<uint64_t>(1024u >> 4) << 32;                  // stride byte offset = 1024 B
  d |= static_cast<uint64_t>(1) << 62;                           // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMA
template <int R>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup (all its warps execute it): producers give registers to consumers
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Accumulator fragment of wgmma m64nNk16 (f32): register i of thread (warp w of the warpgroup, lane l)
// holds row 16*w + l/4 + 8*((i>>1)&1), column 8*(i>>2) + 2*(l&3) + (i&1).
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b,
                                             uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b,
                                             uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}


// ----------------------------------------------------------------------------------------------
// host: TMA descriptor construction (driver entry point fetched at run time; no -lcuda needed)
// ----------------------------------------------------------------------------------------------
// 2D fp16 row-major tensor [rows][cols] (cols contiguous, row pitch `ld` elements), box
// [box_rows][64 cols], 128B swizzle.  Out-of-bounds elements read as zero.
int make_tmap_f16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                     uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols = 64);

// 2D fp32 row-major tensor [rows][cols] (row pitch `ld` elements), box [box_rows][32 cols] (128 B), 128B swizzle.
int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                     uint32_t box_rows);

// 4D fp16 view [d3][d2][d1][d0] (d0 contiguous; strides in elements for d1..d3), box {b0,b1,b2,b3},
// 128B swizzle (b0 * 2 bytes must be 128).  Out-of-bounds elements read as zero.
int make_tmap_f16_4d(CUtensorMap* out, const void* base, const uint64_t dims[4],
                     const uint64_t strides_elems[3], const uint32_t box[4]);
int make_tmap_f32_4d_dense(CUtensorMap* out, const void* base, const uint64_t dims[4],
                           const uint64_t strides_bytes[3], const uint32_t box[4]);

}  // namespace srb
