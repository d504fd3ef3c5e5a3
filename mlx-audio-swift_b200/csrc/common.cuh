// Shared plumbing for libb200audio: status codes, error text, launch counting, device buffers, and the small device
// helpers every engine uses (warp / block sums, range-reduced sin).  sm_90a only; no CPU fallback anywhere.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200audio_internal.h"

namespace b2a {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

void set_last_error(const std::string& msg);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define B2A_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess)                                                                  \
            throw b2a::Error(B2A_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

#define B2A_CHECK(cond, code, msg)                         \
    do {                                                   \
        if (!(cond)) throw b2a::Error((code), (msg));      \
    } while (0)

// Runs `fn`, maps exceptions to status codes (never lets one cross the C ABI).
template <class F>
static inline int32_t guarded(F&& fn) {
    try {
        fn();
        return B2A_OK;
    } catch (const Error& e) {
        set_last_error(e.what());
        return e.code;
    } catch (const std::exception& e) {
        set_last_error(e.what());
        return B2A_ERR_GENERATION_FAILED;
    } catch (...) {
        set_last_error("unknown error");
        return B2A_ERR_GENERATION_FAILED;
    }
}

void require_device(int device);  // throws B2A_ERR_CUDA when there is no usable device

// RAII device buffer (cudaMalloc / cudaFree), grow-only resize.
template <class T>
struct DBuf {
    T* p = nullptr;
    size_t n = 0;
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    DBuf(DBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    ~DBuf() { if (p) cudaFree(p); }
    void alloc(size_t count) {
        if (count <= n) return;
        if (p) cudaFree(p);
        p = nullptr;
        B2A_CUDA(cudaMalloc(&p, count * sizeof(T)));
        n = count;
    }
    void upload(const T* host, size_t count, cudaStream_t s = 0) {
        alloc(count);
        B2A_CUDA(cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, s));
    }
};

// Pinned host staging buffer, grow-only.
template <class T>
struct HBuf {
    T* p = nullptr;
    size_t n = 0;
    HBuf() = default;
    HBuf(const HBuf&) = delete;
    HBuf& operator=(const HBuf&) = delete;
    ~HBuf() { if (p) cudaFreeHost(p); }
    void alloc(size_t count) {
        if (count <= n) return;
        if (p) cudaFreeHost(p);
        p = nullptr;
        B2A_CUDA(cudaMallocHost(&p, count * sizeof(T)));
        n = count;
    }
};

// Named-tensor lookup over the b2a_tensor table passed across the ABI.
struct TensorTable {
    std::map<std::string, const b2a_tensor*> m;
    TensorTable(const b2a_tensor* t, int n) {
        for (int i = 0; i < n; ++i) m[t[i].name] = &t[i];
    }
    const b2a_tensor* find(const std::string& name) const {
        auto it = m.find(name);
        return it == m.end() ? nullptr : it->second;
    }
    const b2a_tensor& get(const std::string& name) const {
        auto* t = find(name);
        if (!t) throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "missing tensor: " + name);
        return *t;
    }
    static int64_t numel(const b2a_tensor& t) {
        int64_t n = 1;
        for (int i = 0; i < t.ndim; ++i) n *= t.shape[i];
        return n;
    }
    // fp32 copy of a tensor of dtype f32 or bf16
    std::vector<float> f32(const std::string& name, int64_t expect_numel = -1) const {
        const b2a_tensor& t = get(name);
        int64_t n = numel(t);
        if (expect_numel >= 0 && n != expect_numel)
            throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "bad shape for tensor: " + name);
        std::vector<float> v(n);
        if (t.dtype == B2A_DTYPE_F32) {
            memcpy(v.data(), t.data, n * sizeof(float));
        } else if (t.dtype == B2A_DTYPE_BF16) {
            const uint16_t* s = (const uint16_t*)t.data;
            for (int64_t i = 0; i < n; ++i) {
                uint32_t u = (uint32_t)s[i] << 16;
                memcpy(&v[i], &u, 4);
            }
        } else {
            throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "bad dtype for tensor: " + name);
        }
        return v;
    }
};

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Programmatic dependent launch (PDL): every kernel of the decode step is launched with
// programmaticStreamSerializationAllowed so that its prologue (barrier init and -- for the
// GEMMs -- the TMA prefetch of the first ring-full of WEIGHTS, which never depend on the previous kernel) overlaps
// with the tail of the kernel before it.  Device side: pdl_trigger() lets the next kernel start launching,
// pdl_wait() blocks until the previous kernel has completed and its writes are visible.  B2A_PDL=0 disables it.
bool pdl_enabled();

template <class... KArgs, class... Args>
static inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    B2A_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...));
    count_launch();
}

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// sum over a CTA of THREADS threads; red holds THREADS / 32 floats
template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < THREADS / 32; ++i) t += red[i];
    return t;
}

// sin with an explicit two-term 2*pi range reduction + MUFU.SIN: |error| < 5e-7 for |x| < 1e4 (the libdevice sinf slow
// path costs ~40 dependent instructions per call and made every Snake epilogue issue bound)
__device__ __forceinline__ float fast_sin(float x) {
    const float k = rintf(x * 0.15915494309189535f);
    float r = fmaf(k, -6.28318548202514648f, x);
    r = fmaf(k, 1.7484555e-7f, r);
    return __sinf(r);
}
#endif

}  // namespace b2a
