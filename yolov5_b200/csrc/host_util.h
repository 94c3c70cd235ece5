// Host-side helpers shared by the translation units of liby5b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

namespace y5 {

// records a thread-local message retrievable through y5_last_error(); returns `code`
int set_error(int code, const char* fmt, ...);
int sm_count();
// CTAs for a grid-stride loop over `total` items: one item per thread, at most `ctas_per_sm` CTAs per SM
int grid_stride_ctas(long long total, int threads, int ctas_per_sm);
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

struct LaunchDims {
    dim3 grid, block;
    size_t smem;
    cudaStream_t stream;
    // programmatic dependent launch: the kernel may be scheduled while its predecessor in the stream drains, so it must
    // begin with griddep_wait().  Y5_PDL=0 turns the attribute off.
    bool pdl = false;
    unsigned cluster = 1;  // CTAs per cluster along x
};

int launch_args(const char* what, const void* kernel, const LaunchDims& d, void** args);

// Every kernel of the library is launched here: counts one launch for y5_launch_count() and returns 0, or records
// "<what> launch failed: ..." and returns the CUDA error code.  The thread's last runtime error is read and cleared too, so
// an earlier unchecked runtime call of the entry point surfaces here and no error is left behind for the caller.
template <typename... KArgs, typename... Args>
int launch(const char* what, void (*kernel)(KArgs...), const LaunchDims& d, Args&&... args) {
    return [&](KArgs... coerced) {
        void* ptrs[] = {&coerced..., nullptr};
        return launch_args(what, reinterpret_cast<const void*>(kernel), d, ptrs);
    }(std::forward<Args>(args)...);
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, and one process
// may drive several GPUs (DataParallel, a model on cuda:1 while cuda:0 is current ...)
cudaError_t ensure_dyn_smem(const void* kernel, int bytes);

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
using EncodeIm2colFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// resolved through cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda
EncodeTiledFn driver_fn_encode_tiled();
EncodeIm2colFn driver_fn_encode_im2col();


CUtensorMapSwizzle swizzle_for_row_bytes(int row_bytes);
CUtensorMapDataType tm_dtype(int dtype);
// tiled tensor map of `rank` dims (innermost first); on failure records a message and returns Y5_E_DRIVER
int encode_tiled(CUtensorMap* map, int dtype, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                 const cuuint32_t* box, CUtensorMapSwizzle sw, const char* what);
// im2col tensor map over an NHWC view (element strides xs/ys/ns), filter kh x kw, conv stride / padding
int encode_im2col(CUtensorMap* map, int dtype, const void* base, int C, int W, int H, int N, long long xs, long long ys, long long ns,
                  int kh, int kw, int stride, int pad_h, int pad_w, uint32_t channels_per_pixel, uint32_t pixels_per_column,
                  CUtensorMapSwizzle sw);

}  // namespace y5
