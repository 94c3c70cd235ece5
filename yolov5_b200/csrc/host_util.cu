#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <set>
#include <utility>

#include "../../include/y5b200.h"
#include "host_util.h"

namespace y5 {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int launch_args(const char* what, const void* kernel, const LaunchDims& d, void** args) {
    static const bool pdl_on = [] { const char* e = getenv("Y5_PDL"); return !(e && e[0] == '0'); }();
    cudaLaunchAttribute attr[2];
    unsigned n = 0;
    if (d.pdl && pdl_on) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n++].val.programmaticStreamSerializationAllowed = 1;
    }
    if (d.cluster > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n++].val.clusterDim = {d.cluster, 1, 1};
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = d.grid;
    cfg.blockDim = d.block;
    cfg.dynamicSmemBytes = d.smem;
    cfg.stream = d.stream;
    cfg.attrs = attr;
    cfg.numAttrs = n;
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaLaunchKernelExC(&cfg, kernel, args);
    const cudaError_t last = cudaGetLastError();
    if (e == cudaSuccess) e = last;
    if (e != cudaSuccess) return set_error(int(e), "%s launch failed: %s", what, cudaGetErrorString(e));
    return 0;
}

int grid_stride_ctas(long long total, int threads, int ctas_per_sm) {
    const long long ctas = (total + threads - 1) / threads, cap = static_cast<long long>(sm_count()) * ctas_per_sm;
    return static_cast<int>(ctas < cap ? ctas : cap);
}

int sm_count() {
    static int per_dev[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    int n = per_dev[dev];
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        per_dev[dev] = n;
    }
    return n;
}

cudaError_t ensure_dyn_smem(const void* kernel, int bytes) {
    static std::mutex mu;
    static std::set<std::pair<const void*, int>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    const auto key = std::make_pair(kernel, dev);
    if (done.count(key)) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done.insert(key);
    return e;
}

static void* driver_entry(const char* name) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return fn;
}
EncodeTiledFn driver_fn_encode_tiled() {
    static EncodeTiledFn fn = reinterpret_cast<EncodeTiledFn>(driver_entry("cuTensorMapEncodeTiled"));
    return fn;
}
EncodeIm2colFn driver_fn_encode_im2col() {
    static EncodeIm2colFn fn = reinterpret_cast<EncodeIm2colFn>(driver_entry("cuTensorMapEncodeIm2col"));
    return fn;
}

CUtensorMapSwizzle swizzle_for_row_bytes(int row_bytes) {
    return row_bytes >= 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}
CUtensorMapDataType tm_dtype(int dtype) { return dtype == Y5_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16; }

// L2 promotion (the granularity at which a TMA read pulls its neighbourhood into L2): 256 B helps when the bytes next to a box
// are read soon after (the next channel chunk of the same pixels, the next pixel of a dense tensor); on a channel SLICE of a
// wider tensor (a C3 branch reading one half of the stacked cv1|cv2 output: 128 B out of every 256 B) it doubles the DRAM reads
// (ncu, yolov5l model.2.m*.cv1: 417 MB read for a 210 MB operand).  -> never promote beyond the slice's own contiguous bytes.
static CUtensorMapL2promotion promotion_for(unsigned long long row_bytes, unsigned long long pitch_bytes) {
    if (row_bytes == pitch_bytes || row_bytes >= 256) return CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    if (row_bytes >= 128) return CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
    if (row_bytes >= 64) return CU_TENSOR_MAP_L2_PROMOTION_L2_64B;
    return CU_TENSOR_MAP_L2_PROMOTION_NONE;
}

int encode_tiled(CUtensorMap* map, int dtype, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                 const cuuint32_t* box, CUtensorMapSwizzle sw, const char* what) {
    auto fn = driver_fn_encode_tiled();
    if (!fn) return set_error(Y5_E_DRIVER, "cuTensorMapEncodeTiled entry point not available");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, tm_dtype(dtype), rank, const_cast<void*>(base), dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    sw, promotion_for(dims[0] * 2, rank > 1 ? strides_bytes[0] : dims[0] * 2), CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error(Y5_E_DRIVER, "cuTensorMapEncodeTiled(%s) failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u stride0 %llu",
                         what, int(r), rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                         (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1],
                         rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, (unsigned long long)strides_bytes[0]);
    return 0;
}

int encode_im2col(CUtensorMap* map, int dtype, const void* base, int C, int W, int H, int N, long long xs, long long ys, long long ns,
                  int kh, int kw, int stride, int pad_h, int pad_w, uint32_t channels_per_pixel, uint32_t pixels_per_column,
                  CUtensorMapSwizzle sw) {
    auto fn = driver_fn_encode_im2col();
    if (!fn) return set_error(Y5_E_DRIVER, "cuTensorMapEncodeIm2col entry point not available");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)xs * 2, (cuuint64_t)ys * 2, (cuuint64_t)ns * 2};
    // Bounding box of filter-window base pixels: lower corner = -pad, upper corner = pad - (k-1) (dilation 1),
    // relative to the tensor's first / last pixel; the window taps {s, r} are passed per copy as im2col offsets.
    int lower[2] = {-pad_w, -pad_h};
    int upper[2] = {pad_w - (kw - 1), pad_h - (kh - 1)};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = fn(map, tm_dtype(dtype), 4, const_cast<void*>(base), dims, strides, lower, upper, channels_per_pixel, pixels_per_column,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, promotion_for((unsigned long long)C * 2, (unsigned long long)xs * 2),
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error(Y5_E_DRIVER, "cuTensorMapEncodeIm2col failed (%d): C %d W %d H %d N %d k %dx%d s %d p %d,%d", int(r), C, W, H, N,
                         kh, kw, stride, pad_h, pad_w);
    // Driver-side quirk also worked around by CUTLASS (cute/atom/copy_traits_sm90_im2col.hpp): for tensors smaller
    // than 128 KiB, drivers <= 13.1 set a descriptor bit that makes the im2col walk fault; clear it.
    int drv = 0;
    cudaDriverGetVersion(&drv);
    const unsigned long long span = (unsigned long long)N * ns * 2;
    if (drv <= 13010 && span < 131072ull) reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
    return 0;
}


}  // namespace y5

extern "C" Y5_API int y5_version(void) { return 2; }
extern "C" Y5_API const char* y5_last_error(void) { return y5::g_err; }
extern "C" Y5_API int64_t y5_launch_count(void) { return y5::g_launches.load(std::memory_order_relaxed); }
