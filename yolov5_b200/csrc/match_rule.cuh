// The detection<->label matching rule of process_batch (utils/metrics.py:255-264), shared by the box path (match_kernel,
// post_kernels.cu) and the mask path (match_iou_kernel, mask_metrics.cu).
#pragma once
#include <stdint.h>

namespace y5 {

constexpr int kMatchMaxDet = 4096;

// Called by every thread of a block that owns one image.  s_best[d] / s_iou[d]: detection d's best same-class label (-1: none)
// and that IoU, for d < n.  d is a true positive at threshold t when that IoU >= iouv[t] and no lower-index detection claims
// the same label at t (np.unique keeps the first detection per label).  Rows n..max_det-1 of `correct` are zeroed.
__device__ __forceinline__ void match_assign(const int* s_best, const float* s_iou, int n, int max_det, const float* __restrict__ iouv,
                                             int niou, uint8_t* __restrict__ correct) {
    for (int i = threadIdx.x; i < n * niou; i += blockDim.x) {
        const int d = i / niou, t = i - d * niou;
        const float thr = iouv[t];
        const int bl = s_best[d];
        bool ok = bl >= 0 && s_iou[d] >= thr;
        for (int e = 0; ok && e < d; ++e)
            if (s_best[e] == bl && s_iou[e] >= thr) ok = false;
        correct[static_cast<long long>(d) * niou + t] = ok ? 1 : 0;
    }
    for (int i = n * niou + threadIdx.x; i < max_det * niou; i += blockDim.x) correct[i] = 0;
}

}  // namespace y5
