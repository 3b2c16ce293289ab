// Device string gather for get_matches (SURVEY.md §8f row 1), for sm_90a.
//
// StringGrouper.get_matches (string_grouper/string_grouper.py:455-468) gathers the left and
// right strings of every match by position (`Series.iloc[matches_list.master_side]`).  The packed strings are
// already in HBM for K1 and the match positions are there after K4, so the gather runs on the device and one
// contiguous (offsets, bytes) pair per side goes back to the host, where it is wrapped as an Arrow string array
// without touching the individual strings.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

__global__ void gather_len_kernel(const int64_t *__restrict__ offsets, int64_t doc_base, int64_t n_sel,
                                  const int32_t *__restrict__ pos, int64_t *__restrict__ len) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_sel) {
        const int64_t d = doc_base + pos[i];
        len[i] = offsets[d + 1] - offsets[d];
    } else if (i == n_sel) {
        len[i] = 0;
    }
}

// one warp per selected string
__global__ void gather_bytes_kernel(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ offsets,
                                    int64_t doc_base, int64_t n_sel, const int32_t *__restrict__ pos,
                                    const int64_t *__restrict__ out_offsets, uint8_t *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n_sel) return;
    const int64_t d = doc_base + pos[i];
    const int64_t s = offsets[d], n = offsets[d + 1] - s, o = out_offsets[i];
    for (int64_t k = lane_id(); k < n; k += 32) out[o + k] = bytes[s + k];
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_gather_workspace_bytes(int64_t n_sel) {
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, (int64_t *)nullptr, (int64_t *)nullptr, n_sel + 1);
    return align_up((size_t)(n_sel + 2) * 8, 256) + align_up(b, 256) + 1024;
}

// out_offsets[n_sel+1]: start of every selected string in the gathered byte buffer; out_offsets[n_sel] = total bytes.
int sg_gather_offsets(const int64_t *offsets, int64_t doc_base, int64_t n_sel, const int32_t *positions,
                      int64_t *out_offsets, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_sel < 0) return fail(SG_ERR_INVALID, "negative n_sel");
    Arena ar(ws, ws_bytes);
    int64_t *len = ar.take<int64_t>((size_t)n_sel + 2);
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, len, out_offsets, n_sel + 1);
    char *tmp = ar.take<char>(b);
    if (!ar.ok()) return fail(SG_ERR_INVALID, "gather workspace too small (%zu < %zu)", ws_bytes, ar.off);
    gather_len_kernel<<<(unsigned)((n_sel + 1 + 255) / 256), 256, 0, st>>>(offsets, doc_base, n_sel, positions, len);
    SG_LAUNCH_CHECK();
    SG_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, b, len, out_offsets, n_sel + 1, st));
    return SG_OK;
}

int sg_gather_bytes(const uint8_t *bytes, const int64_t *offsets, int64_t doc_base, int64_t n_sel,
                    const int32_t *positions, const int64_t *out_offsets, uint8_t *out_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_sel <= 0) return SG_OK;
    gather_bytes_kernel<<<(unsigned)((n_sel + 7) / 8), 256, 0, st>>>(bytes, offsets, doc_base, n_sel, positions,
                                                                     out_offsets, out_bytes);
    SG_LAUNCH_CHECK();
    return SG_OK;
}

}  // extern "C"
