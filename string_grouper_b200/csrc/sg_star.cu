// Star groups on the device, for sm_90a: group_similar_strings(linkage='star').
//
// Greedy star clustering (the pivot rule) of the match graph.  Serial statement: visit the strings in rank order; a
// string not yet assigned becomes a pivot and takes every unassigned neighbour.  rep[v] is the pivot of v's group,
// so every string is its own representative or directly matched to it.  Ranks: 'first' orders by index, 'centroid'
// by the similarity sum of sg_group_reps (same bits) descending, then by index.
//
// The serial rule runs in rounds with the same result.  From the states at the start of a round, pv[v] = the smallest
// rank among v's pivot neighbours and blk[v] = the smallest rank among its undecided neighbours.  v is ready once
// blk[v] > min(pv[v], rank[v]): every neighbour ranked below that minimum is then decided and no pivot, which is all
// the serial rule looks at before v's turn.  A ready v becomes a pivot if pv[v] > rank[v] and joins the pivot of rank
// pv[v] otherwise.  The undecided string of smallest rank is always ready, so every round decides at least one
// string and the loop ends on every input; real match lists need about a dozen rounds, a path whose ranks increase
// along it needs one round per string.
#include <cub/cub.cuh>

#include "sg_common.cuh"

namespace sg {

constexpr int32_t STAR_NONE = 0x7f7f7f7f;      // the byte-wise 0x7f fill: above every rank (n < STAR_NONE)
constexpr int STAR_ROUNDS_PER_CHECK = 8;       // rounds between two read-backs of the decided count

// ascending key = similarity sum descending; -0.0 and +0.0 share one key, as they compare equal on the host
__global__ void star_key_kernel(int64_t n, const double *__restrict__ weight, unsigned long long *__restrict__ key) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long b = (unsigned long long)__double_as_longlong(__dadd_rn(weight[i], 0.0));
    key[i] = (b >> 63) ? b : ~(b | 0x8000000000000000ull);      // complement of the order-preserving bits
}

// rank[order[k]] = k; order_in is the identity that the stable sort permuted
__global__ void star_rank_kernel(int64_t n, const int32_t *__restrict__ order, int32_t *__restrict__ rank) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) rank[order[k]] = (int32_t)k;
}

__global__ void star_iota_kernel(int64_t n, int32_t *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)i;
}

// One pass over the stored pairs, both directions (the list may be asymmetric).  rep[]: -1 undecided, rep[v] == v
// pivot, anything else a member.  Pairs whose ends are both decided change nothing.
__global__ void star_edge_kernel(int64_t nnz, const int32_t *__restrict__ row, const int32_t *__restrict__ col,
                                 const int32_t *__restrict__ rank, const int32_t *__restrict__ rep,
                                 int32_t *__restrict__ pv, int32_t *__restrict__ blk) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const int32_t u = row[e], v = col[e];
    if (u == v) return;
    const int32_t su = rep[u], sv = rep[v];
    if (su < 0 && sv < 0) {
        atomicMin(blk + u, rank[v]);
        atomicMin(blk + v, rank[u]);
    } else if (su < 0) {
        if (sv == v) atomicMin(pv + u, rank[v]);
    } else if (sv < 0) {
        if (su == u) atomicMin(pv + v, rank[u]);
    }
}

// One pass over the strings: decides the ready ones, *decided += their number, clears blk of the others for the
// next round (pv keeps its pivots: a pivot stays one).
__global__ void star_decide_kernel(int64_t n, const int32_t *__restrict__ rank, const int32_t *__restrict__ order,
                                   const int32_t *__restrict__ pv, int32_t *__restrict__ blk, int32_t *__restrict__ rep,
                                   unsigned long long *__restrict__ decided) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool now = false;
    if (i < n && rep[i] < 0) {
        const int32_t r = rank[i], p = pv[i];
        if (blk[i] > (p < r ? p : r)) {
            rep[i] = p < r ? order[p] : (int32_t)i;
            now = true;
        } else {
            blk[i] = STAR_NONE;
        }
    }
    const unsigned votes = __ballot_sync(FULL, now);
    if (lane_id() == 0 && votes) atomicAdd(decided, (unsigned long long)__popc(votes));
}

static size_t star_sort_bytes(int64_t n) {
    size_t b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                    (int32_t *)nullptr, (int32_t *)nullptr, n);
    return b;
}

}  // namespace sg

using namespace sg;

extern "C" {

size_t sg_group_star_workspace_bytes(int64_t n) {
    const size_t i32 = align_up((size_t)(n + 1) * 4, 256), u64 = align_up((size_t)(n + 1) * 8, 256);
    return 5 * i32 + 4 * u64 + align_up(star_sort_bytes(n), 256) + 1024;
}

// Matches (row, col, score) sorted by row over n strings -> rep[i] = the pivot of i's star group.  centroid = 0:
// strings ranked by index; 1: by similarity sum descending, then index.  Reads one counter back every
// STAR_ROUNDS_PER_CHECK rounds; the rounds after the last one change nothing.
int sg_group_star(int64_t n, int64_t nnz, const int32_t *row, const int32_t *col, const double *score, int centroid,
                  int32_t *rep, void *ws, size_t ws_bytes, void *stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n <= 0) return SG_OK;
    if (n >= STAR_NONE) return fail(SG_ERR_INVALID, "star groups: %lld strings, at most %d", (long long)n, STAR_NONE - 1);
    Arena ar(ws, ws_bytes);
    int32_t *rank = ar.take<int32_t>((size_t)n + 1);
    int32_t *order = ar.take<int32_t>((size_t)n + 1);
    int32_t *iota = ar.take<int32_t>((size_t)n + 1);
    int32_t *pv = ar.take<int32_t>((size_t)n + 1);
    int32_t *blk = ar.take<int32_t>((size_t)n + 1);
    double *weight = ar.take<double>((size_t)n + 1);
    unsigned long long *best = ar.take<unsigned long long>((size_t)n + 1);
    unsigned long long *key = ar.take<unsigned long long>((size_t)n + 1);
    unsigned long long *key_sorted = ar.take<unsigned long long>((size_t)n + 1);
    size_t sort_bytes = star_sort_bytes(n);
    void *sort_tmp = ar.take<char>(sort_bytes);
    unsigned long long *decided = best + n;      // best[n] is not part of the row sums' scratch
    if (!ar.ok()) return fail(SG_ERR_INVALID, "star workspace too small (%zu < %zu)", ws_bytes, ar.off);
    const unsigned gn = (unsigned)((n + 255) / 256);
    const unsigned ge = (unsigned)((nnz + 255) / 256);

    if (centroid) {
        // iota = identity labels of the row sums, then the values the stable sort permutes into the rank order
        int rc = group_row_weights(n, nnz, row, score, iota, weight, best, st);
        if (rc != SG_OK) return rc;
        star_key_kernel<<<gn, 256, 0, st>>>(n, weight, key);
        SG_LAUNCH_CHECK();
        SG_CUDA_TRY(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, key, key_sorted, iota, order, n, 0, 64, st));
        star_rank_kernel<<<gn, 256, 0, st>>>(n, order, rank);
        SG_LAUNCH_CHECK();
    } else {
        star_iota_kernel<<<gn, 256, 0, st>>>(n, rank);
        SG_LAUNCH_CHECK();
        order = rank;
    }
    SG_CUDA_TRY(cudaMemsetAsync(rep, 0xff, (size_t)n * 4, st));
    SG_CUDA_TRY(cudaMemsetAsync(pv, 0x7f, (size_t)n * 4, st));
    SG_CUDA_TRY(cudaMemsetAsync(blk, 0x7f, (size_t)n * 4, st));
    SG_CUDA_TRY(cudaMemsetAsync(decided, 0, sizeof(unsigned long long), st));
    unsigned long long done = 0, before = 0;
    for (int64_t round = 1;; ++round) {
        if (nnz > 0) {
            star_edge_kernel<<<ge, 256, 0, st>>>(nnz, row, col, rank, rep, pv, blk);
            SG_LAUNCH_CHECK();
        }
        star_decide_kernel<<<gn, 256, 0, st>>>(n, rank, order, pv, blk, rep, decided);
        SG_LAUNCH_CHECK();
        if (round % STAR_ROUNDS_PER_CHECK) continue;
        SG_CUDA_TRY(cudaMemcpyAsync(&done, decided, sizeof(done), cudaMemcpyDeviceToHost, st));
        SG_CUDA_TRY(cudaStreamSynchronize(st));
        if (done >= (unsigned long long)n) break;
        // every round decides a string; no progress means indices outside [0, n) in the list
        if (done == before) return fail(SG_ERR_INVALID, "star groups made no progress (%llu of %lld decided)", done,
                                        (long long)n);
        before = done;
    }
    return SG_OK;
}

}  // extern "C"
