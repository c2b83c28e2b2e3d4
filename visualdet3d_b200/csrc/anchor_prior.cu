// The 3-D anchor priors of the reference's det_precompute (scripts/imdb_precompute_3d.py: read_one_split, lines 106-135) on the GPU.
// For every (frame, class) segment of a batch: calc_iou of every anchor against the segment's 2-D boxes, the first-maximum box of each
// anchor (torch.max(dim=1)), positives where that maximum is > fg_iou_threshold, and each box's maximum over all anchors (usable objects).
// Each positive's (z, sin 2a, cos 2a) and its square are added into the bin (scale row, ratio column) of its anchor, in the reference's
// order: frame, then class, then anchor index.  A bin's sums are therefore the reference's sequential float64 sums, bit for bit.
//
// Kernels (one launch each per batch, after a memset of the box keys and a copy of the batch's offsets):
//   prior_iou_kernel<T>: one thread per (segment, anchor), the segment's boxes staged in shared memory.  T is the IoU's dtype (float
//     when the labels are python floats, double when the test augmentation left numpy float64 values: torch.tensor's inference).  Writes
//     the anchor's positive box (or -1) and folds each box's max IoU into an order-independent integer atomicMax key.
//   prior_walk_kernel: one block per (bin, class).  It walks the bin's anchors (ascending index, from the host-built bin order) frame by
//     frame, 1024 (frame, anchor) pairs per step: the step's positives are compacted in order into shared memory, then six lanes of warp
//     0 add them one at a time (three sums, three squares).  No float atomics.  The class's bin-0 block also counts the usable boxes.
// Built with -fmad=false: x * x + s rounds twice, as numpy's squared += x ** 2 does, and calc_iou rounds like torch's elementwise ops.
#include "common.cuh"
#include "loss_common.cuh"
#include <math.h>
#include <string.h>
#include <vector>

namespace vd3d {

constexpr int AP_MAX_K = 512;                   // boxes per (frame, class) segment
constexpr int AP_IOU_THREADS = 256;
constexpr int AP_WALK_THREADS = 512;
constexpr int AP_PER_THREAD = 2;
constexpr int AP_STEP = AP_WALK_THREADS * AP_PER_THREAD;
constexpr int AP_MAX_SEGMENTS = 65535;

template <class T> struct IouOf;
template <> struct IouOf<float> {
    __host__ __device__ static float at(const float* a, const float* b) { return calc_iou(a, b); }
};
template <> struct IouOf<double> {
    __host__ __device__ static double at(const float* a, const double* b) { return calc_iou(a, b); }
};

// IoU >= 0, so the bits of its float64 value order like the value (the float32 IoU widens exactly)
__host__ __device__ inline unsigned long long iou_key(double v) {
    unsigned long long k;
    memcpy(&k, &v, sizeof k);
    return k;
}
__host__ __device__ inline double key_iou(unsigned long long k) {
    double v;
    memcpy(&v, &k, sizeof v);
    return v;
}

// Workspace: [bin_start (n_bins + 1) | offsets (S + 1)] ints, then the positive box of every (segment, anchor) [S][N] int32, then one
// 64-bit key per box, each region 256-byte aligned.
struct PriorLayout {
    size_t ints, flags, keys, total;
};

static PriorLayout prior_layout(int N, int n_bins, int S, int K_total) {
    PriorLayout L;
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    L.ints = 0;
    L.flags = up((size_t)(n_bins + 1 + S + 1) * sizeof(int));
    L.keys = up(L.flags + (size_t)S * N * sizeof(int));
    L.total = L.keys + (size_t)(K_total > 0 ? K_total : 1) * sizeof(unsigned long long);
    return L;
}

template <class T>
__global__ void __launch_bounds__(AP_IOU_THREADS) prior_iou_kernel(const float* __restrict__ anchors, int N, const int* __restrict__ offsets,
                                                                   const T* __restrict__ boxes, T thr, int* __restrict__ flags,
                                                                   unsigned long long* __restrict__ gt_key) {
    __shared__ T s_box[AP_MAX_K * 4];
    __shared__ unsigned long long s_key[AP_MAX_K];
    const int s = blockIdx.y;
    const int k0 = offsets[s], K = offsets[s + 1] - k0;
    const int n = blockIdx.x * AP_IOU_THREADS + threadIdx.x;
    const bool live = n < N;
    if (K <= 0) {
        if (live) flags[(size_t)s * N + n] = -1;
        return;
    }
    for (int i = threadIdx.x; i < K * 4; i += AP_IOU_THREADS) s_box[i] = boxes[(size_t)k0 * 4 + i];
    for (int i = threadIdx.x; i < K; i += AP_IOU_THREADS) s_key[i] = 0ull;
    __syncthreads();
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (live)
        for (int c = 0; c < 4; ++c) a[c] = anchors[(size_t)n * 4 + c];
    const int lane = threadIdx.x & 31;
    T best = 0;
    int arg = 0;
    for (int k = 0; k < K; ++k) {
        const T v = IouOf<T>::at(a, s_box + 4 * k);
        if (k == 0 || v > best) { best = v; arg = k; }               // first maximum, like max(dim=1)
        const unsigned long long key = live ? iou_key((double)v) : 0ull;
        const unsigned hi = __reduce_max_sync(0xffffffffu, (unsigned)(key >> 32));
        const unsigned lo = __reduce_max_sync(0xffffffffu, (unsigned)(key >> 32) == hi ? (unsigned)key : 0u);
        if (lane == 0) atomicMax(s_key + k, ((unsigned long long)hi << 32) | lo);
    }
    if (live) flags[(size_t)s * N + n] = best > thr ? arg : -1;
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += AP_IOU_THREADS)
        if (s_key[i]) atomicMax(gt_key + k0 + i, s_key[i]);
}

__global__ void __launch_bounds__(AP_WALK_THREADS) prior_walk_kernel(const int* __restrict__ order, const int* __restrict__ bin_start, int N,
                                                                     const int* __restrict__ offsets, int B, int T, const double* __restrict__ gt3,
                                                                     const int* __restrict__ flags, const unsigned long long* __restrict__ gt_key,
                                                                     double thr, int f64, long long* __restrict__ examine,
                                                                     double* __restrict__ sums, double* __restrict__ squared,
                                                                     long long* __restrict__ usable) {
    __shared__ double s_val[AP_STEP][3];
    __shared__ int s_warp[AP_WALK_THREADS / 32 + 1];
    const int bin = blockIdx.x, t = blockIdx.y, n_bins = gridDim.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b0 = bin_start[bin], nb = bin_start[bin + 1] - b0;
    const size_t cell = (size_t)t * n_bins + bin;
    // lanes 0..2 of warp 0 carry the three sums, lanes 3..5 the three squares, in registers across the whole batch
    double acc = 0.0;
    if (tid < 6) acc = tid < 3 ? sums[cell * 3 + tid] : squared[cell * 3 + tid - 3];
    long long count = 0;
    const long long total = (long long)B * nb;
    for (long long e0 = 0; e0 < total; e0 += AP_STEP) {
        int g[AP_PER_THREAD], seg[AP_PER_THREAD];
        int mine = 0;
#pragma unroll
        for (int j = 0; j < AP_PER_THREAD; ++j) {
            const long long e = e0 + (long long)tid * AP_PER_THREAD + j;
            g[j] = -1;
            seg[j] = 0;
            if (e < total) {
                const int b = (int)(e / nb), i = (int)(e - (long long)b * nb);
                const int n = order[b0 + i];
                seg[j] = b * T + t;
                if (n >= 0 && n < N) g[j] = flags[(size_t)seg[j] * N + n];
            }
            mine += g[j] >= 0;
        }
        // exclusive prefix of `mine` over the block, in thread order: a shuffle scan per warp, then the warps in order
        int inc = mine;
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        if (tid == 0) {
            int run = 0;
            for (int w = 0; w < AP_WALK_THREADS / 32; ++w) {
                const int v = s_warp[w];
                s_warp[w] = run;
                run += v;
            }
            s_warp[AP_WALK_THREADS / 32] = run;
        }
        __syncthreads();
        int slot = s_warp[warp] + inc - mine;
        const int cnt = s_warp[AP_WALK_THREADS / 32];
#pragma unroll
        for (int j = 0; j < AP_PER_THREAD; ++j)
            if (g[j] >= 0) {
                const double* r = gt3 + (size_t)(offsets[seg[j]] + g[j]) * 3;
                s_val[slot][0] = r[0];
                s_val[slot][1] = r[1];
                s_val[slot][2] = r[2];
                ++slot;
            }
        __syncthreads();
        if (tid < 6) {
            const int c = tid < 3 ? tid : tid - 3;
            for (int k = 0; k < cnt; ++k) {
                const double v = s_val[k][c];
                acc = __dadd_rn(acc, tid < 3 ? v : __dmul_rn(v, v));
            }
        }
        count += cnt;
        __syncthreads();                                             // s_val and s_warp are reused by the next step
    }
    if (tid < 3) sums[cell * 3 + tid] = acc;
    else if (tid < 6) squared[cell * 3 + tid - 3] = acc;
    if (tid == 0) examine[cell] += count;
    if (bin == 0 && tid < 32) {                                      // usable objects of class t: boxes whose max IoU is > thr
        long long u = 0;
        for (int b = 0; b < B; ++b) {
            const int s = b * T + t;
            for (int k = offsets[s] + lane; k < offsets[s + 1]; k += 32) {
                const double m = key_iou(gt_key[k]);
                u += f64 ? m > thr : (float)m > (float)thr;
            }
        }
        for (int o = 16; o > 0; o >>= 1) u += __shfl_down_sync(0xffffffffu, u, o);
        if (lane == 0) usable[t] += u;
    }
}

// Sizes and host-side offsets / bin starts shared by both entries.
static int check_prior_args(const char* who, int N, int n_bins, const int* bin_start, const int* offsets, int B, int T, int K_total) {
    VD3D_REQUIRE(N > 0 && n_bins > 0 && n_bins <= 65535, "%s: N=%d n_bins=%d (N >= 1, 1 <= n_bins <= 65535)", who, N, n_bins);
    VD3D_REQUIRE(B > 0 && T > 0 && T <= 65535 && (long long)B * T <= AP_MAX_SEGMENTS, "%s: B=%d T=%d (B * T <= %d)", who, B, T,
                 AP_MAX_SEGMENTS);
    VD3D_REQUIRE(K_total >= 0, "%s: K_total=%d", who, K_total);
    VD3D_REQUIRE(bin_start[0] == 0 && bin_start[n_bins] == N, "%s: bin_start must run from 0 to N=%d, got %d .. %d", who, N, bin_start[0],
                 bin_start[n_bins]);
    for (int i = 0; i < n_bins; ++i)
        VD3D_REQUIRE(bin_start[i] <= bin_start[i + 1], "%s: bin_start decreases at bin %d", who, i);
    const int S = B * T;
    VD3D_REQUIRE(offsets[0] == 0 && offsets[S] == K_total, "%s: offsets must run from 0 to K_total=%d, got %d .. %d", who, K_total, offsets[0],
                 offsets[S]);
    for (int s = 0; s < S; ++s) {
        const int K = offsets[s + 1] - offsets[s];
        VD3D_REQUIRE(K >= 0 && K <= AP_MAX_K, "%s: segment %d holds %d boxes (0 .. %d)", who, s, K, AP_MAX_K);
    }
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" long long vd3d_anchor_prior_workspace_bytes(int N, int n_bins, int B, int T, int K_total) {
    if (N <= 0 || n_bins <= 0 || n_bins > 65535 || B <= 0 || T <= 0 || (long long)B * T > AP_MAX_SEGMENTS || K_total < 0 ||
        K_total > AP_MAX_K * B * T) {
        set_error("anchor_prior_workspace_bytes: bad sizes N=%d n_bins=%d B=%d T=%d K_total=%d", N, n_bins, B, T, K_total);
        return VD3D_EINVAL;
    }
    return (long long)prior_layout(N, n_bins, B * T, K_total).total;
}

extern "C" int vd3d_anchor_prior_accumulate(const float* anchors, const int* order, const int* bin_start_host, int N, int n_bins,
                                            const int* offsets_host, int B, int T, const void* boxes, int boxes_f64, const double* gt3,
                                            int K_total, double fg_iou_threshold, long long* examine, double* sums, double* squared,
                                            long long* usable, void* workspace, long long workspace_bytes, void* stream) {
    VD3D_REQUIRE(anchors && order && bin_start_host && offsets_host && examine && sums && squared && usable && workspace,
                 "anchor_prior_accumulate: null argument");
    VD3D_REQUIRE(K_total == 0 || (boxes && gt3), "anchor_prior_accumulate: null boxes");
    int rc = check_prior_args("anchor_prior_accumulate", N, n_bins, bin_start_host, offsets_host, B, T, K_total);
    if (rc) return rc;
    const int S = B * T;
    const PriorLayout L = prior_layout(N, n_bins, S, K_total);
    VD3D_REQUIRE(workspace_bytes >= (long long)L.total, "anchor_prior_accumulate: workspace of %lld bytes, need %lld", workspace_bytes,
                 (long long)L.total);
    std::vector<int> ints((size_t)n_bins + 1 + S + 1);
    memcpy(ints.data(), bin_start_host, sizeof(int) * (n_bins + 1));
    memcpy(ints.data() + n_bins + 1, offsets_host, sizeof(int) * (S + 1));
    char* ws = (char*)workspace;
    int* d_bin_start = (int*)(ws + L.ints);
    int* d_offsets = d_bin_start + n_bins + 1;
    int* flags = (int*)(ws + L.flags);
    unsigned long long* keys = (unsigned long long*)(ws + L.keys);
    cudaStream_t st = (cudaStream_t)stream;
    VD3D_CUDA(cudaMemcpyAsync(d_bin_start, ints.data(), ints.size() * sizeof(int), cudaMemcpyHostToDevice, st));   // pageable: staged before return
    if (K_total > 0) VD3D_CUDA(cudaMemsetAsync(keys, 0, (size_t)K_total * sizeof(unsigned long long), st));
    const dim3 grid(cdiv(N, AP_IOU_THREADS), S);
    if (boxes_f64)
        prior_iou_kernel<double><<<grid, AP_IOU_THREADS, 0, st>>>(anchors, N, d_offsets, (const double*)boxes, fg_iou_threshold, flags, keys);
    else
        prior_iou_kernel<float><<<grid, AP_IOU_THREADS, 0, st>>>(anchors, N, d_offsets, (const float*)boxes, (float)fg_iou_threshold, flags,
                                                                  keys);
    VD3D_CHECK_LAUNCH("anchor_prior_iou");
    prior_walk_kernel<<<dim3(n_bins, T), AP_WALK_THREADS, 0, st>>>(order, d_bin_start, N, d_offsets, B, T, gt3, flags, keys,
                                                                   fg_iou_threshold, boxes_f64, examine, sums, squared, usable);
    VD3D_CHECK_LAUNCH("anchor_prior_walk");
    return VD3D_OK;
}

// The same accumulation on the host, in the reference's loop order (frame, class, anchor): the parity checker.
template <class T>
static void prior_host(const float* anchors, const int* bin_of, int N, int n_bins, const int* offsets, int B, int Tn, const T* boxes,
                       const double* gt3, double thr, long long* examine, double* sums, double* squared, long long* usable) {
    const T th = (T)thr;
    std::vector<T> gmax;
    for (int b = 0; b < B; ++b)
        for (int t = 0; t < Tn; ++t) {
            const int s = b * Tn + t, k0 = offsets[s], K = offsets[s + 1] - k0;
            if (K == 0) continue;
            gmax.assign(K, (T)0);
            for (int n = 0; n < N; ++n) {
                T best = 0;
                int arg = 0;
                for (int k = 0; k < K; ++k) {
                    const T v = IouOf<T>::at(anchors + (size_t)n * 4, boxes + (size_t)(k0 + k) * 4);
                    if (k == 0 || v > best) { best = v; arg = k; }
                    if (n == 0 || v > gmax[k]) gmax[k] = v;
                }
                if (!(best > th)) continue;
                const size_t cell = (size_t)t * n_bins + bin_of[n];
                const double* r = gt3 + (size_t)(k0 + arg) * 3;
                examine[cell] += 1;
                for (int c = 0; c < 3; ++c) {
                    sums[cell * 3 + c] = sums[cell * 3 + c] + r[c];
                    squared[cell * 3 + c] = squared[cell * 3 + c] + r[c] * r[c];
                }
            }
            for (int k = 0; k < K; ++k) usable[t] += gmax[k] > th;
        }
}

extern "C" int vd3d_anchor_prior_host(const float* anchors, const int* order, const int* bin_start, int N, int n_bins, const int* offsets,
                                      int B, int T, const void* boxes, int boxes_f64, const double* gt3, int K_total, double fg_iou_threshold,
                                      long long* examine, double* sums, double* squared, long long* usable) {
    VD3D_REQUIRE(anchors && order && bin_start && offsets && examine && sums && squared && usable, "anchor_prior_host: null argument");
    VD3D_REQUIRE(K_total == 0 || (boxes && gt3), "anchor_prior_host: null boxes");
    int rc = check_prior_args("anchor_prior_host", N, n_bins, bin_start, offsets, B, T, K_total);
    if (rc) return rc;
    // the bin order must list every anchor once, ascending within each bin: the walk order of the device entry
    std::vector<int> bin_of(N, -1);
    for (int bin = 0; bin < n_bins; ++bin)
        for (int i = bin_start[bin]; i < bin_start[bin + 1]; ++i) {
            const int n = order[i];
            VD3D_REQUIRE(n >= 0 && n < N && bin_of[n] < 0, "anchor_prior_host: order[%d] = %d is out of range or repeated", i, n);
            VD3D_REQUIRE(i == bin_start[bin] || order[i - 1] < n, "anchor_prior_host: bin %d's anchors are not ascending", bin);
            bin_of[n] = bin;
        }
    if (boxes_f64)
        prior_host<double>(anchors, bin_of.data(), N, n_bins, offsets, B, T, (const double*)boxes, gt3, fg_iou_threshold, examine, sums,
                           squared, usable);
    else
        prior_host<float>(anchors, bin_of.data(), N, n_bins, offsets, B, T, (const float*)boxes, gt3, fg_iou_threshold, examine, sums,
                          squared, usable);
    return VD3D_OK;
}
