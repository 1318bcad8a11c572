// The scope widget's per-tick step (Scope_Widget.handle_new_data, friture/scope.py:78-133) for many
// scopes, each call one trigger launch over all of its ticks and one launch that writes the curves.
#include "frt_internal.cuh"

namespace {

constexpr int SC_THREADS = 256;
constexpr int SC_WARPS = SC_THREADS / 32;
constexpr int SC_GROUP = 32;                                  // ticks whose window maxima are formed together
constexpr long long SC_NOT_DRAWN = LLONG_MIN;                 // a tick that drew nothing

struct ScopeArgs {
    const float *x;                 // row s * n_ch: the trigger channel of scope s
    long long stride, lead, origin, row_len;
    int n_ticks, buffer, width, trigger;
    int q, rem, cap;                // whole segments per search window, the samples after them, ring slots
    long long *start;               // [S][n_ticks]
};

// np.max: a NaN anywhere makes the maximum NaN (fmaxf would drop it).
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }

__device__ __forceinline__ float warp_nan_max(float m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = nan_max(m, __shfl_xor_sync(0xffffffffu, m, o));
    return m;
}

// One CTA per scope.  Tick r reads d = x[e - 2w, e), e = lead + (r+1)*buffer, and searches
// s = d[w/2, w/2 + w) (scope.py:96-103).  The search windows of consecutive ticks are `buffer` apart,
// so they lie on one grid of buffer-long segments starting at tick 0's search start c0: tick r's
// window is segments r .. r+q-1 and the first `rem` samples of segment r+q (q = w / buffer, rem =
// w % buffer).  Every segment's maximum M and the maximum P of its first rem samples are formed
// once, in a shared ring of cap >= q + SC_GROUP slots, and each tick's maximum from q + 1 of them.
// level = max * 2 / 3 in double (scope.py:105); the first i with s[i] < level <= s[i+1], compared in
// double, is found 256 pairs at a time with warp ballots, stopping at the first block that holds one.
__global__ void __launch_bounds__(SC_THREADS) scope_trigger_kernel(const ScopeArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    float *seg_max = (float *)smem, *seg_pre = seg_max + a.cap;
    __shared__ double s_level[SC_GROUP];
    __shared__ int s_hit[3];
    const int s = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    long long *start = a.start + (size_t)s * a.n_ticks;
    const int w = a.width, h = w / 2;
    if (!a.trigger) {                        // scrolling: the last w samples (scope.py:89-94)
        for (int r = tid; r < a.n_ticks; r += SC_THREADS)
            start[r] = a.origin + a.lead + (long long)(r + 1) * a.buffer - w;
        return;
    }
    const float *x = a.x + (size_t)s * a.stride;
    const long long c0 = a.lead + a.buffer - 2ll * w + h;
    const int seg_read = a.q > 0 ? a.buffer : a.rem;   // with q == 0 only the prefixes are read
    if (tid < 3) s_hit[tid] = INT_MAX;
    long long next_seg = 0;
    int it = 0;                              // crossing-search passes so far: s_hit[it % 3] is this pass's
    for (int r0 = 0; r0 < a.n_ticks; r0 += SC_GROUP) {
        const int nr = min(SC_GROUP, a.n_ticks - r0);
        // the segments this group needs that no earlier group formed
        const long long last_seg = (long long)r0 + nr - 1 + a.q;
        for (long long k = next_seg + warp; k <= last_seg; k += SC_WARPS) {
            const long long base = c0 + k * a.buffer;
            float m = -INFINITY, p = -INFINITY;
            for (int j = lane; j < seg_read; j += 32) {
                if (base + j >= a.row_len) break;    // past the row: only a last segment nobody reads whole
                const float v = __ldg(x + base + j);
                m = nan_max(m, v);
                if (j < a.rem) p = nan_max(p, v);
            }
            m = warp_nan_max(m);
            p = warp_nan_max(p);
            if (lane == 0) {
                seg_max[k % a.cap] = m;
                seg_pre[k % a.cap] = p;
            }
        }
        next_seg = last_seg + 1;
        __syncthreads();
        // one warp per tick: its window maximum, then level
        for (int t = warp; t < nr; t += SC_WARPS) {
            const long long r = r0 + t;
            float m = -INFINITY;
            for (int k = lane; k < a.q; k += 32) m = nan_max(m, seg_max[(r + k) % a.cap]);
            if (lane == 0 && a.rem) m = nan_max(m, seg_pre[(r + a.q) % a.cap]);
            m = warp_nan_max(m);
            if (lane == 0) s_level[t] = __ddiv_rn(__dmul_rn((double)m, 2.0), 3.0);
        }
        __syncthreads();
        for (int t = 0; t < nr; t++) {
            const double level = s_level[t];
            const long long cr = c0 + (long long)(r0 + t) * a.buffer;
            int hit = INT_MAX;
            if (level == level) {            // a NaN level compares false everywhere: no trigger
                for (int i0 = 0; i0 < w - 1; i0 += SC_THREADS, it++) {
                    const int i = i0 + tid;
                    bool cross = false;
                    if (i < w - 1) {
                        const double lo = __ldg(x + cr + i), hi = __ldg(x + cr + i + 1);
                        cross = lo < level && hi >= level;
                    }
                    const unsigned b = __ballot_sync(0xffffffffu, cross);
                    if (lane == 0 && b) atomicMin(&s_hit[it % 3], i0 + warp * 32 + __ffs(b) - 1);
                    __syncthreads();
                    // three slots: this pass's, the next pass's (reset two passes ago), and the last
                    // pass's, which every thread has read once it passed this barrier
                    hit = s_hit[it % 3];
                    if (tid == 0) s_hit[(it + 2) % 3] = INT_MAX;
                    if (hit != INT_MAX) {
                        it++;
                        break;
                    }
                }
            }
            // scope.py:111-112: the curve starts at shift - w/2 = i within d, d at cr - h
            if (tid == 0) start[r0 + t] = hit == INT_MAX ? SC_NOT_DRAWN : a.origin + cr - h + hit;
        }
        __syncthreads();
    }
}

// scope.py:127-133 for the last tick of the call that drew: scaled_y = 1 - (y + 1) / 2 in double,
// rounded once to float32, for each channel of the scope; drawn[s] = the time range it drew at.
__global__ void __launch_bounds__(SC_THREADS) scope_curve_kernel(const float *x, long long stride, int n_ch,
                                                                long long origin, const long long *start,
                                                                int n_ticks, int n_points, float *curve,
                                                                long long curve_stride, double timerange,
                                                                double *drawn) {
    __shared__ long long s_col;
    const int s = blockIdx.y, tid = threadIdx.x;
    if (tid < 32) {
        long long col = -1;
        for (int base = n_ticks - 1; base >= 0; base -= 32) {
            const int r = base - tid;
            const long long v = r >= 0 ? start[(size_t)s * n_ticks + r] : SC_NOT_DRAWN;
            const unsigned b = __ballot_sync(0xffffffffu, v != SC_NOT_DRAWN);
            if (b) {
                col = __shfl_sync(0xffffffffu, v, __ffs(b) - 1) - origin;   // the latest tick that drew
                break;
            }
        }
        if (tid == 0) s_col = col;
    }
    __syncthreads();
    const long long col = s_col;
    if (col < 0) return;                     // no tick drew: the scope keeps its curve (scope.py:108-109)
    if (blockIdx.x == 0 && tid == 0) drawn[s] = timerange;
    const int j = blockIdx.x * SC_THREADS + tid;
    if (j >= n_points) return;
    for (int k = 0; k < n_ch; k++) {
        const size_t row = (size_t)s * n_ch + k;
        const double y = __ldg(x + row * stride + col + j);
        curve[row * curve_stride + j] = __double2float_rn(__dsub_rn(1.0, __dmul_rn(__dadd_rn(y, 1.0), 0.5)));
    }
}

}   // namespace

extern "C" int frt_scope_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_scopes, int n_ch,
                                 int64_t lead, int n_ticks, int buffer, int width, int trigger, int64_t origin,
                                 int64_t *start_dev, float *curve_dev, int64_t curve_stride, double timerange,
                                 double *drawn_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_scopes >= 1 && n_scopes <= 65535, "n_scopes must be in 1..65535");
    FRT_CHECK_ARG(h, n_ch == 1 || n_ch == 2, "n_ch must be 1 or 2");
    FRT_CHECK_ARG(h, n_ticks >= 0 && buffer >= 1, "bad shape");
    FRT_CHECK_ARG(h, width >= 2 && width <= (1 << 29), "width must be in 2..2^29");
    const int64_t need = trigger ? 2 * (int64_t)width : width;
    FRT_CHECK_ARG(h, lead >= 0 && lead + buffer >= need, "lead must be >= 0 and >= need - buffer");
    if (n_ticks == 0) return FRT_OK;
    FRT_CHECK_ARG(h, x_dev && start_dev && curve_dev && drawn_dev, "NULL buffer");
    const int64_t row_len = lead + (int64_t)n_ticks * buffer;
    const int n_points = trigger ? 2 * (width / 2) : width;
    FRT_CHECK_ARG(h, (int64_t)n_scopes * n_ch == 1 || x_stride >= row_len,
                  "rows overlap: x_stride must be >= lead + n_ticks * buffer");
    FRT_CHECK_ARG(h, (int64_t)n_scopes * n_ch == 1 || curve_stride >= n_points,
                  "curve rows overlap: curve_stride must be >= the point count");
    ScopeArgs a{};
    a.x = x_dev;
    a.stride = x_stride * n_ch;
    a.lead = lead;
    a.origin = origin;
    a.row_len = row_len;
    a.n_ticks = n_ticks;
    a.buffer = buffer;
    a.width = width;
    a.trigger = trigger != 0;
    a.q = width / buffer;
    a.rem = width % buffer;
    a.cap = a.q + SC_GROUP;
    a.start = (long long *)start_dev;
    const size_t smem = a.trigger ? 2 * sizeof(float) * a.cap : 0;
    FRT_CHECK_ARG(h, !a.trigger || a.q <= 25000, "width / buffer must be <= 25000 in trigger mode");
    int rc = frt_launch(h, scope_trigger_kernel, n_scopes, SC_THREADS, smem, (cudaStream_t)stream, a);
    if (rc != FRT_OK) return rc;
    const dim3 grid((unsigned)((n_points + SC_THREADS - 1) / SC_THREADS), (unsigned)n_scopes);
    return frt_launch(h, scope_curve_kernel, grid, SC_THREADS, 0, (cudaStream_t)stream, x_dev, (long long)x_stride,
                      n_ch, (long long)origin, (const long long *)start_dev, n_ticks, n_points, curve_dev,
                      (long long)curve_stride, timerange, drawn_dev);
}
