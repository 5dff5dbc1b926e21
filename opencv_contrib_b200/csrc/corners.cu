// corners.cu -- cudaimgproc's corner detectors (cv::cuda::createHarrisCorner, createMinEigenValCorner,
// createGoodFeaturesToTrackDetector; modules/cudaimgproc/src/corners.cpp, gftt.cpp, cuda/corners.cu, cuda/gftt.cu).
//
// Response: one fused kernel per (criterion, depth, aperture).  A CTA stages its 32 x 16 output tile plus the block-sum
// and derivative halos of the source in shared memory (first border, on source coordinates), runs the separable Sobel /
// Scharr row pass and column pass there, fills the derivative cells outside the image from the mapped in-image cells
// (second border: the reference's block sum reads Dx / Dy through the border rule), sums the structure tensor and writes
// the response.  No Dx / Dy / row-buffer planes reach HBM.  The detector's launch also folds the image's maximum response
// into an order-preserving int with atomicMax.
//
// Detect: candidates (3x3 local maxima above max * qualityLevel) are appended as unique 64-bit keys (response bits,
// raster index), then one cooperative kernel sorts them (bitonic, descending: response, then raster index), applies the
// capacity cut and, with minDistance >= 1, runs the reference's sequential grid rule as parallel rounds of greedy
// selection, and compacts the accepted corners in priority order.  Nothing returns to the host.
//
// Built with -fmad=false: every operation rounds once, as oracle/corners_model.py restates it.
#include "common.cuh"

#include <algorithm>
#include <climits>
#include <cmath>

namespace b2f {
namespace {

constexpr int CT_W = 32, CT_H = 16, C_THREADS = 256;  // response tile and CTA (32 x 8 threads, two rows each)
constexpr int C_MAX_BLOCK = 31;                        // the block-sum halo must stay inside one tile (see k_corner_response)
constexpr int S_THREADS = 512, S_CHUNK = 1024;         // selection kernel: CTA size, bitonic shared-memory chunk
constexpr int BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_REFLECT101 = 4;

// cudev's border rules (cudev/ptr2d/extrapolation.hpp): idx_low(idx_high(i)), valid for any i and any len >= 1.  The
// reference's Sobel / Scharr filters and its block sums use the same rules.
__host__ __device__ __forceinline__ int border_index(int i, int len, int border) {
    const int last = len - 1;
    if (border == BORDER_REPLICATE) return max(min(i, last), 0);
    if (border == BORDER_REFLECT) {
        const int hi = last - abs(last - i) + (i > last);
        return (abs(hi) - (hi < 0)) % len;
    }
    const int hi = abs(last - abs(last - i)) % len;
    return abs(hi) % len;
}

struct DerivTaps {
    float dx_row[7], dx_col[7];  // d/dx: derivative along x, smoothing (scaled) along y
    float dy_row[7], dy_col[7];  // d/dy: smoothing (scaled) along x, derivative along y
};

__device__ __forceinline__ int max_key(float f) {  // signed-int order equals float order (finite values)
    const int b = __float_as_int(f);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float key_value(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }
__device__ __forceinline__ unsigned sort_bits(float f) {  // unsigned order equals float order
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

size_t response_smem(int bs, int ld) {
    const int R = ld / 2, RW = CT_W + bs - 1, RH = CT_H + bs - 1, SW = RW + 2 * R, SH = RH + 2 * R;
    return sizeof(float) * ((size_t)SH * SW + 2 * (size_t)SH * RW + 2 * (size_t)RH * RW);
}

// LD / LS: derivative / smoothing kernel lengths (ksize 1: 3 / 1; Scharr: 3 / 3; ksize 3, 5, 7: ksize / ksize)
template <bool HARRIS, typename T, int LD, int LS>
__global__ void __launch_bounds__(C_THREADS)
    k_corner_response(const T *__restrict__ src, size_t step, int rows, int cols, int border, int bs, DerivTaps taps,
                      float k, float *__restrict__ dst, size_t dstep, int *__restrict__ max_out) {
    extern __shared__ float sm[];
    constexpr int R = LD / 2;
    const int h0 = bs / 2, RW = CT_W + bs - 1, RH = CT_H + bs - 1, SW = RW + 2 * R, SH = RH + 2 * R;
    float *s_src = sm, *s_rx = s_src + SH * SW, *s_ry = s_rx + SH * RW, *s_dx = s_ry + SH * RW, *s_dy = s_dx + RH * RW;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const int x0 = blockIdx.x * CT_W, y0 = blockIdx.y * CT_H;
    const int vy0 = y0 - h0, vx0 = x0 - h0;  // image coordinates of region cell (0, 0)

    // first border: the source, on source coordinates
    for (int i = tid; i < SH * SW; i += C_THREADS) {
        const int r = i / SW, c = i - r * SW;
        const int sy = border_index(vy0 - R + r, rows, border), sx = border_index(vx0 - R + c, cols, border);
        const T *row = reinterpret_cast<const T *>(reinterpret_cast<const char *>(src) + (size_t)sy * step);
        s_src[i] = static_cast<float>(row[sx]);
    }
    __syncthreads();
    // row pass (the reference's row filter: sum = sum + src * kernel[k], k = 0 .. len - 1, anchor len / 2)
    for (int i = tid; i < SH * RW; i += C_THREADS) {
        const int r = i / RW, c = i - r * RW;
        const float *p = s_src + r * SW + c + R;
        float sx = 0.f, sy = 0.f;
#pragma unroll
        for (int t = 0; t < LD; ++t) sx = sx + p[t - LD / 2] * taps.dx_row[t];
#pragma unroll
        for (int t = 0; t < LS; ++t) sy = sy + p[t - LS / 2] * taps.dy_row[t];
        s_rx[i] = sx;
        s_ry[i] = sy;
    }
    __syncthreads();
    // column pass, for the region cells inside the image
    for (int i = tid; i < RH * RW; i += C_THREADS) {
        const int r = i / RW, c = i - r * RW;
        const int vy = vy0 + r, vx = vx0 + c;
        if (vy < 0 || vy >= rows || vx < 0 || vx >= cols) continue;
        float dx = 0.f, dy = 0.f;
#pragma unroll
        for (int t = 0; t < LS; ++t) dx = dx + s_rx[(r + R + t - LS / 2) * RW + c] * taps.dx_col[t];
#pragma unroll
        for (int t = 0; t < LD; ++t) dy = dy + s_ry[(r + R + t - LD / 2) * RW + c] * taps.dy_col[t];
        s_dx[i] = dx;
        s_dy[i] = dy;
    }
    __syncthreads();
    // second border: a cell outside the image that a block sum reads (at most bs - 1 - bs / 2 past the last row or
    // column) takes the derivatives of its mapped cell, which lies inside the region because that reach and the halo
    // (at most C_MAX_BLOCK / 2) are shorter than the tile in both directions
    const int reach_end = bs - 1 - h0;
    for (int i = tid; i < RH * RW; i += C_THREADS) {
        const int r = i / RW, c = i - r * RW;
        const int vy = vy0 + r, vx = vx0 + c;
        if (vy >= 0 && vy < rows && vx >= 0 && vx < cols) continue;
        if (vy > rows - 1 + reach_end || vx > cols - 1 + reach_end) continue;  // past every output pixel's block
        const int j = (border_index(vy, rows, border) - vy0) * RW + (border_index(vx, cols, border) - vx0);
        s_dx[i] = s_dx[j];
        s_dy[i] = s_dy[j];
    }
    __syncthreads();

    int best = INT_MIN;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int ty = threadIdx.y + half * 8, y = y0 + ty, x = x0 + threadIdx.x;
        if (y >= rows || x >= cols) continue;
        float a = 0.f, b = 0.f, c = 0.f;
        for (int i = 0; i < bs; ++i) {
            const float *px = s_dx + (ty + i) * RW + threadIdx.x, *py = s_dy + (ty + i) * RW + threadIdx.x;
            for (int j = 0; j < bs; ++j) {
                const float dx = px[j], dy = py[j];
                a = a + dx * dx;
                b = b + dx * dy;
                c = c + dy * dy;
            }
        }
        float v;
        if (HARRIS) {
            v = a * c - b * b - k * (a + c) * (a + c);
        } else {
            a = a * 0.5f;
            c = c * 0.5f;
            v = (a + c) - sqrtf((a - c) * (a - c) + b * b);
        }
        dst[(size_t)y * dstep + x] = v;
        best = max(best, max_key(v));
    }
    if (max_out) {  // the image's maximum response (cuda::minMax over the whole image, gftt.cpp:120)
        __shared__ int s_best[C_THREADS / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
        if ((tid & 31) == 0) s_best[tid >> 5] = best;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < C_THREADS / 32; ++w) best = max(best, s_best[w]);
            if (best != INT_MIN) atomicMax(max_out, best);
        }
    }
}

// Device state of one detect, zeroed (max: INT_MIN) by k_gftt_reset in front of the response launch.
struct GfttState {
    int max_key;
    int count;          // candidates found
    unsigned barrier;   // arrivals at the selection kernel's grid barrier
    int undecided[3];   // per-round undecided counts, rotating
    int info[4];        // b2f_gftt_info: candidates, kept, capped, rounds
};

__global__ void k_gftt_reset(GfttState *st) {
    st->max_key = INT_MIN;
    st->count = 0;
    st->barrier = 0;
    st->undecided[0] = st->undecided[1] = st->undecided[2] = 0;
}

// findCorners (gftt.cu:55-88): inside the 1-pixel frame, under the mask, above the threshold, equal to its 3x3 maximum.
__global__ void __launch_bounds__(256)
    k_gftt_candidates(const float *__restrict__ eig, size_t estep, int rows, int cols, const unsigned char *__restrict__ mask,
                      size_t mstep, double quality, GfttState *st, unsigned long long *__restrict__ keys) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    bool cand = false;
    float val = 0.f;
    if (y > 0 && y < rows - 1 && x > 0 && x < cols - 1 && (!mask || mask[(size_t)y * mstep + x])) {
        const float threshold = static_cast<float>(static_cast<double>(key_value(st->max_key)) * quality);
        const float *r0 = eig + (size_t)(y - 1) * estep + x, *r1 = r0 + estep, *r2 = r1 + estep;
        val = r1[0];
        if (val > threshold) {
            float m = val;
            m = fmaxf(r0[-1], m); m = fmaxf(r0[0], m); m = fmaxf(r0[1], m);
            m = fmaxf(r1[-1], m); m = fmaxf(r1[1], m);
            m = fmaxf(r2[-1], m); m = fmaxf(r2[0], m); m = fmaxf(r2[1], m);
            cand = val == m;
        }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, cand);
    if (!ballot) return;
    const int lane = threadIdx.x, leader = __ffs(ballot) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(&st->count, __popc(ballot));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (cand)
        keys[base + __popc(ballot & ((1u << lane) - 1))] =
            (static_cast<unsigned long long>(sort_bits(val)) << 32) | static_cast<unsigned>(y * cols + x);
}

__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned &epoch) {
    __syncthreads();
    ++epoch;
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        const unsigned target = epoch * gridDim.x;
        unsigned seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
    }
    __syncthreads();
}

__device__ __forceinline__ void cmp_swap(unsigned long long &a, unsigned long long &b, bool desc) {
    if (desc ? a < b : a > b) {
        const unsigned long long t = a;
        a = b;
        b = t;
    }
}

// bitonic steps (k, j_first .. 1) of every S_CHUNK-element chunk, in shared memory
__device__ void bitonic_chunks(unsigned long long *keys, int n2, int k_first, int k_last, int j_first,
                               unsigned long long *s) {
    for (int base = blockIdx.x * S_CHUNK; base < n2; base += gridDim.x * S_CHUNK) {
        for (int i = threadIdx.x; i < S_CHUNK; i += S_THREADS) s[i] = __ldcg(keys + base + i);
        for (int k = k_first; k <= k_last; k <<= 1) {
            for (int j = k == k_first ? j_first : k >> 1; j > 0; j >>= 1) {
                __syncthreads();
                const int t = threadIdx.x, i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                cmp_swap(s[i], s[i + j], ((base + i) & k) == 0);
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < S_CHUNK; i += S_THREADS) keys[base + i] = s[i];
        __syncthreads();
    }
}

// One candidate's decision in round `round` of the greedy rule: rejected (2) when a higher-priority conflicting candidate
// was accepted in an earlier round, accepted (1) when every one of them was rejected in an earlier round, else
// undecided (0).  Only earlier rounds count, so the number of rounds is a property of the candidates, not of timing.
// state: 0 undecided, else 2 (decision round + 1) + 1 if accepted.  Conflict: the reference's test, gftt.cpp:159-191
// -- the other corner lies in the 3x3 cells around this one's cell and float(dx*dx + dy*dy) < minDistance^2.
__device__ int decide(int i, int round, const unsigned long long *keys, const int *owner, volatile int *state, int rows,
                      int cols, int cell, int gw, int gh, int reach, double md2) {
    const unsigned p = static_cast<unsigned>(__ldcg(keys + i));
    const int px = p % cols, py = p / cols;
    const int xc = static_cast<int>(__fdiv_rn(static_cast<float>(px), static_cast<float>(cell)));
    const int yc = static_cast<int>(__fdiv_rn(static_cast<float>(py), static_cast<float>(cell)));
    const int cx1 = max(0, xc - 1), cy1 = max(0, yc - 1), cx2 = min(gw - 1, xc + 1), cy2 = min(gh - 1, yc + 1);
    const int qx1 = max((int)min((long long)cx1 * cell, (long long)cols), px - reach);
    const int qx2 = min((int)min((long long)(cx2 + 1) * cell, (long long)cols) - 1, px + reach);
    const int qy1 = max((int)min((long long)cy1 * cell, (long long)rows), py - reach);
    const int qy2 = min((int)min((long long)(cy2 + 1) * cell, (long long)rows) - 1, py + reach);
    bool pending = false;
    for (int qy = qy1; qy <= qy2; ++qy) {
        const int *orow = owner + (size_t)qy * cols;
        const float dy = static_cast<float>(py) - static_cast<float>(qy);
        for (int qx = qx1; qx <= qx2; ++qx) {
            const int j = __ldcg(orow + qx);
            if (j < 0 || j >= i) continue;
            const float dx = static_cast<float>(px) - static_cast<float>(qx);
            if (!(static_cast<double>(dx * dx + dy * dy) < md2)) continue;
            const int s = state[j];
            const bool known = s != 0 && (s >> 1) <= round;
            if (known && (s & 1)) return 2;
            if (!known) pending = true;
        }
    }
    return pending ? 0 : 1;
}

__device__ __forceinline__ int block_sum(int v, int *s_tmp) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_tmp[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
    for (int w = 0; w < S_THREADS / 32; ++w) t += s_tmp[w];
    return t;
}

struct SelectArgs {
    unsigned long long *keys;
    int *owner;  // rows x cols, priority of the candidate at each pixel or -1
    int *state;  // per kept candidate: 0 undecided, else 2 (decision round + 1) + 1 if accepted
    int *block_counts;
    GfttState *st;
    float2 *corners;
    int *count_out;
    int rows, cols, keep_cap, max_corners, out_cap;
    int cell, gw, gh, reach;
    double md, md2;
};

__global__ void __launch_bounds__(S_THREADS) k_gftt_select(SelectArgs A) {
    __shared__ unsigned long long s_keys[S_CHUNK];
    __shared__ int s_tmp[S_THREADS / 32 + 1];
    const int gtid = blockIdx.x * S_THREADS + threadIdx.x, gsz = gridDim.x * S_THREADS;
    unsigned epoch = 0;
    GfttState *st = A.st;
    const int n = *(volatile int *)&st->count;
    int n2 = S_CHUNK;
    while (n2 < n) n2 <<= 1;
    const bool grid_rule = A.md >= 1.0;
    for (int i = n + gtid; i < n2; i += gsz) A.keys[i] = 0ull;  // padding sorts last
    if (grid_rule)
        for (size_t i = gtid; i < (size_t)A.rows * A.cols; i += gsz) A.owner[i] = -1;
    grid_barrier(&st->barrier, epoch);

    // bitonic sort, descending: response, then raster index (the keys are unique)
    bitonic_chunks(A.keys, n2, 2, S_CHUNK, 1, s_keys);
    grid_barrier(&st->barrier, epoch);
    for (int k = 2 * S_CHUNK; k <= n2; k <<= 1) {
        for (int j = k >> 1; j >= S_CHUNK; j >>= 1) {
            for (int t = gtid; t < n2 / 2; t += gsz) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                unsigned long long a = __ldcg(A.keys + i), b = __ldcg(A.keys + i + j);
                const bool desc = (i & k) == 0;
                if (desc ? a < b : a > b) {
                    A.keys[i] = b;
                    A.keys[i + j] = a;
                }
            }
            grid_barrier(&st->barrier, epoch);
        }
        bitonic_chunks(A.keys, n2, k, k, S_CHUNK / 2, s_keys);
        grid_barrier(&st->barrier, epoch);
    }

    const int total = min(n, A.keep_cap);  // the capacity cut: the first keep_cap candidates in this order
    const int limit = A.max_corners > 0 ? min(A.max_corners, A.out_cap) : A.out_cap;
    int rounds = 0;
    if (!grid_rule) {
        const int m = min(total, limit);
        for (int i = gtid; i < m; i += gsz) {
            const unsigned p = static_cast<unsigned>(__ldcg(A.keys + i));
            A.corners[i] = make_float2(static_cast<float>(p % A.cols), static_cast<float>(p / A.cols));
        }
        if (gtid == 0) *A.count_out = m;
    } else {
        for (int i = gtid; i < total; i += gsz) {
            A.owner[static_cast<unsigned>(__ldcg(A.keys + i))] = i;
            A.state[i] = 0;
        }
        grid_barrier(&st->barrier, epoch);
        volatile int *state = A.state;
        for (;; ++rounds) {
            if (gtid == 0) st->undecided[(rounds + 1) % 3] = 0;  // last read before the previous barrier
            int und = 0;
            for (int i = gtid; i < total; i += gsz) {
                if (state[i] != 0) continue;
                const int d = decide(i, rounds, A.keys, A.owner, state, A.rows, A.cols, A.cell, A.gw, A.gh, A.reach, A.md2);
                if (d) state[i] = 2 * (rounds + 1) + (d == 1);
                else ++und;
            }
            und = block_sum(und, s_tmp);
            if (threadIdx.x == 0 && und) atomicAdd(&st->undecided[rounds % 3], und);
            grid_barrier(&st->barrier, epoch);
            if (*(volatile int *)&st->undecided[rounds % 3] == 0) break;
        }
        ++rounds;
        // compaction in priority order: contiguous ranges per CTA, offsets from the preceding CTAs' counts
        const int per = (total + gridDim.x - 1) / gridDim.x;
        const int lo = min(total, blockIdx.x * per), hi = min(total, lo + per);
        int mine = 0;
        for (int i = lo + threadIdx.x; i < hi; i += S_THREADS) mine += state[i] & 1;
        mine = block_sum(mine, s_tmp);
        if (threadIdx.x == 0) A.block_counts[blockIdx.x] = mine;
        grid_barrier(&st->barrier, epoch);
        int offset = 0, all = 0;
        for (int b = 0; b < (int)gridDim.x; ++b) {
            const int v = *(volatile int *)&A.block_counts[b];
            if (b < (int)blockIdx.x) offset += v;
            all += v;
        }
        for (int t0 = lo; t0 < hi; t0 += S_THREADS) {
            const int i = t0 + threadIdx.x;
            const bool acc = i < hi && (state[i] & 1);
            const unsigned ball = __ballot_sync(0xffffffffu, acc);
            __syncthreads();
            if ((threadIdx.x & 31) == 0) s_tmp[threadIdx.x >> 5] = __popc(ball);
            __syncthreads();
            int before = 0, tile = 0;
            for (int w = 0; w < S_THREADS / 32; ++w) {
                if (w < (int)(threadIdx.x >> 5)) before += s_tmp[w];
                tile += s_tmp[w];
            }
            const int rank = offset + before + __popc(ball & ((1u << (threadIdx.x & 31)) - 1));
            if (acc && rank < limit) {
                const unsigned p = static_cast<unsigned>(__ldcg(A.keys + i));
                A.corners[rank] = make_float2(static_cast<float>(p % A.cols), static_cast<float>(p / A.cols));
            }
            offset += tile;
        }
        if (gtid == 0) *A.count_out = min(all, limit);
    }
    if (gtid == 0) {
        st->info[0] = n;
        st->info[1] = total;
        st->info[2] = n > A.keep_cap;
        st->info[3] = rounds;
    }
}

// -------------------------------------------------------------------------------------------- dispatch
using ResponseKernel = void (*)(const void *, size_t, int, int, int, int, DerivTaps, float, float *, size_t, int *);

template <bool H, typename T, int LD, int LS>
ResponseKernel response_kernel() {
    return reinterpret_cast<ResponseKernel>(&k_corner_response<H, T, LD, LS>);
}

template <bool H, typename T>
ResponseKernel pick_aperture(int ksize) {
    switch (ksize) {
        case 1: return response_kernel<H, T, 3, 1>();
        case 5: return response_kernel<H, T, 5, 5>();
        case 7: return response_kernel<H, T, 7, 7>();
        default: return response_kernel<H, T, 3, 3>();  // 3 and Scharr
    }
}

ResponseKernel pick_response(bool harris, int type, int ksize) {
    if (harris) return type == B2F_8UC1 ? pick_aperture<true, unsigned char>(ksize) : pick_aperture<true, float>(ksize);
    return type == B2F_8UC1 ? pick_aperture<false, unsigned char>(ksize) : pick_aperture<false, float>(ksize);
}

// Every instantiation may need up to response_smem(C_MAX_BLOCK, 7) bytes of dynamic shared memory.
void set_response_smem(Ctx &c) {
    static DeviceOnce once;
    once.run(c, [&] {
        const int bytes = static_cast<int>(response_smem(C_MAX_BLOCK, 7));
        for (int h = 0; h < 2; ++h)
            for (int t = 0; t < 2; ++t)
                for (int ks : {1, 3, 5, 7})
                    c.check(cudaFuncSetAttribute(reinterpret_cast<const void *>(pick_response(h, t ? B2F_32FC1 : B2F_8UC1, ks)),
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    });
}

// getDerivKernels(kx, ky, dx, dy, ksize, false, CV_32F) (Sobel: getSobelKernels; ksize <= 0: Scharr)
void deriv_kernel(int order, int ksize, std::vector<int> &k) {
    if (ksize <= 0) {
        k = order ? std::vector<int>{-1, 0, 1} : std::vector<int>{3, 10, 3};
        return;
    }
    if (ksize == 1 && order > 0) ksize = 3;
    if (ksize == 1) {
        k = {1};
        return;
    }
    if (ksize == 3) {
        k = order ? std::vector<int>{-1, 0, 1} : std::vector<int>{1, 2, 1};
        return;
    }
    std::vector<int> v(ksize + 1, 0);
    v[0] = 1;
    for (int i = 0; i < ksize - order - 1; ++i) {
        int oldval = v[0];
        for (int j = 1; j <= ksize; ++j) {
            const int newval = v[j] + v[j - 1];
            v[j - 1] = oldval;
            oldval = newval;
        }
    }
    for (int i = 0; i < order; ++i) {
        int oldval = -v[0];
        for (int j = 1; j <= ksize; ++j) {
            const int newval = v[j - 1] - v[j];
            v[j - 1] = oldval;
            oldval = newval;
        }
    }
    v.resize(ksize);
    k = v;
}

}  // namespace
}  // namespace b2f

// ================================================================================================ the handle
struct b2f_corners : b2f_handle {
    bool detector = false;
    int src_type = 0, block_size = 3, ksize = 3, border = b2f::BORDER_REFLECT101;
    bool harris = false;
    float k = 0.f;
    b2f_gftt_params G{};
    b2f::DerivTaps taps{};

    // detect workspace (arena), laid out for (rows, cols)
    int rows = 0, cols = 0, blocks = 0;
    b2f::Plane eig{};
    unsigned long long *keys = nullptr;
    int *owner = nullptr, *state = nullptr, *block_counts = nullptr;
    b2f::GfttState *st = nullptr;

    struct Key {
        const void *base = nullptr, *img = nullptr, *mask = nullptr, *corners = nullptr, *count = nullptr;
        size_t step = 0, mstep = 0;
        int rows = 0, cols = 0, type = 0, capacity = 0, max_corners = 0, block_size = 0, harris = 0;
        double quality = 0, md = 0, k = 0;
        bool operator==(const Key &o) const {
            return base == o.base && img == o.img && mask == o.mask && corners == o.corners && count == o.count &&
                   step == o.step && mstep == o.mstep && rows == o.rows && cols == o.cols && type == o.type &&
                   capacity == o.capacity && max_corners == o.max_corners && block_size == o.block_size &&
                   harris == o.harris && quality == o.quality && md == o.md && k == o.k;
        }
    };
    b2f::GraphCache<Key> graph;

    int calc(const b2f_image *, const b2f_image *, b2f_image *, cudaStream_t) override { return B2F_BAD_ARG; }
    int set_param(int, double) override { return B2F_BAD_ARG; }
    int get_param(int, double *) const override { return B2F_BAD_ARG; }
    const char *default_name() const override { return detector ? "CornersDetector.GFTT" : "CornernessCriteria"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"corner_response", "gftt_candidates", "gftt_select", "gftt_reset"};
        return cls >= 0 && cls < 4 ? n[cls] : "";
    }
    size_t workspace_bytes(int, int, int) override { return arena.capacity(); }

    // CornerBase's constructor (corners.cpp:83-113): scale and the derivative kernels
    int setup(int type, int bs, int ks, double kk, int brd, bool is_harris) {
        if (type != B2F_8UC1 && type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
        if (brd != b2f::BORDER_REFLECT101 && brd != b2f::BORDER_REPLICATE && brd != b2f::BORDER_REFLECT) return B2F_BAD_ARG;
        if (!(ks <= 0 || ks == 1 || ks == 3 || ks == 5 || ks == 7)) return B2F_BAD_ARG;
        if (bs < 1 || bs > b2f::C_MAX_BLOCK) return B2F_BAD_ARG;
        src_type = type;
        block_size = bs;
        ksize = ks;
        border = brd;
        harris = is_harris;
        k = static_cast<float>(kk);
        double scale = static_cast<double>(1 << ((ks > 0 ? ks : 3) - 1)) * bs;
        if (ks < 0) scale *= 2.;
        if (type == B2F_8UC1) scale *= 255.;
        scale = 1. / scale;
        std::vector<int> d, s;
        b2f::deriv_kernel(1, ks, d);
        b2f::deriv_kernel(0, ks, s);
        const float fs = static_cast<float>(scale);
        for (size_t i = 0; i < d.size(); ++i) taps.dx_row[i] = taps.dy_col[i] = static_cast<float>(d[i]);
        for (size_t i = 0; i < s.size(); ++i) taps.dx_col[i] = taps.dy_row[i] = static_cast<float>(s[i]) * fs;
        return B2F_OK;
    }

    static int image_ok(const b2f_image *im, int type) {
        if (!im || !im->data || im->rows < 1 || im->cols < 1) return B2F_BAD_ARG;
        if (im->type != type) return B2F_UNSUPPORTED_TYPE;
        const size_t es = type == B2F_8UC1 ? 1 : 4;
        if (im->step < (size_t)im->cols * es || im->step % es || reinterpret_cast<uintptr_t>(im->data) % es) return B2F_BAD_ARG;
        return B2F_OK;
    }

    void launch_response(b2f::Ctx &c, const b2f_image *src, float *dst, size_t dstep, int *max_out) {
        using namespace b2f;
        set_response_smem(c);
        const int ld = ksize == 5 ? 5 : ksize == 7 ? 7 : 3;
        const size_t smem = response_smem(block_size, ld);
        const dim3 grid(div_up(src->cols, CT_W), div_up(src->rows, CT_H)), block(32, 8);
        const double bytes = (double)src->rows * src->cols * ((src->type == B2F_8UC1 ? 1 : 4) + 4);
        B2F_LAUNCH(c, 0, bytes, pick_response(harris, src->type, ksize), grid, block, smem, src->data, src->step,
                   src->rows, src->cols, border, block_size, taps, k, dst, dstep, max_out);
    }

    int keep_cap(int r, int cc) const { return std::max(1000, static_cast<int>(static_cast<double>(r) * cc * 0.05)); }
    int capacity(int r, int cc) const { return G.max_corners > 0 ? std::min(G.max_corners, keep_cap(r, cc)) : keep_cap(r, cc); }

    int layout(b2f::Ctx &c, int r, int cc) {
        using namespace b2f;
        if (r == rows && cc == cols && arena.capacity() > 0) return B2F_OK;
        if (arena.capacity() > 0) c.check(cudaStreamSynchronize(c.stream));  // re-layout of a live arena
        int occ = 0;
        c.check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_gftt_select, S_THREADS, 0));
        if (!c.ok()) return B2F_CUDA_ERROR;
        if (occ < 1) return B2F_CUDA_ERROR;
        blocks = sm_count();
        size_t n2 = S_CHUNK;
        while (n2 < (size_t)r * cc) n2 <<= 1;
        for (int pass = 0; pass < 2 && c.ok(); ++pass) {
            Arena tmp;
            Arena &A = pass == 0 ? tmp : arena;
            A.begin(pass == 0);
            eig = A.plane(r, cc);
            keys = static_cast<unsigned long long *>(A.bytes(n2 * sizeof(unsigned long long)));
            owner = static_cast<int *>(A.bytes((size_t)r * cc * sizeof(int)));
            state = static_cast<int *>(A.bytes((size_t)keep_cap(r, cc) * sizeof(int)));
            block_counts = static_cast<int *>(A.bytes((size_t)blocks * sizeof(int)));
            st = static_cast<GfttState *>(A.bytes(sizeof(GfttState)));
            if (pass == 0) c.check(arena.reserve(A.used()));
        }
        if (!c.ok()) return B2F_CUDA_ERROR;
        rows = r;
        cols = cc;
        graph.destroy();
        return B2F_OK;
    }

    void schedule(b2f::Ctx &c, const b2f_image *img, const b2f_image *mask, float *corners, int cap, int *count_dev) {
        using namespace b2f;
        B2F_LAUNCH(c, 3, 0.0, k_gftt_reset, dim3(1), dim3(1), 0, st);
        launch_response(c, img, eig.p, eig.pitch, &st->max_key);
        B2F_LAUNCH(c, 1, 4.0 * rows * cols * (mask ? 1.25 : 1.0), k_gftt_candidates, dim3(div_up(cols, 32), div_up(rows, 8)),
                   dim3(32, 8), 0, eig.p, (size_t)eig.pitch, rows, cols, mask ? static_cast<const unsigned char *>(mask->data) : nullptr,
                   mask ? mask->step : 0, G.quality_level, st, keys);
        SelectArgs A{};
        A.keys = keys;
        A.owner = owner;
        A.state = state;
        A.block_counts = block_counts;
        A.st = st;
        A.corners = reinterpret_cast<float2 *>(corners);
        A.count_out = count_dev;
        A.rows = rows;
        A.cols = cols;
        A.keep_cap = keep_cap(rows, cols);
        A.max_corners = G.max_corners;
        A.out_cap = cap;
        A.md = G.min_distance;
        A.md2 = G.min_distance * G.min_distance;
        A.cell = G.min_distance >= 1.0 ? cv_round(G.min_distance) : 1;
        A.gw = (cols + A.cell - 1) / A.cell;
        A.gh = (rows + A.cell - 1) / A.cell;
        A.reach = static_cast<int>(std::min(std::floor(G.min_distance), 65536.0));
        if (c.ok()) {
            c.pre(2, 0.0);
            void *args[] = {&A};
            c.check(cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(k_gftt_select), dim3(blocks), dim3(S_THREADS),
                                                args, 0, c.stream));
            c.post(2);
        }
    }
};

namespace {
bool gftt_params_ok(const b2f_gftt_params &p) {
    return p.quality_level > 0 && p.min_distance >= 0 && p.max_corners >= 0;  // gftt.cpp:94
}
}  // namespace

extern "C" {

int b2f_harris_create(int src_type, int block_size, int ksize, double k, int border_type, b2f_corners **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    auto *h = new (std::nothrow) b2f_corners();
    if (!h) return B2F_OUT_OF_MEMORY;
    const int st = h->setup(src_type, block_size, ksize, k, border_type, true);
    if (st != B2F_OK) {
        delete h;
        return st;
    }
    *out = h;
    return B2F_OK;
}

int b2f_mineig_create(int src_type, int block_size, int ksize, int border_type, b2f_corners **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    auto *h = new (std::nothrow) b2f_corners();
    if (!h) return B2F_OUT_OF_MEMORY;
    const int st = h->setup(src_type, block_size, ksize, 0.0, border_type, false);
    if (st != B2F_OK) {
        delete h;
        return st;
    }
    *out = h;
    return B2F_OK;
}

int b2f_corners_compute(b2f_corners *h, const b2f_image *src, b2f_image *dst, void *cuda_stream) {
    using namespace b2f;
    if (!h || !src || !dst) return B2F_BAD_ARG;
    int st = b2f_corners::image_ok(src, h->src_type);
    if (st != B2F_OK) return st;
    st = b2f_corners::image_ok(dst, B2F_32FC1);
    if (st != B2F_OK) return st;
    if (dst->rows != src->rows || dst->cols != src->cols) return B2F_SIZE_MISMATCH;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(src->data, s);
    if (!h->bind_device()) return B2F_BAD_ARG;
    Ctx c = h->make_ctx(s);
    h->stats.calls++;
    h->launch_response(c, src, static_cast<float *>(dst->data), dst->step / 4, nullptr);
    return h->finish(c, s);
}

void b2f_gftt_default_params(b2f_gftt_params *p) {
    if (!p) return;
    p->max_corners = 1000;
    p->quality_level = 0.01;
    p->min_distance = 0.0;
    p->block_size = 3;
    p->use_harris = 0;
    p->harris_k = 0.04;
}

int b2f_gftt_create(int src_type, const b2f_gftt_params *p, b2f_corners **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    b2f_gftt_params P;
    b2f_gftt_default_params(&P);
    if (p) P = *p;
    if (!gftt_params_ok(P)) return B2F_BAD_ARG;
    auto *h = new (std::nothrow) b2f_corners();
    if (!h) return B2F_OUT_OF_MEMORY;
    const int st = h->setup(src_type, P.block_size, 3, P.harris_k, b2f::BORDER_REFLECT101, P.use_harris != 0);
    if (st != B2F_OK) {
        delete h;
        return st;
    }
    h->detector = true;
    h->G = P;
    *out = h;
    return B2F_OK;
}

int b2f_gftt_set_params(b2f_corners *h, const b2f_gftt_params *p) {
    if (!h || !p || !h->detector || !gftt_params_ok(*p)) return B2F_BAD_ARG;
    b2f_corners tmp;
    const int st = tmp.setup(h->src_type, p->block_size, 3, p->harris_k, b2f::BORDER_REFLECT101, p->use_harris != 0);
    if (st != B2F_OK) return st;
    h->setup(h->src_type, p->block_size, 3, p->harris_k, b2f::BORDER_REFLECT101, p->use_harris != 0);
    h->G = *p;
    return B2F_OK;
}

int b2f_gftt_get_params(const b2f_corners *h, b2f_gftt_params *p) {
    if (!h || !p || !h->detector) return B2F_BAD_ARG;
    *p = h->G;
    return B2F_OK;
}

int b2f_gftt_capacity(const b2f_corners *h, int rows, int cols, int *capacity) {
    if (!h || !capacity || !h->detector || rows < 1 || cols < 1) return B2F_BAD_ARG;
    *capacity = h->capacity(rows, cols);
    return B2F_OK;
}

int b2f_gftt_detect(b2f_corners *h, const b2f_image *image, const b2f_image *mask, float *corners, int capacity,
                    int *count, void *cuda_stream) {
    using namespace b2f;
    if (!h || !h->detector || !corners || !count) return B2F_BAD_ARG;
    int st = b2f_corners::image_ok(image, h->src_type);
    if (st != B2F_OK) return st;
    if (mask) {  // gftt.cpp:114
        st = b2f_corners::image_ok(mask, B2F_8UC1);
        if (st != B2F_OK) return st;
        if (mask->rows != image->rows || mask->cols != image->cols) return B2F_SIZE_MISMATCH;
    }
    if ((long long)image->rows * image->cols > INT_MAX / 2) return B2F_BAD_ARG;  // raster indices in 32 bits
    if (capacity < h->capacity(image->rows, image->cols)) return B2F_BAD_ARG;
    if (reinterpret_cast<uintptr_t>(corners) % sizeof(float2) || reinterpret_cast<uintptr_t>(count) % sizeof(int))
        return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(image->data, s);
    if (!h->bind_device()) return B2F_BAD_ARG;
    int coop = 0, d = -1;
    if (cudaGetDevice(&d) != cudaSuccess || cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, d) != cudaSuccess ||
        !coop) {
        cudaGetLastError();
        return B2F_NO_DEVICE;
    }
    cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
    if (s && cudaStreamIsCapturing(s, &capturing) != cudaSuccess) cudaGetLastError();
    // the workspace is laid out (allocated, after a synchronise of the stream) by a detect outside any capture
    if (capturing != cudaStreamCaptureStatusNone && !(h->rows == image->rows && h->cols == image->cols && h->arena.capacity()))
        return B2F_BAD_ARG;
    Ctx c = h->make_ctx(s);
    h->stats.calls++;
    if (h->layout(c, image->rows, image->cols) != B2F_OK || !c.ok()) return h->finish(c, s);
    b2f_corners::Key key;
    key.base = h->arena.capacity() ? static_cast<const void *>(h->eig.p) : nullptr;
    key.img = image->data;
    key.mask = mask ? mask->data : nullptr;
    key.corners = corners;
    key.count = count;
    key.step = image->step;
    key.mstep = mask ? mask->step : 0;
    key.rows = image->rows;
    key.cols = image->cols;
    key.type = image->type;
    key.capacity = capacity;
    key.max_corners = h->G.max_corners;
    key.quality = h->G.quality_level;
    key.md = h->G.min_distance;
    key.block_size = h->block_size;  // the taps and the criterion are baked into the response launch
    key.harris = h->harris;
    key.k = h->k;
    auto body = [&](Ctx &g) { h->schedule(g, image, mask, corners, capacity, count); };
    // inside the caller's own capture the launches go straight into the caller's graph
    c.capturing = capturing != cudaStreamCaptureStatusNone;
    if (!h->profiling && !c.capturing) {
        h->graph.run(*h, c, s, key, body);
    } else {
        body(c);
    }
    return h->finish(c, s);
}

int b2f_gftt_last_info(b2f_corners *h, b2f_gftt_info *out, void *cuda_stream) {
    using namespace b2f;
    if (!h || !out || !h->detector) return B2F_BAD_ARG;
    *out = b2f_gftt_info{};
    if (!h->st) return B2F_OK;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(h->device);
    int v[4] = {0, 0, 0, 0};
    cudaError_t e = cudaMemcpyAsync(v, h->st->info, sizeof(v), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        h->last_cuda_error = static_cast<int>(e);
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    out->candidates = v[0];
    out->kept = v[1];
    out->capped = v[2];
    out->rounds = v[3];
    return B2F_OK;
}

int b2f_corners_last_cuda_error(const b2f_corners *h) { return h ? h->last_cuda_error : 0; }

void b2f_corners_destroy(b2f_corners *h) { delete h; }

}  // extern "C"
