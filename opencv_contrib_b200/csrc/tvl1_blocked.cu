// tvl1_blocked.cu -- see tvl1_blocked.cuh for the design.
#include "tvl1_blocked.cuh"

#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace b2f {

namespace {

constexpr int R = TVL1_REGION;            // region edge (pixels)
constexpr int NT = TVL1_BLOCK_THREADS;    // 512
constexpr int PLANE_F = R * R;            // floats per staged plane
constexpr int N_IN = 10;                  // Ix, Iy, grad, rho_c, u1, u2, p11, p12, p21, p22
constexpr int N_OUT = 6;                  // u1, u2, p11, p12, p21, p22
constexpr int EX_F = 32 * R;              // floats per exchange array (32 thread-rows x 64)
constexpr size_t SMEM_BYTES = sizeof(float) * (size_t)(N_IN * PLANE_F + 4 * EX_F);

struct Regs {
    float Ix[2][4], Iy[2][4], gr[2][4], rc[2][4];
    float u1[2][4], u2[2][4], p11[2][4], p12[2][4], p21[2][4], p22[2][4];
};

__device__ __forceinline__ void ld4(const float *s, float (&d)[4]) {
    const float4 v = *reinterpret_cast<const float4 *>(s);
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
}
__device__ __forceinline__ void st4(float *s, const float (&d)[4]) {
    *reinterpret_cast<float4 *>(s) = make_float4(d[0], d[1], d[2], d[3]);
}

// K iterations on the register-resident region.  ex = 4 exchange arrays [u1 | u2 | p12 | p22].
// gxb/gyb: global coordinates of the thread's first pixel; W/H image size (BORDER only).
template <bool BORDER>
__device__ __forceinline__ void tile_iterate(Regs &r, float *ex, int iters, const Tvl1Scalars k, int lx, int tr,
                                             int gxb, int gyb, int W, int H) {
    float *ex_u1 = ex, *ex_u2 = ex + EX_F, *ex_p12 = ex + 2 * EX_F, *ex_p22 = ex + 3 * EX_F;
    const int mine = tr * R + 4 * lx;
    const int up = max(tr - 1, 0) * R + 4 * lx;
    const int dn = min(tr + 1, 31) * R + 4 * lx;


    // publish the bottom rows of p12/p22 for the first primal update
    st4(ex_p12 + mine, r.p12[1]);
    st4(ex_p22 + mine, r.p22[1]);
    __syncthreads();

    for (int it = 0; it < iters; ++it) {
        // ---------------- primal update (estimateU) ----------------
        float up12[4], up22[4];
        ld4(ex_p12 + up, up12);
        ld4(ex_p22 + up, up22);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float l11 = __shfl_up_sync(0xffffffffu, r.p11[j][3], 1, 16);
            const float l21 = __shfl_up_sync(0xffffffffu, r.p21[j][3], 1, 16);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float pl11 = i ? r.p11[j][i ? i - 1 : 0] : l11;
                float pl21 = i ? r.p21[j][i ? i - 1 : 0] : l21;
                float pu12 = j ? r.p12[0][i] : up12[i];
                float pu22 = j ? r.p22[0][i] : up22[i];
                if (BORDER) {
                    if (gxb + i == 0) { pl11 = 0.f; pl21 = 0.f; }
                    if (gyb + j == 0) { pu12 = 0.f; pu22 = 0.f; }
                }
                float a, b;
                tvl1_update_u(k, r.Ix[j][i], r.Iy[j][i], r.gr[j][i], r.rc[j][i], r.u1[j][i], r.u2[j][i],
                              r.p11[j][i], pl11, r.p12[j][i], pu12, r.p21[j][i], pl21, r.p22[j][i], pu22, a, b);
                r.u1[j][i] = a;
                r.u2[j][i] = b;
            }
        }
        st4(ex_u1 + mine, r.u1[0]);
        st4(ex_u2 + mine, r.u2[0]);
        __syncthreads();

        // ---------------- dual update (estimateDualVariables) ----------------
        float dn1[4], dn2[4];
        ld4(ex_u1 + dn, dn1);
        ld4(ex_u2 + dn, dn2);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float r1 = __shfl_down_sync(0xffffffffu, r.u1[j][0], 1, 16);
            const float r2 = __shfl_down_sync(0xffffffffu, r.u2[j][0], 1, 16);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float c1 = r.u1[j][i], c2 = r.u2[j][i];
                const float ur1 = i < 3 ? r.u1[j][i < 3 ? i + 1 : 3] : r1;
                const float ur2 = i < 3 ? r.u2[j][i < 3 ? i + 1 : 3] : r2;
                const float ud1 = j == 0 ? r.u1[1][i] : dn1[i];
                const float ud2 = j == 0 ? r.u2[1][i] : dn2[i];
                float ux1 = __fsub_rn(ur1, c1), uy1 = __fsub_rn(ud1, c1);
                float ux2 = __fsub_rn(ur2, c2), uy2 = __fsub_rn(ud2, c2);
                if (BORDER) {
                    if (gxb + i == W - 1) { ux1 = 0.f; ux2 = 0.f; }
                    if (gyb + j == H - 1) { uy1 = 0.f; uy2 = 0.f; }
                }
                tvl1_update_p2(k.taut, ux1, uy1, ux2, uy2, r.p11[j][i], r.p12[j][i], r.p21[j][i], r.p22[j][i]);
            }
        }
        st4(ex_p12 + mine, r.p12[1]);
        st4(ex_p22 + mine, r.p22[1]);
        __syncthreads();
    }
}

struct InPlanes {
    Plane p[N_IN];
};
struct OutPlanes {
    Plane p[N_OUT];
};

// One 64x64 region per CTA; plain coalesced loads/stores through the shared staging buffer.
__global__ void __launch_bounds__(NT, 1)
    k_tvl1_blocked(InPlanes in, OutPlanes out, int rows, int cols, Tvl1Scalars k, int iters, int tile) {
    extern __shared__ __align__(16) float smem[];
    float *stage = smem;
    float *ex = smem + N_IN * PLANE_F;

    const int tid = threadIdx.x;
    const int lx = tid & 15, tr = tid >> 4;
    const int gx0 = blockIdx.x * tile - iters;  // region origin (may be negative)
    const int gy0 = blockIdx.y * tile - iters;

    // ---- stage the region (zero fill outside the image) ----
#pragma unroll 1
    for (int pl = 0; pl < N_IN; ++pl) {
        const Plane P = in.p[pl];
        float *dst = stage + pl * PLANE_F;
#pragma unroll
        for (int n = 0; n < PLANE_F / NT; ++n) {
            const int idx = tid + n * NT;
            const int ry = idx >> 6, rx = idx & 63;
            const int gy = gy0 + ry, gx = gx0 + rx;
            float v = 0.f;
            if (gx >= 0 && gy >= 0 && gx < cols && gy < rows) v = __ldg(&P.at(gy, gx));
            dst[idx] = v;
        }
    }
    __syncthreads();

    Regs r;
    {
        const int o0 = (2 * tr) * R + 4 * lx, o1 = o0 + R;
        ld4(stage + 0 * PLANE_F + o0, r.Ix[0]);  ld4(stage + 0 * PLANE_F + o1, r.Ix[1]);
        ld4(stage + 1 * PLANE_F + o0, r.Iy[0]);  ld4(stage + 1 * PLANE_F + o1, r.Iy[1]);
        ld4(stage + 2 * PLANE_F + o0, r.gr[0]);  ld4(stage + 2 * PLANE_F + o1, r.gr[1]);
        ld4(stage + 3 * PLANE_F + o0, r.rc[0]);  ld4(stage + 3 * PLANE_F + o1, r.rc[1]);
        ld4(stage + 4 * PLANE_F + o0, r.u1[0]);  ld4(stage + 4 * PLANE_F + o1, r.u1[1]);
        ld4(stage + 5 * PLANE_F + o0, r.u2[0]);  ld4(stage + 5 * PLANE_F + o1, r.u2[1]);
        ld4(stage + 6 * PLANE_F + o0, r.p11[0]); ld4(stage + 6 * PLANE_F + o1, r.p11[1]);
        ld4(stage + 7 * PLANE_F + o0, r.p12[0]); ld4(stage + 7 * PLANE_F + o1, r.p12[1]);
        ld4(stage + 8 * PLANE_F + o0, r.p21[0]); ld4(stage + 8 * PLANE_F + o1, r.p21[1]);
        ld4(stage + 9 * PLANE_F + o0, r.p22[0]); ld4(stage + 9 * PLANE_F + o1, r.p22[1]);
    }

    const int gxb = gx0 + 4 * lx, gyb = gy0 + 2 * tr;
    const bool border = gx0 <= 0 || gy0 <= 0 || gx0 + R >= cols || gy0 + R >= rows;
    if (border)
        tile_iterate<true>(r, ex, iters, k, lx, tr, gxb, gyb, cols, rows);
    else
        tile_iterate<false>(r, ex, iters, k, lx, tr, gxb, gyb, cols, rows);

    // ---- write the centre tile back through the staging buffer ----
    {
        const int o0 = (2 * tr) * R + 4 * lx, o1 = o0 + R;
        st4(stage + 0 * PLANE_F + o0, r.u1[0]);  st4(stage + 0 * PLANE_F + o1, r.u1[1]);
        st4(stage + 1 * PLANE_F + o0, r.u2[0]);  st4(stage + 1 * PLANE_F + o1, r.u2[1]);
        st4(stage + 2 * PLANE_F + o0, r.p11[0]); st4(stage + 2 * PLANE_F + o1, r.p11[1]);
        st4(stage + 3 * PLANE_F + o0, r.p12[0]); st4(stage + 3 * PLANE_F + o1, r.p12[1]);
        st4(stage + 4 * PLANE_F + o0, r.p21[0]); st4(stage + 4 * PLANE_F + o1, r.p21[1]);
        st4(stage + 5 * PLANE_F + o0, r.p22[0]); st4(stage + 5 * PLANE_F + o1, r.p22[1]);
    }
    __syncthreads();
    const int tw = min(tile, cols - (int)blockIdx.x * tile);
    const int th = min(tile, rows - (int)blockIdx.y * tile);
    const int n_out = tw * th;
#pragma unroll 1
    for (int pl = 0; pl < N_OUT; ++pl) {
        const Plane P = out.p[pl];
        const float *src = stage + pl * PLANE_F;
        for (int idx = tid; idx < n_out; idx += NT) {
            const int ty = idx / tw, tx = idx - ty * tw;
            P.at(gy0 + iters + ty, gx0 + iters + tx) = src[(iters + ty) * R + iters + tx];
        }
    }
}


// ---------------------------------------------------------------------------------------------
// Persistent TMA variant.  One CTA per SM walks its tiles; the 10 input planes of a region arrive
// through cp.async.bulk.tensor (zero fill outside the image = the border ghost values), the next
// region is prefetched into the same staging buffer as soon as the current one sits in registers,
// so the HBM stream overlaps the K iterations; results leave as 8-byte vector stores straight
// from registers (they drain while the next tile computes).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int x, int y, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}

struct TmaMaps {
    CUtensorMap in[N_IN];
};
// Output descriptors of the TMA-store epilogue: the six planes of the state a launch writes, 48 x 48 boxes (the centre
// tile of an 8-pixel halo).  The tensor extent is the image, so the parts of an edge tile outside it are clipped.
constexpr int OT = R - 16;            // centre tile edge served by the TMA-store epilogue
constexpr int OT_F = OT * OT;         // floats per staged output tile
struct TmaOutMaps {
    CUtensorMap out[N_OUT];
};
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *src, int x, int y) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(src)) : "memory");
}

// One lane of a fully converged warp (the canonical TMA-issue guard: the branch is warp-uniform).
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(pred));
    return pred != 0;
}

// mode: 0 nothing, 1 = scalar store of element 0, 2 = float2 store (decided once per thread-row).
__device__ __forceinline__ void store_pairs(float *p, const float (&v)[4], int m0, int m1) {
    if (m0 == 2) *reinterpret_cast<float2 *>(p) = make_float2(v[0], v[1]);
    else if (m0 == 1) p[0] = v[0];
    if (m1 == 2) *reinterpret_cast<float2 *>(p + 2) = make_float2(v[2], v[3]);
    else if (m1 == 1) p[2] = v[2];
}

// CLOCKS (measurement aid, tools/gpu_probe_tile_cost.py): the kernel plus clock64 stamps of thread 0 around the
// phases of every tile, written to this buffer (8 values per tile: before wait, after wait, after fill, before the
// iterations, after them, after the epilogue).
__device__ long long *g_tvl1_clock_buf = nullptr;

// The halo is a multiple of 4 (tvl1_tma_launch), so every region origin is 16-byte aligned: the TMA box is exactly the
// region and threads read their pixels out of the staged rows with conflict-free LDS.128.
template <bool CLOCKS = false>
__global__ void __launch_bounds__(NT, 1)
    k_tvl1_blocked_tma(const __grid_constant__ TmaMaps maps, Plane o_u1, Plane o_u2, Plane o_p11, Plane o_p12,
                       Plane o_p21, Plane o_p22, int rows, int cols, Tvl1Scalars k, int iters, int halo, int tile,
                       int tiles_x, int ntiles, const int *__restrict__ iters_dev,
                       const __grid_constant__ TmaOutMaps omaps, int tma_store) {
    if (iters_dev) {  // device-side convergence loop: the iteration count of this pass is decided on the GPU
        iters = __ldg(iters_dev);
        if (iters < 0) return;  // pass not needed (every thread takes the same branch)
    }
    extern __shared__ __align__(1024) float smem[];
    float *stage = smem;
    float *ex = smem + N_IN * PLANE_F;
    // the six output tiles of the TMA-store epilogue alias the exchange arrays
    constexpr int EX_AREA_F = N_OUT * OT_F > 4 * EX_F ? N_OUT * OT_F : 4 * EX_F;
    uint64_t *bar = reinterpret_cast<uint64_t *>(ex + EX_AREA_F);

    const int tid = threadIdx.x;
    const int lx = tid & 15, tr = tid >> 4;
    constexpr uint32_t kPlaneBytes = PLANE_F * sizeof(float);

    // The ten plane loads of a region are issued by ten warps (one elected lane each, each announcing its own 16 KB on
    // the barrier), the six stores of the TMA-store epilogue by the other six.  One lane issuing all ten loads would
    // put them on the critical path, every other warp waiting for it at the first barrier.
    const int wid = tid >> 5;
    const bool leader = elect_one();
    const bool load_issuer = leader && wid < N_IN;
    const bool store_issuer = leader && wid >= N_IN && wid < N_IN + N_OUT;
    if (tid == 0) {
        mbar_init(bar, N_IN);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    // bit 1 of tma_store: walk the tiles from the last to the first.  Passes alternate direction, so a pass begins where the
    // previous kernel of the stream ended: the first region of every CTA -- the cold load nothing hides -- is then the data
    // written (or read) last, i.e. still in L2.
    const bool rev = (tma_store & 2) != 0;
    tma_store &= 1;
    int t = blockIdx.x;
    auto issue_loads = [&](int tx, int ty) {
        const int bx = (tx * tile - halo) & ~3, by = ty * tile - halo;  // & ~3: see `shift` below
        mbar_expect_tx(bar, kPlaneBytes);
        tma_load_2d(stage + wid * PLANE_F, &maps.in[wid], bx, by, bar);
    };
    if (load_issuer && t < ntiles) {
        const int tt = rev ? ntiles - 1 - t : t;
        const int ty = tt / tiles_x, tx = tt - ty * tiles_x;
        issue_loads(tx, ty);
    }
    uint32_t parity = 0;
    for (; t < ntiles; t += gridDim.x) {
        const int tt = rev ? ntiles - 1 - t : t;
        const int ty = tt / tiles_x, tx = tt - ty * tiles_x;
        const int gx0 = tx * tile - halo, gy0 = ty * tile - halo;
        // Region origins are multiples of 4, so the rounding of the box origin above is a no-op and `shift` is 0.  Both
        // stay: without them ptxas schedules the per-tile set-up differently, and a single-stream 1080p pair measured
        // about 2 % slower on an H100.
        const int shift = gx0 - (gx0 & ~3);
        long long clk[6];
        if (CLOCKS) clk[0] = clock64();
        mbar_wait(bar, parity);
        parity ^= 1;
        if (CLOCKS) clk[1] = clock64();

        Regs r;
        {
            const int o0 = (2 * tr) * R + shift + 4 * lx, o1 = o0 + R;
            auto ldrow = [&](int pl, float (&a)[4], float (&b)[4]) {
                ld4(stage + pl * PLANE_F + o0, a);
                ld4(stage + pl * PLANE_F + o1, b);
            };
            ldrow(0, r.Ix[0], r.Ix[1]);
            ldrow(1, r.Iy[0], r.Iy[1]);
            ldrow(2, r.gr[0], r.gr[1]);
            ldrow(3, r.rc[0], r.rc[1]);
            ldrow(4, r.u1[0], r.u1[1]);
            ldrow(5, r.u2[0], r.u2[1]);
            ldrow(6, r.p11[0], r.p11[1]);
            ldrow(7, r.p12[0], r.p12[1]);
            ldrow(8, r.p21[0], r.p21[1]);
            ldrow(9, r.p22[0], r.p22[1]);
        }
        if (tma_store && store_issuer)  // the previous tile's TMA stores have read their staging tiles
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncthreads();  // the staging buffer is free again
        if (CLOCKS) clk[2] = clock64();

        // No proxy fence here: the generic-proxy reads of the staging buffer completed before the barrier above (their
        // values sit in registers); the copy engine only overwrites it (the consumer-release -> producer-load hand-off
        // of every TMA pipeline).  The fence used to compile to MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC in the issuing warp.
        const int tn = t + gridDim.x;
        if (load_issuer && tn < ntiles) {
            const int tnn = rev ? ntiles - 1 - tn : tn;
            const int ny = tnn / tiles_x, nx = tnn - ny * tiles_x;
            issue_loads(nx, ny);
        }

        const int gxb = gx0 + 4 * lx, gyb = gy0 + 2 * tr;
        const bool border = gx0 <= 0 || gy0 <= 0 || gx0 + R >= cols || gy0 + R >= rows;
        if (CLOCKS) clk[3] = clock64();
        if (border)
            tile_iterate<true>(r, ex, iters, k, lx, tr, gxb, gyb, cols, rows);
        else
            tile_iterate<false>(r, ex, iters, k, lx, tr, gxb, gyb, cols, rows);
        if (CLOCKS) clk[4] = clock64();

        if (tma_store) {
            // centre tile -> six dense 48 x 48 tiles in shared memory (over the exchange arrays) -> one TMA store each.
            // 12 STS.128 per thread replace 24 predicated STG.64 and their address arithmetic; the copy engine clips
            // edge tiles against the image.  (halo == 8 and tile == 48 here.)
            float *ot = ex;
            const int ox = 4 * lx - 8, oy = 2 * tr - 8;
            if (ox >= 0 && ox < OT) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    if (oy + j >= 0 && oy + j < OT) {
                        float *d = ot + (oy + j) * OT + ox;
                        st4(d, r.u1[j]);
                        st4(d + OT_F, r.u2[j]);
                        st4(d + 2 * OT_F, r.p11[j]);
                        st4(d + 3 * OT_F, r.p12[j]);
                        st4(d + 4 * OT_F, r.p21[j]);
                        st4(d + 5 * OT_F, r.p22[j]);
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (store_issuer) {
                tma_store_2d(&omaps.out[wid - N_IN], ot + (wid - N_IN) * OT_F, tx * tile, ty * tile);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            if (CLOCKS && tid == 0 && g_tvl1_clock_buf) {
                clk[5] = clock64();
#pragma unroll
                for (int i = 0; i < 6; ++i) g_tvl1_clock_buf[(size_t)t * 8 + i] = clk[i];
            }
            continue;
        }
        // centre tile -> global, 8-byte stores (halo, tile and gx0 are even, so pairs never straddle);
        // all six output planes share one pitch, so one element offset serves them all
        const int rx = 4 * lx;
        const bool okx0 = rx >= halo && rx < R - halo && gxb < cols;
        const bool okx1 = rx + 2 >= halo && rx + 2 < R - halo && gxb + 2 < cols;
        const int m0 = okx0 ? (gxb + 1 < cols ? 2 : 1) : 0;
        const int m1 = okx1 ? (gxb + 3 < cols ? 2 : 1) : 0;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int ry = 2 * tr + j, gy = gyb + j;
            if (ry >= halo && ry < R - halo && gy < rows && (m0 | m1)) {
                const size_t off = (size_t)gy * o_u1.pitch + gxb;
                store_pairs(o_u1.p + off, r.u1[j], m0, m1);
                store_pairs(o_u2.p + off, r.u2[j], m0, m1);
                store_pairs(o_p11.p + off, r.p11[j], m0, m1);
                store_pairs(o_p12.p + off, r.p12[j], m0, m1);
                store_pairs(o_p21.p + off, r.p21[j], m0, m1);
                store_pairs(o_p22.p + off, r.p22[j], m0, m1);
            }
        }
    }
    if (tma_store && store_issuer)  // the staging tiles must outlive the copy engine's reads of them
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side of the TMA variant
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encoder() {
    static const EncodeTiledFn fn = [] {  // a function-local static is initialised once, thread-safely
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                       q == cudaDriverEntryPointSuccess
                   ? reinterpret_cast<EncodeTiledFn>(p)
                   : nullptr;
    }();
    return fn;
}

static bool encode_plane(CUtensorMap *m, const Plane &P, int rows, int cols) {
    EncodeTiledFn enc = get_encoder();
    if (!enc) return false;
    const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t gstr[1] = {(cuuint64_t)P.pitch * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)R, (cuuint32_t)R};
    const cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, P.p, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Generic 2-D float32 tiled tensor map (used by the Farneback persistent kernel as well): width x height elements,
// row pitch in bytes, box_w x box_h element boxes, out-of-bounds elements read as zero.
bool tma_encode_2d_f32(void *map_out, const float *base, uint64_t width, uint64_t height, uint64_t pitch_bytes,
                       uint32_t box_w, uint32_t box_h) {
    EncodeTiledFn enc = get_encoder();
    if (!enc) return false;
    const cuuint64_t gdim[2] = {width, height};
    const cuuint64_t gstr[1] = {pitch_bytes};
    const cuuint32_t box[2] = {box_w, box_h};
    const cuuint32_t estr[2] = {1, 1};
    return enc(static_cast<CUtensorMap *>(map_out), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), gdim,
               gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// one block = the input descriptors (64 x 64 boxes), followed by the output descriptors (48 x 48 boxes on the planes
// of the other state) of the TMA-store epilogue
size_t tvl1_tma_maps_bytes() { return sizeof(TmaMaps) + sizeof(TmaOutMaps); }

bool tvl1_tma_build_maps(void *dst, const Tvl1BlockedPlanes &B, int cur, int rows, int cols) {
    TmaMaps *m = static_cast<TmaMaps *>(dst);
    const Tvl1State &si = B.s[cur];
    const Plane in[N_IN] = {B.I1wx, B.I1wy, B.grad, B.rho_c, si.u1, si.u2, si.p11, si.p12, si.p21, si.p22};
    for (int i = 0; i < N_IN; ++i)
        if (!encode_plane(&m->in[i], in[i], rows, cols)) return false;
    TmaOutMaps *om = reinterpret_cast<TmaOutMaps *>(m + 1);
    const Tvl1State &so = B.s[cur ^ 1];
    const Plane out[N_OUT] = {so.u1, so.u2, so.p11, so.p12, so.p21, so.p22};
    for (int i = 0; i < N_OUT; ++i)
        if (!tma_encode_2d_f32(&om->out[i], out[i].p, (uint64_t)cols, (uint64_t)rows, (uint64_t)out[i].pitch * sizeof(float),
                               OT, OT))
            return false;
    return true;
}
static const TmaOutMaps *out_maps(const void *maps) {
    return reinterpret_cast<const TmaOutMaps *>(static_cast<const TmaMaps *>(maps) + 1);
}

// staged planes, then the four exchange arrays with room for the six 48 x 48 output tiles of the TMA-store epilogue
// (they alias the exchange arrays), then the barrier
constexpr size_t smem_tma_bytes() {
    return sizeof(float) * ((size_t)N_IN * PLANE_F + ((size_t)N_OUT * OT_F > 4 * (size_t)EX_F ? (size_t)N_OUT * OT_F : 4 * (size_t)EX_F)) + 64;
}
static_assert(smem_tma_bytes() <= 227 * 1024, "TV-L1 TMA kernel: shared memory over the 227 KB limit");

void tvl1_tma_launch(Ctx &c, int cls, const void *maps, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                     const Tvl1Scalars &k, int iters, int num_sms) {
    const Tvl1State &so = B.s[cur ^ 1];
    const TmaMaps *m = static_cast<const TmaMaps *>(maps);
    const TmaOutMaps *om = out_maps(maps);
    // Halo rounded up to a multiple of 4: with iters <= TVL1_KMAX every halo and tile is then a multiple of 4, so every
    // pass -- also the 6-iteration one that ends a 30-iteration warp -- takes the 64-wide boxes and the conflict-free
    // LDS.128 fill.  Passes with an 8-pixel halo leave through the TMA-store epilogue, the others through 8-byte stores.
    const int halo = (iters + 3) & ~3;
    const int tile = R - 2 * halo;
    const int tiles_x = div_up(cols, tile), tiles_y = div_up(rows, tile);
    const int ntiles = tiles_x * tiles_y;
    const int grid = ntiles < num_sms ? ntiles : num_sms;
    const double bytes = 64.0 * (double)rows * cols * iters;
    // passes alternate their walking direction (see the kernel); `cur` flips with every pass and is 0 for the pass that
    // follows the warp kernel, which ended at the bottom of the image
    static const bool norev = getenv("B2F_DBG_TVL1_NOREV") != nullptr;
    const bool reverse = !norev && cur == 0;
    // measurement aid (tools/gpu_probe_tile_cost.py): run fewer iterations than the geometry was laid out for, so the
    // per-tile cost of a pass (TMA wait, register fill, epilogue) separates from the per-iteration cost.  Results are
    // garbage with it; never set outside that probe.
    if (const char *dbg = getenv("B2F_DBG_TVL1_ITERS")) iters = atoi(dbg) < iters ? atoi(dbg) : iters;
    if (halo == 8 && !c.capturing && getenv("B2F_DBG_TVL1_CLOCKS")) {  // phase clocks of every tile
        static long long *buf = nullptr;
        static size_t cap = 0;
        const size_t need = (size_t)ntiles * 8;
        if (need > cap) {
            cudaFree(buf);
            cudaMalloc(&buf, need * sizeof(long long));
            cap = need;
            cudaMemcpyToSymbol(g_tvl1_clock_buf, &buf, sizeof(buf));
        }
        cudaMemsetAsync(buf, 0, need * sizeof(long long), c.stream);
        B2F_LAUNCH(c, cls, bytes, k_tvl1_blocked_tma<true>, dim3(grid), dim3(NT), smem_tma_bytes(), *m, so.u1, so.u2,
                   so.p11, so.p12, so.p21, so.p22, rows, cols, k, iters, halo, tile, tiles_x, ntiles, nullptr, *om, 1);
        cudaStreamSynchronize(c.stream);
        std::vector<long long> h(need);
        cudaMemcpy(h.data(), buf, need * sizeof(long long), cudaMemcpyDeviceToHost);
        double ph[6] = {0, 0, 0, 0, 0, 0};  // wait, fill, issue+setup, iterations, epilogue, gap to the next tile of the CTA
        int n = 0, ngap = 0;
        for (int t = 0; t < ntiles; ++t) {
            const long long *q = &h[(size_t)t * 8];
            for (int i = 0; i < 5; ++i) ph[i] += (double)(q[i + 1] - q[i]);
            ++n;
            if (t + grid < ntiles) { ph[5] += (double)(h[(size_t)(t + grid) * 8] - q[5]); ++ngap; }
        }
        fprintf(stderr, "tvl1 clocks %dx%d iters %d tiles %d: wait %.0f fill %.0f setup %.0f iterate %.0f (%.0f / iteration) "
                        "epilogue %.0f loop-back %.0f cycles per tile\n", cols, rows, iters, ntiles, ph[0] / n, ph[1] / n,
                ph[2] / n, ph[3] / n, iters ? ph[3] / n / iters : 0.0, ph[4] / n, ngap ? ph[5] / ngap : 0.0);
        return;
    }
    B2F_LAUNCH(c, cls, bytes, k_tvl1_blocked_tma<>, dim3(grid), dim3(NT), smem_tma_bytes(), *m, so.u1, so.u2, so.p11,
               so.p12, so.p21, so.p22, rows, cols, k, iters, halo, tile, tiles_x, ntiles, nullptr, *om,
               (halo == 8 ? 1 : 0) | (reverse ? 2 : 0));
}

// One pass whose iteration count (0..8; negative = skip the pass) is read from device memory at run time: fixed
// geometry (8-pixel halo, 48-pixel tiles, 64-wide boxes) so the launch can sit in a CUDA graph's while-loop body.
void tvl1_tma_launch_dev(Ctx &c, int cls, const void *maps, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                         const Tvl1Scalars &k, const int *iters_dev, int num_sms) {
    const Tvl1State &so = B.s[cur ^ 1];
    const int halo = 8, tile = R - 2 * halo;
    const int tiles_x = div_up(cols, tile), tiles_y = div_up(rows, tile);
    const int ntiles = tiles_x * tiles_y;
    const int grid = ntiles < num_sms ? ntiles : num_sms;
    const TmaMaps *m = static_cast<const TmaMaps *>(maps);
    B2F_LAUNCH(c, cls, 0.0, k_tvl1_blocked_tma<>, dim3(grid), dim3(NT), smem_tma_bytes(), *m, so.u1, so.u2, so.p11,
               so.p12, so.p21, so.p22, rows, cols, k, 0, halo, tile, tiles_x, ntiles, iters_dev, *out_maps(maps), 1);
}

void tvl1_blocked_init(Ctx &c) {
    static DeviceOnce attrs;
    attrs.run(c, [&] {
        c.check(cudaFuncSetAttribute(k_tvl1_blocked, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        c.check(cudaFuncSetAttribute(k_tvl1_blocked_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem_tma_bytes()));
        c.check(cudaFuncSetAttribute(k_tvl1_blocked_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem_tma_bytes()));
    });
}

int tvl1_blocked_pick_k(int knob, int remaining, int rows, int cols) {
    (void)rows;
    (void)cols;
    int kk = knob > 0 ? knob : 8;
    if (kk > TVL1_KMAX) kk = TVL1_KMAX;
    if (kk > remaining) kk = remaining;
    return kk;
}

void tvl1_blocked_launch(Ctx &c, int cls, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                         const Tvl1Scalars &k, int iters) {
    const Tvl1State &si = B.s[cur], &so = B.s[cur ^ 1];
    InPlanes in;
    in.p[0] = B.I1wx; in.p[1] = B.I1wy; in.p[2] = B.grad; in.p[3] = B.rho_c;
    in.p[4] = si.u1; in.p[5] = si.u2; in.p[6] = si.p11; in.p[7] = si.p12; in.p[8] = si.p21; in.p[9] = si.p22;
    OutPlanes out;
    out.p[0] = so.u1; out.p[1] = so.u2; out.p[2] = so.p11; out.p[3] = so.p12; out.p[4] = so.p21; out.p[5] = so.p22;
    const int tile = R - 2 * iters;
    const dim3 grid(div_up(cols, tile), div_up(rows, tile));
    const double bytes = 64.0 * (double)rows * cols * iters;  // algorithmic: 64 B / px / iteration
    B2F_LAUNCH(c, cls, bytes, k_tvl1_blocked, grid, dim3(NT), SMEM_BYTES, in, out, rows, cols, k, iters, tile);
}

}  // namespace b2f
