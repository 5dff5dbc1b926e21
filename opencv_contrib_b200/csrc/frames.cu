// frames.cu -- cv::cuda::interpolateFrames (cudalegacy/src/interpolate_frames.cpp:54-111), the consumer
// that sits right after the flow solvers (SURVEY.md 8f rank 2).
//
// The reference runs 13 launches: four times {clear coverage, forward splat with a 2x2 point-spread
// function and float atomics, normalise} (NPP_staging.cu:1838-1905,1956-1968,2022-2063) and one blend
// through two linear-filtered textures (:1648-1702).  Here: one memset, ONE splat kernel that scatters
// both flow pairs (3 atomics per tap instead of 4: the two splats of a pair share their weights), and one
// kernel that normalises, writes the reference's scratch layout back and blends -- the blend only reads
// the interpolated flows at its own pixel, so normalisation fuses into it.  HBM-bound: 6 plane reads +
// 24 atomics per pixel in the splat, 8 reads + 7 writes + 2-4 bilinear fetches in the blend.
//
// B2F_INTERP_REFERENCE keeps the reference's three defects (documented in include/b200flow.h);
// B2F_INTERP_CORRECTED removes them.
#include "common.cuh"

namespace b2f {
namespace {

struct FramePlanes {
    const float *frame0, *frame1, *fu, *fv, *bu, *bv;
    float *out;
    float *cov0, *cov1, *fwdU, *fwdV, *bwdU, *bwdV;
    int w, h, s;  // s = stride in floats, shared by every plane (interpolate_frames.cpp:82)
};

// One 2x2 splat of up to three values that share weights (ForwardWarpKernel_PSF2x2, NPP_staging.cu:1838-1905:
// same coordinate arithmetic, same tap order, value*weight rounded before the atomic add).
__device__ __forceinline__ void splat3(float u, float v, float time_scale, int j, int i, int w, int h, int s,
                                       float a, float b, float *__restrict__ dstA, float *__restrict__ dstB,
                                       float *__restrict__ norm) {
    const float cx = u * time_scale + (float)j + 1.0f;
    const float cy = v * time_scale + (float)i + 1.0f;
    float px, py;
    const float dx = modff(cx, &px);
    const float dy = modff(cy, &py);
    int tx = (int)px, ty = (int)py;
    auto tap = [&](float weight) {
        if (!((tx >= w) || (tx < 0) || (ty >= h) || (ty < 0))) {
            const int o = ty * s + tx;
            atomicAdd(dstA + o, a * weight);
            atomicAdd(dstB + o, b * weight);
            atomicAdd(norm + o, weight);
        }
    };
    tap(dx * dy);
    tx -= 1;
    tap((1.0f - dx) * dy);
    ty -= 1;
    tap((1.0f - dx) * (1.0f - dy));
    tx += 1;
    tap(dx * (1.0f - dy));
}

__global__ void __launch_bounds__(256) k_interp_splat(FramePlanes P, float pos) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= P.h || j >= P.w) return;
    const int o = i * P.s + j;
    const float fu = __ldg(P.fu + o), fv = __ldg(P.fv + o);
    splat3(fu, fv, pos, j, i, P.w, P.h, P.s, fu, fv, P.fwdU, P.fwdV, P.cov0);
    const float bu = __ldg(P.bu + o), bv = __ldg(P.bv + o);
    splat3(bu, bv, 1.0f - pos, j, i, P.w, P.h, P.s, bu, bv, P.bwdU, P.bwdV, P.cov1);
}

// unnormalised coordinates, linear filter, clamp addressing (cudev::Texture defaults + cudaFilterModeLinear,
// NPP_staging.cu:1696-1697).  Weights carry 8 fractional bits like the texture unit (CUDA programming guide,
// "linear filtering").  Called as tex(y, x) by the reference.
__device__ __forceinline__ float tex_linear(const float *__restrict__ img, int w, int h, int s, float y, float x) {
    const float xb = x - 0.5f, yb = y - 0.5f;
    const float fx = floorf(xb), fy = floorf(yb);
    const float ax = floorf((xb - fx) * 256.f + 0.5f) * (1.f / 256.f);
    const float ay = floorf((yb - fy) * 256.f + 0.5f) * (1.f / 256.f);
    const int x0 = (int)fminf(fmaxf(fx, -2.f), (float)w + 1.f), y0 = (int)fminf(fmaxf(fy, -2.f), (float)h + 1.f);
    const int xa = clampi(x0, 0, w - 1), xc = clampi(x0 + 1, 0, w - 1);
    const int ya = clampi(y0, 0, h - 1), yc = clampi(y0 + 1, 0, h - 1);
    const float t00 = __ldg(img + ya * s + xa), t01 = __ldg(img + ya * s + xc);
    const float t10 = __ldg(img + yc * s + xa), t11 = __ldg(img + yc * s + xc);
    return (1.f - ax) * (1.f - ay) * t00 + ax * (1.f - ay) * t01 + (1.f - ax) * ay * t10 + ax * ay * t11;
}

__device__ __forceinline__ float normalise(float value, float scale) {  // NormalizeKernel, NPP_staging.cu:1956-1968
    const float inv = (scale == 0.0f) ? 1.0f : (1.0f / scale);
    return value * inv;
}

template <bool CORRECTED>
__global__ void __launch_bounds__(128) k_interp_blend(FramePlanes P, float theta) {
    const int ix = blockIdx.x * blockDim.x + threadIdx.x;
    const int iy = blockIdx.y * blockDim.y + threadIdx.y;
    if (ix >= P.w || iy >= P.h) return;
    const int pos = ix + P.s * iy;
    float c0 = P.cov0[pos], c1 = P.cov1[pos];
    float u, v, ur, vr;
    if (CORRECTED) {
        u = normalise(P.fwdU[pos], c0);
        v = normalise(P.fwdV[pos], c0);
        ur = normalise(P.bwdU[pos], c1);
        vr = normalise(P.bwdV[pos], c1);
    } else {
        // The second splat of each pair clears the coverage with MemsetKernel, which indexes i*w + j
        // (NPP_staging.cu:1985-1996): only the first w*h floats of the pitched plane are cleared, the rest
        // accumulates the same weights a second time.
        const bool cleared = pos < P.w * P.h;
        const float c0b = cleared ? c0 : c0 + c0;
        const float c1b = cleared ? c1 : c1 + c1;
        u = normalise(P.fwdU[pos], c0);
        v = normalise(P.fwdV[pos], c0b);
        // 4th splat targets bwdU again (NPP_staging.cu:1779-1787): the normalised bwdU receives the bv
        // splat on top and is normalised a second time; bwdV is never written.
        ur = normalise(normalise(P.bwdU[pos], c1) + P.bwdV[pos], c1b);
        vr = 0.0f;
        c0 = c0b;
        c1 = c1b;
    }
    // leave the scratch planes as the reference leaves them
    P.fwdU[pos] = u;
    P.fwdV[pos] = v;
    P.bwdU[pos] = ur;
    P.bwdV[pos] = vr;
    if (!CORRECTED) {
        P.cov0[pos] = c0;
        P.cov1[pos] = c1;
    }

    const float x = (float)ix + 0.5f, y = (float)iy + 0.5f;
    const bool b0 = c0 > 1e-4f, b1 = c1 > 1e-4f;
    float r;
    if (b0 && b1) {  // visible in both frames
        const float *second = CORRECTED ? P.frame1 : P.frame0;  // NPP_staging.cu:1666 samples texSrc0 twice
        r = tex_linear(P.frame0, P.w, P.h, P.s, y - v * theta, x - u * theta) * (1.0f - theta) +
            tex_linear(second, P.w, P.h, P.s, y + v * (1.0f - theta), x + u * (1.0f - theta)) * theta;
    } else if (b0) {  // first frame only
        r = tex_linear(P.frame0, P.w, P.h, P.s, y - v * theta, x - u * theta);
    } else {  // second frame only
        r = tex_linear(P.frame1, P.w, P.h, P.s, y - vr * (1.0f - theta), x - ur * (1.0f - theta));
    }
    P.out[pos] = r;
}

}  // namespace
}  // namespace b2f

extern "C" int b2f_interpolate_frames(const b2f_image *frame0, const b2f_image *frame1, const b2f_image *fu,
                                      const b2f_image *fv, const b2f_image *bu, const b2f_image *bv, float pos,
                                      b2f_image *new_frame, b2f_image *buf, int flags, void *cuda_stream) {
    using namespace b2f;
    if (!frame0 || !frame0->data || !new_frame || !buf || !buf->data) return B2F_BAD_ARG;
    if (frame0->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;  // interpolate_frames.cpp:57
    if (frame0->rows <= 0 || frame0->cols <= 0 || frame0->step % sizeof(float) != 0 ||
        frame0->step < frame0->cols * sizeof(float))
        return B2F_BAD_ARG;
    const b2f_image *same[] = {frame1, fu, fv, bu, bv, new_frame};
    for (const b2f_image *m : same) {
        if (!m || !m->data) return B2F_BAD_ARG;
        if (m->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
        if (m->rows != frame0->rows || m->cols != frame0->cols) return B2F_SIZE_MISMATCH;  // :58-62
        if (m->step != frame0->step) return B2F_BAD_ARG;                                     // :82
    }
    if (buf->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    if (buf->rows != 6 * frame0->rows || buf->cols != frame0->cols) return B2F_SIZE_MISMATCH;  // :66
    if (buf->step != frame0->step) return B2F_BAD_ARG;
    if (flags != B2F_INTERP_REFERENCE && flags != B2F_INTERP_CORRECTED) return B2F_BAD_ARG;

    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(frame0->data, s);
    FramePlanes P;
    P.w = frame0->cols;
    P.h = frame0->rows;
    P.s = static_cast<int>(frame0->step / sizeof(float));
    P.frame0 = static_cast<const float *>(frame0->data);
    P.frame1 = static_cast<const float *>(frame1->data);
    P.fu = static_cast<const float *>(fu->data);
    P.fv = static_cast<const float *>(fv->data);
    P.bu = static_cast<const float *>(bu->data);
    P.bv = static_cast<const float *>(bv->data);
    P.out = static_cast<float *>(new_frame->data);
    float *b = static_cast<float *>(buf->data);
    const size_t plane = (size_t)P.s * P.h;
    P.cov0 = b;
    P.cov1 = b + plane;
    P.fwdU = b + 2 * plane;
    P.fwdV = b + 3 * plane;
    P.bwdU = b + 4 * plane;
    P.bwdV = b + 5 * plane;

    // buf.setTo(0), :67 -- the 6h x w view only: the columns past w of a pitched buf belong to the caller
    const size_t row = (size_t)P.w * sizeof(float);
    cudaError_t e = buf->step == row ? cudaMemsetAsync(b, 0, 6 * plane * sizeof(float), s)
                                     : cudaMemset2DAsync(b, buf->step, 0, row, 6 * (size_t)P.h, s);
    if (e == cudaSuccess) {
        const dim3 block(32, 8), grid(div_up(P.w, 32), div_up(P.h, 8));
        k_interp_splat<<<grid, block, 0, s>>>(P, pos);
        const dim3 block2(32, 4), grid2(div_up(P.w, 32), div_up(P.h, 4));
        if (flags == B2F_INTERP_CORRECTED)
            k_interp_blend<true><<<grid2, block2, 0, s>>>(P, pos);
        else
            k_interp_blend<false><<<grid2, block2, 0, s>>>(P, pos);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && s == nullptr) e = cudaDeviceSynchronize();  // interpolate_frames.cpp:107-108
    if (e != cudaSuccess) {
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    return B2F_OK;
}
