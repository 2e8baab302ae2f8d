/*
 * views.cu -- StereoView::set_scale on the device (reference:
 * lib/stereo_view.cc:24-46, 97-188; mve::image::blur_gaussian,
 * byte_to_float_image): per-scale Gaussian blur of the byte image, then the
 * 3x3 quadratic-fit gradient (2 ch) and Hessian (3 ch). This is the producer
 * of the Gauss-Newton kernels' image inputs (SURVEY.md section 8f, "next"
 * row 1); doing it here shrinks the per-scale upload from 41.5 MB to 2 MB per
 * 2 MP view.
 *
 * Bit-compatible with the CPU: fp32 blur with the reference's operation
 * order (value * weight, then add; no FMA contraction; normalise by the
 * weight sum), kernel weights from the host's expf, fp64 stencil with the
 * 6x9 matrix applied term by term.
 */
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "common.cuh"

namespace smvsb {

namespace {

/* blur radius ceil(2.884 * (0.12 * 2^scale + 0.2)): 45 at scale 7, 90 at
 * scale 8, the coarsest scale a surface starts at */
constexpr int BLUR_MAX_KS = 90;

struct BlurKernel
{
    int ks;
    float w[BLUR_MAX_KS + 1];
    float wsum;
};

__device__ __forceinline__ float
pixel_value (uint8_t v)
{
    /* mve::image::byte_to_float_image: v / 255, clamped */
    float const f = __fdiv_rn(static_cast<float>(v), 255.0f);
    return fminf(1.0f, fmaxf(0.0f, f));
}

__device__ __forceinline__ float
pixel_value (float v)
{
    return v;
}

/* x pass: (byte -> float, v / 255, clamped ->) blur along x. C = 3: the
 * three interleaved channels of a colour view, each on its own
 * (mve::image::blur_gaussian works channel by channel). */
template <typename T, int C>
__global__ void
blur_x_kernel (T const* __restrict__ img, int w, int h,
    BlurKernel const k, float* __restrict__ out)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y;
    if (x >= w)
        return;
    T const* row = img + static_cast<size_t>(y) * w * C;
    float acc[C];
#pragma unroll
    for (int ch = 0; ch < C; ++ch)
        acc[ch] = 0.0f;
    for (int i = -k.ks; i <= k.ks; ++i)
    {
        int const xi = min(max(x + i, 0), w - 1);
#pragma unroll
        for (int ch = 0; ch < C; ++ch)
            acc[ch] = __fadd_rn(acc[ch], __fmul_rn(pixel_value(
                row[C * xi + ch]), k.w[abs(i)]));
    }
    float* o = out + (static_cast<size_t>(y) * w + x) * C;
#pragma unroll
    for (int ch = 0; ch < C; ++ch)
        o[ch] = __fdiv_rn(acc[ch], k.wsum);
}

/* y pass into `gray`. C = 3 then desaturates like
 * mve::image::desaturate<float>(DESATURATE_LUMINANCE), v0 * 0.21f +
 * v1 * 0.72f + v2 * 0.07f evaluated left to right
 * (StereoView::initialize_image_gradients, lib/stereo_view.cc:24-62), and
 * writes the blurred colour image (StereoView::scaleimage) to colour_out
 * when it is not null. */
template <int C>
__global__ void
blur_y_kernel (float const* __restrict__ in, int w, int h,
    BlurKernel const k, float* __restrict__ gray,
    float* __restrict__ colour_out)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y;
    if (x >= w)
        return;
    float acc[C];
#pragma unroll
    for (int ch = 0; ch < C; ++ch)
        acc[ch] = 0.0f;
    for (int i = -k.ks; i <= k.ks; ++i)
    {
        int const yi = min(max(y + i, 0), h - 1);
        float const* p = in + (static_cast<size_t>(yi) * w + x) * C;
        float const wgt = k.w[abs(i)];
#pragma unroll
        for (int ch = 0; ch < C; ++ch)
            acc[ch] = __fadd_rn(acc[ch], __fmul_rn(p[ch], wgt));
    }
    float v[C];
#pragma unroll
    for (int ch = 0; ch < C; ++ch)
        v[ch] = __fdiv_rn(acc[ch], k.wsum);
    size_t const pix = static_cast<size_t>(y) * w + x;
    if constexpr (C == 1)
        gray[pix] = v[0];
    else
    {
        if (colour_out != nullptr)
        {
#pragma unroll
            for (int ch = 0; ch < C; ++ch)
                colour_out[C * pix + ch] = v[ch];
        }
        gray[pix] = __fadd_rn(__fadd_rn(__fmul_rn(v[0], 0.21f),
            __fmul_rn(v[1], 0.72f)), __fmul_rn(v[2], 0.07f));
    }
}

__global__ void
byte_to_float_kernel (uint8_t const* __restrict__ img, int n,
    float* __restrict__ out)
{
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    float const v = __fdiv_rn(static_cast<float>(img[i]), 255.0f);
    out[i] = fminf(1.0f, fmaxf(0.0f, v));
}

/* compute_gradients_and_hessian, lib/stereo_view.cc:97-188, of pixel pix.
 * at(a, b) is the blurred image at offset (a, b) from the pixel; row r of
 * the 6x9 matrix times the 3x3 neighbourhood (x offset outer, y offset
 * inner), all nine terms in order like math::Matrix::mult; zero on the
 * one-pixel image border (inside = false).
 *   mode 0: write float2 gradient            (main view, shading gradient)
 *   mode 1: write packed texel gx gy hxx hxy hyy 0 0 0 (neighbours)        */
template <typename At>
__device__ __forceinline__ void
store_grad_hess (At const& at, bool inside, int mode,
    float* __restrict__ out, size_t pix)
{
    double r[6] = {0, 0, 0, 0, 0, 0};
    if (inside)
    {
        double v[9];
        int c = 0;
#pragma unroll
        for (int a = -1; a < 2; ++a)
#pragma unroll
            for (int b = -1; b < 2; ++b)
                v[c++] = at(a, b);
        double const s6 = 1.0 / 6.0, s3 = -1.0 / 3.0, s4 = 1.0 / 4.0;
        double const M[6][9] = {
            { s6, s6, s6, s3, s3, s3, s6, s6, s6 },
            { s6, s3, s6, s6, s3, s6, s6, s3, s6 },
            { s4, 0.0, -s4, 0.0, 0.0, 0.0, -s4, 0.0, s4 },
            { -s6, -s6, -s6, 0.0, 0.0, 0.0, s6, s6, s6 },
            { -s6, 0.0, s6, -s6, 0.0, s6, -s6, 0.0, s6 },
            { -1.0 / 9.0, 2.0 / 9.0, -1.0 / 9.0, 2.0 / 9.0, 5.0 / 9.0,
              2.0 / 9.0, -1.0 / 9.0, 2.0 / 9.0, -1.0 / 9.0 } };
#pragma unroll
        for (int row = 0; row < 5; ++row)
        {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 9; ++k)
                s = __dadd_rn(s, __dmul_rn(M[row][k], v[k]));
            r[row] = s;
        }
    }
    if (mode == 0)
    {
        reinterpret_cast<float2*>(out)[pix] = make_float2(
            static_cast<float>(r[3]), static_cast<float>(r[4]));
    }
    else
    {
        float4 a, b;
        a.x = static_cast<float>(r[3]);
        a.y = static_cast<float>(r[4]);
        a.z = static_cast<float>(__dmul_rn(2.0, r[0]));
        a.w = static_cast<float>(r[2]);
        b.x = static_cast<float>(__dmul_rn(2.0, r[1]));
        b.y = b.z = b.w = 0.0f;
        reinterpret_cast<float4*>(out)[2 * pix] = a;
        reinterpret_cast<float4*>(out)[2 * pix + 1] = b;
    }
}

__global__ void
grad_hess_kernel (float const* __restrict__ in, int w, int h, int mode,
    float* __restrict__ out)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y;
    if (x >= w)
        return;
    store_grad_hess([&](int a, int b) {
            return in[static_cast<size_t>(y + b) * w + (x + a)]; },
        x >= 1 && x < w - 1 && y >= 1 && y < h - 1, mode, out,
        static_cast<size_t>(y) * w + x);
}

__global__ void
unpack_texels_kernel (float const* __restrict__ texels, int n,
    float* __restrict__ grad, float* __restrict__ hess)
{
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    float4 const a = reinterpret_cast<float4 const*>(texels)[2 * i];
    float4 const b = reinterpret_cast<float4 const*>(texels)[2 * i + 1];
    grad[2 * i] = a.x; grad[2 * i + 1] = a.y;
    hess[3 * i] = a.z; hess[3 * i + 1] = a.w; hess[3 * i + 2] = b.x;
}

/* ------------------------------------------------------------------ */
/*
 * The same three steps as ONE kernel with the image tile staged by the TMA
 * engine (north star: "image pyramids staged to shared memory via TMA"). A
 * block owns a TW x TH output tile and needs it plus a halo of R = ks + 1
 * pixels (blur radius + the 3x3 stencil). One elected thread arms an mbarrier
 * with the byte count and issues one bulk asynchronous copy
 * (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes, SASS
 * UBLKCP) per tile row -- 16-byte aligned spans of the image rows, clipped to
 * the image; the block waits on the mbarrier. The reference clamps indices at
 * the image border (edge replication, mve::image::blur_gaussian): blocks on
 * the border fill the cells outside the image from the edge pixels before
 * use. Then blur along x, blur along y (both with the CPU's operation order)
 * and the 6x9 stencil run out of shared memory: the two float images the
 * three-kernel version writes and reads back (16 B per pixel of DRAM traffic)
 * never exist. Needs a row pitch that is a multiple of 16 bytes; other widths
 * keep the three kernels.
 *
 * (A tiled tensor map -- cp.async.bulk.tensor.2d, which would also do the
 * clipping in hardware -- was tried first: the UTMALDG raised "illegal
 * instruction" on the GPU box although cuTensorMapEncodeTiled accepted the
 * descriptor; with no way to debug the descriptor offline, the row-wise bulk
 * copies are what ships.)
 */
constexpr int FT_W = 64, FT_H = 32, FT_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(FT_THREADS)
set_scale_tma_kernel (T const* __restrict__ img, int w, int h, int R,
    int box_w, BlurKernel const k, int mode, float* __restrict__ out,
    float* __restrict__ blur_out)
{
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long bar;
    constexpr int A = 16 / static_cast<int>(sizeof(T));   /* pixels per 16 B */
    int const rows_in = FT_H + 2 * R;
    size_t const in_bytes = (static_cast<size_t>(box_w) * rows_in * sizeof(T)
        + 127) / 128 * 128;
    T* s_in = reinterpret_cast<T*>(smem);
    float* s_bx = reinterpret_cast<float*>(smem + in_bytes);
    int const bw = FT_W + 2;                     /* blurred columns kept */
    float* s_by = s_bx + static_cast<size_t>(rows_in) * bw;

    int const tid = threadIdx.x;
    int const x0 = blockIdx.x * FT_W, y0 = blockIdx.y * FT_H;
    /* aligned column span [xs, xe) and row span [ys, ye) inside the image */
    int const xs = max(0, (x0 - R) & ~(A - 1) );
    int const xe = min(w, (x0 + FT_W + R + A - 1) & ~(A - 1));
    int const ys = max(0, y0 - R), ye = min(h, y0 + FT_H + R);
    int const col0 = (x0 - R) - xs;              /* tile column of x0 - R */
    unsigned const bar_addr = static_cast<unsigned>(
        __cvta_generic_to_shared(&bar));
    if (tid == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;"
            :: "r"(bar_addr));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        unsigned const row_bytes = static_cast<unsigned>((xe - xs)
            * sizeof(T));
        unsigned const bytes = row_bytes * static_cast<unsigned>(ye - ys);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
            :: "r"(bar_addr), "r"(bytes) : "memory");
        for (int gy = ys; gy < ye; ++gy)
        {
            unsigned const dst = static_cast<unsigned>(
                __cvta_generic_to_shared(s_in + static_cast<size_t>(
                gy - (y0 - R)) * box_w));
            T const* src = img + static_cast<size_t>(gy) * w + xs;
            asm volatile("cp.async.bulk.shared::cluster.global"
                ".mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                :: "r"(dst), "l"(src), "r"(row_bytes), "r"(bar_addr)
                : "memory");
        }
    }
    {
        unsigned done = 0;
        while (!done)
            asm volatile("{\n.reg .pred p;\n"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n"
                "selp.u32 %0, 1, 0, p;\n}"
                : "=r"(done) : "r"(bar_addr) : "memory");
    }

    /* edge replication where the tile leaves the image: tile cell (r, c)
     * holds image pixel (y0 - R + r, xs + c) */
    int const cols = col0 + FT_W + 2 * R;        /* cells the blur can touch */
    if (x0 - R < 0 || y0 - R < 0 || x0 + FT_W + R > w || y0 + FT_H + R > h)
    {
        for (int i = tid; i < cols * rows_in; i += FT_THREADS)
        {
            int const r = i / cols, c = i % cols;
            int const gx = xs + c, gy = y0 - R + r;
            /* with xs clipped to 0 the columns left of the image are the
             * NEGATIVE tile columns: they are folded onto column 0 by the
             * clamped reads below; here only cells at or right of xs */
            if (gx >= w || gy < 0 || gy >= h)
            {
                int const sx = min(gx, w - 1) - xs;
                int const sy = min(max(gy, 0), h - 1) - (y0 - R);
                s_in[r * box_w + c] = s_in[sy * box_w + sx];
            }
        }
        __syncthreads();
    }

    /* blur along x: rows of the tile with halo, columns x0 - 1 .. x0 + TW.
     * Tile column of image column gx is gx - xs; left of the image (only
     * when xs = 0) the index is clamped to 0 = edge replication. */
    for (int i = tid; i < rows_in * bw; i += FT_THREADS)
    {
        int const r = i / bw, c = i % bw;
        T const* row = s_in + r * box_w;
        int const centre = col0 + (c - 1 + R);   /* may be < R near x = 0 */
        float acc = 0.0f;
        for (int j = -k.ks; j <= k.ks; ++j)
            acc = __fadd_rn(acc, __fmul_rn(pixel_value(row[max(centre + j,
                0)]), k.w[abs(j)]));
        s_bx[i] = __fdiv_rn(acc, k.wsum);
    }
    __syncthreads();
    /* blur along y: rows y0 - 1 .. y0 + TH */
    for (int i = tid; i < (FT_H + 2) * bw; i += FT_THREADS)
    {
        int const r = i / bw, c = i % bw;
        float const* col = s_bx + (r - 1 + R) * bw + c;
        float acc = 0.0f;
        for (int j = -k.ks; j <= k.ks; ++j)
            acc = __fadd_rn(acc, __fmul_rn(col[j * bw], k.w[abs(j)]));
        s_by[i] = __fdiv_rn(acc, k.wsum);
    }
    __syncthreads();

    /* compute_gradients_and_hessian on the blurred tile */
    for (int i = tid; i < FT_W * FT_H; i += FT_THREADS)
    {
        int const ly = i / FT_W, lx = i % FT_W;
        int const x = x0 + lx, y = y0 + ly;
        if (x >= w || y >= h)
            continue;
        size_t const pix = static_cast<size_t>(y) * w + x;
        if (blur_out != nullptr)
            blur_out[pix] = s_by[(ly + 1) * bw + lx + 1];
        store_grad_hess([&](int a, int b) {
                return s_by[(ly + 1 + b) * bw + (lx + 1 + a)]; },
            x >= 1 && x < w - 1 && y >= 1 && y < h - 1, mode, out, pix);
    }
}

/* Launches the fused kernel if the image qualifies; false = use the three
 * kernels (pitch not a multiple of 16 bytes, misaligned image, or a blur
 * radius too large for shared memory). */
template <typename T>
bool
try_set_scale_tma (smvsb_ctx* c, T const* img_dev, int w, int h,
    BlurKernel const& k, int mode, float* out_dev, float* blur_out)
{
    if ((static_cast<size_t>(w) * sizeof(T)) % 16 != 0
        || reinterpret_cast<uintptr_t>(img_dev) % 16 != 0)
        return false;
    int const R = k.ks + 1;
    int const per16 = 16 / static_cast<int>(sizeof(T));
    /* the aligned span can start up to per16 - 1 pixels left of x0 - R and
     * end as many to the right */
    int const box_w = (FT_W + 2 * R + 2 * (per16 - 1) + per16 - 1) / per16
        * per16;
    int const rows_in = FT_H + 2 * R;
    size_t const in_bytes = (static_cast<size_t>(box_w) * rows_in * sizeof(T)
        + 127) / 128 * 128;
    size_t const smem = in_bytes + (static_cast<size_t>(rows_in)
        + FT_H + 2) * (FT_W + 2) * sizeof(float);
    if (smem > 200 * 1024)
        return false;
    CUDA_CHECK(cudaFuncSetAttribute(set_scale_tma_kernel<T>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    dim3 const grid((w + FT_W - 1) / FT_W, (h + FT_H - 1) / FT_H);
    set_scale_tma_kernel<T><<<grid, FT_THREADS, smem, c->stream>>>(img_dev, w,
        h, R, box_w, k, mode, out_dev, blur_out);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
    return true;
}

} /* namespace */

/* sigma = 0.12 * 2^scale + 0.2 (lib/stereo_view.cc:28), narrowed to float
 * at the call of blur_gaussian<float>(img, float sigma). */
static BlurKernel
make_blur_kernel (int scale)
{
    double const sigma_d = 0.12 * std::pow(2.0, scale) + 0.2;
    float const sigma = static_cast<float>(sigma_d);
    BlurKernel k;
    k.ks = static_cast<int>(std::ceil(sigma * 2.884f));
    if (k.ks > BLUR_MAX_KS)
        throw Error(SMVSB_ERR_INVALID, "blur radius too large for this scale");
    for (int i = 0; i <= k.ks; ++i)
    {
        float const x = static_cast<float>(i);
        k.w[i] = std::exp(-((x * x) / (2.0f * sigma * sigma)));
    }
    float wsum = 0.0f;
    for (int i = -k.ks; i <= k.ks; ++i)
        wsum += k.w[i < 0 ? -i : i];
    k.wsum = wsum;
    return k;
}

/* The three-kernel path's scratch: the x pass's output (one float per
 * channel and pixel) and the blurred gray image. Reserving it for the
 * largest image before a loop of device_set_scale calls keeps the buffers
 * from being reallocated between them. */
void
reserve_set_scale_scratch (smvsb_ctx* c, DevImage::Kind kind, size_t pixels)
{
    c->stage_a.reserve(pixels * (kind == DevImage::RGB_F32 ? 3 : 1));
    c->stage_b.reserve(pixels);
}

void
device_set_scale (smvsb_ctx* c, DevImage const& img, int scale, int mode,
    float* out_dev, float* blur_out)
{
    BlurKernel const k = make_blur_kernel(scale);
    int const w = img.w, h = img.h;
    if (img.kind == DevImage::U8 && try_set_scale_tma(c,
        static_cast<uint8_t const*>(img.p), w, h, k, mode, out_dev, blur_out))
        return;
    if (img.kind == DevImage::F32 && try_set_scale_tma(c,
        static_cast<float const*>(img.p), w, h, k, mode, out_dev, blur_out))
        return;
    reserve_set_scale_scratch(c, img.kind, static_cast<size_t>(w) * h);
    /* a single-channel image's blurred image is the gray image */
    bool const colour = img.kind == DevImage::RGB_F32;
    float* const gray = (!colour && blur_out != nullptr) ? blur_out
        : c->stage_b.p;
    dim3 const block(128, 1), grid((w + 127) / 128, h);
    if (img.kind == DevImage::U8)
        blur_x_kernel<uint8_t, 1><<<grid, block, 0, c->stream>>>(
            static_cast<uint8_t const*>(img.p), w, h, k, c->stage_a.p);
    else if (img.kind == DevImage::F32)
        blur_x_kernel<float, 1><<<grid, block, 0, c->stream>>>(
            static_cast<float const*>(img.p), w, h, k, c->stage_a.p);
    else
        blur_x_kernel<float, 3><<<grid, block, 0, c->stream>>>(
            static_cast<float const*>(img.p), w, h, k, c->stage_a.p);
    CUDA_CHECK(cudaGetLastError());
    if (colour)
        blur_y_kernel<3><<<grid, block, 0, c->stream>>>(c->stage_a.p, w, h, k,
            gray, blur_out);
    else
        blur_y_kernel<1><<<grid, block, 0, c->stream>>>(c->stage_a.p, w, h, k,
            gray, nullptr);
    CUDA_CHECK(cudaGetLastError());
    grad_hess_kernel<<<grid, block, 0, c->stream>>>(gray, w, h, mode,
        out_dev);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 3);
}

/* ------------------------------------------------------------------ */
/* DepthOptimizer::depthmap_bilateral_filter (lib/depth_optimizer.cc:957-1004):
 * joint bilateral filter of the SGM depth with the colour image as guide.  */

constexpr int BILAT_MAX_K = 8;          /* kernel_size (radius), default 5 */

struct BilateralArgs
{
    int w, h, channels, dm_w, dm_h, ks;
    float scale_x, scale_y;
    float two_sigma_sq;                 /* T(2) * 0.1f * 0.1f of math::gaussian */
    float spatial[(2 * BILAT_MAX_K + 1) * (2 * BILAT_MAX_K + 1)];
    unsigned long long exp_tab[32];     /* 2^(i/32) table of expf */
};

/* expf as glibc computes it (sysdeps/ieee754/flt-32/e_expf.c: N = 32 table,
 * cubic in double, one rounding to float), for x <= 0: the range weight must
 * be the bits the CPU produces. Checked against libm on 3e7 arguments in
 * (-87, 0] and on [-1000, 0] (tests/test_cpu_host.py runs the host twin of
 * this function). */
__host__ __device__ __forceinline__ float
expf_like_glibc (float x, unsigned long long const* tab)
{
    /* Below log(2^-150) glibc returns 0 (its underflow branch). The table
     * path must not run there: below about x = -708 the exponent that
     * ki << 47 adds to the table entry wraps past the smallest double
     * exponent, and s turns into +-inf or a huge value. In the bilateral
     * filter (argument -diff^2 / 0.02) two guide values more than 3.77 apart
     * in one window would get an infinite or NaN weight instead of 0. */
    if (x < -0x1.9fe368p6f)
        return 0.0f;
    double const n = 32.0;
    double const c0 = 0x1.c6af84b912394p-5 / n / n / n;
    double const c1 = 0x1.ebfce50fac4f3p-3 / n / n;
    double const c2 = 0x1.62e42ff0c52d6p-1 / n;
    double const inv_ln2_n = 0x1.71547652b82fep+0 * n;
    double const shift = 0x1.8p+52;
#ifdef __CUDA_ARCH__
    double z = __dmul_rn(inv_ln2_n, static_cast<double>(x));
    double kd = __dadd_rn(z, shift);
    unsigned long long const ki = static_cast<unsigned long long>(
        __double_as_longlong(kd));
    kd = __dadd_rn(kd, -shift);
    double const r = __dadd_rn(z, -kd);
    unsigned long long const t = tab[ki % 32] + (ki << 47);
    double const s = __longlong_as_double(static_cast<long long>(t));
    z = __dadd_rn(__dmul_rn(c0, r), c1);
    double const r2 = __dmul_rn(r, r);
    double y = __dadd_rn(__dmul_rn(c2, r), 1.0);
    y = __dadd_rn(__dmul_rn(z, r2), y);
    y = __dmul_rn(y, s);
    return static_cast<float>(y);
#else
    volatile double z = inv_ln2_n * static_cast<double>(x);
    volatile double kd = z + shift;
    unsigned long long ki;
    double const kd_copy = kd;
    memcpy(&ki, &kd_copy, 8);
    kd = kd - shift;
    volatile double r = z - kd;
    unsigned long long const t = tab[ki % 32] + (ki << 47);
    double s;
    memcpy(&s, &t, 8);
    volatile double zz = c0 * r;
    zz = zz + c1;
    volatile double r2 = r * r;
    volatile double y = c2 * r;
    y = y + 1.0;
    volatile double m = zz * r2;
    y = m + y;
    y = y * s;
    return static_cast<float>(y);
#endif
}

/* the table expf_like_glibc reads: 2^(i/32) with i << 47 taken out */
static void
fill_exp_table (unsigned long long* tab)
{
    for (int i = 0; i < 32; ++i)
    {
        double const v = std::exp2(static_cast<double>(i) / 32.0);
        unsigned long long bits;
        memcpy(&bits, &v, 8);
        tab[i] = bits - (static_cast<unsigned long long>(i) << 47);
    }
}

__global__ void __launch_bounds__(128)
bilateral_kernel (BilateralArgs const a, float const* __restrict__ ci,
    float const* __restrict__ dm, float* __restrict__ out)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y;
    if (x >= a.w)
        return;
    int const C = a.channels;
    float centre[4];
    for (int c = 0; c < C; ++c)
        centre[c] = ci[(static_cast<size_t>(y) * a.w + x) * C + c];
    float acc_v = 0.0f, acc_w = 0.0f;
    int const side = 2 * a.ks + 1;
    for (int ky = -a.ks; ky <= a.ks; ++ky)
        for (int kx = -a.ks; kx <= a.ks; ++kx)
        {
            int const cx = min(max(x + kx, 0), a.w - 1);
            int const cy = min(max(y + ky, 0), a.h - 1);
            /* math::clamp(scale * c, 0.f, dm_size - 1.f), then truncation */
            float fx = __fmul_rn(a.scale_x, static_cast<float>(cx));
            float fy = __fmul_rn(a.scale_y, static_cast<float>(cy));
            float const mx = static_cast<float>(a.dm_w) - 1.0f;
            float const my = static_cast<float>(a.dm_h) - 1.0f;
            fx = (fx < 0.0f) ? 0.0f : ((fx > mx) ? mx : fx);
            fy = (fy < 0.0f) ? 0.0f : ((fy > my) ? my : fy);
            int const dx = static_cast<int>(fx), dy = static_cast<int>(fy);
            float const d = dm[static_cast<size_t>(dy) * a.dm_w + dx];
            if (d == 0.0f)
                continue;
            float weight = 1.0f;
            weight = __fmul_rn(weight,
                a.spatial[(ky + a.ks) * side + (kx + a.ks)]);
            for (int c = 0; c < C; ++c)
            {
                float const diff = __fadd_rn(
                    ci[(static_cast<size_t>(cy) * a.w + cx) * C + c],
                    -centre[c]);
                float const arg = -__fdiv_rn(__fmul_rn(diff, diff),
                    a.two_sigma_sq);
                weight = __fmul_rn(weight, expf_like_glibc(arg, a.exp_tab));
            }
            acc_v = __fadd_rn(acc_v, __fmul_rn(d, weight));
            acc_w = __fadd_rn(acc_w, weight);
        }
    out[static_cast<size_t>(y) * a.w + x] =
        (acc_w > 0.0f) ? __fdiv_rn(acc_v, acc_w) : 0.0f;
}

/* initialize_linear without gamma (lib/stereo_view.cc:64-84): shading image =
 * byte_to_float(image), plus its gradient. */
void
device_shading_inputs (smvsb_ctx* c, uint8_t const* img_dev, int w, int h,
    float* shading_dev, float* shading_grad_dev)
{
    int const n = w * h;
    byte_to_float_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(img_dev, n,
        shading_dev);
    CUDA_CHECK(cudaGetLastError());
    dim3 const block(128, 1), grid((w + 127) / 128, h);
    grad_hess_kernel<<<grid, block, 0, c->stream>>>(shading_dev, w, h, 0,
        shading_grad_dev);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 2);
}

/* mve::image::byte_to_float_image of a single-channel image */
void
device_byte_to_float (smvsb_ctx* c, uint8_t const* img_dev, size_t n,
    float* out_dev)
{
    byte_to_float_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0,
        c->stream>>>(img_dev, static_cast<int>(n), out_dev);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
}

void
device_unpack_texels (smvsb_ctx* c, float const* texels, int n, float* grad,
    float* hess)
{
    unpack_texels_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(texels, n,
        grad, hess);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
}

/* w*h*channels guide image and dm_w*dm_h depth on the device -> w*h depth. */
void
device_bilateral_filter (smvsb_ctx* c, float const* ci_dev, int w, int h,
    int channels, float const* dm_dev, int dm_w, int dm_h, float sigma,
    int kernel_size, float* out_dev)
{
    if (kernel_size < 0 || kernel_size > BILAT_MAX_K)
        throw Error(SMVSB_ERR_INVALID, "bilateral kernel_size out of range");
    if (channels < 1 || channels > 4)
        throw Error(SMVSB_ERR_INVALID, "guide image needs 1..4 channels");
    BilateralArgs a;
    a.w = w; a.h = h; a.channels = channels; a.dm_w = dm_w; a.dm_h = dm_h;
    a.ks = kernel_size;
    a.scale_x = static_cast<float>(dm_w) / static_cast<float>(w);
    a.scale_y = static_cast<float>(dm_h) / static_cast<float>(h);
    float const range_sigma = 0.1f;     /* lib/depth_optimizer.cc:996 */
    a.two_sigma_sq = 2.0f * range_sigma * range_sigma;
    int const side = 2 * kernel_size + 1;
    for (int ky = -kernel_size; ky <= kernel_size; ++ky)
        for (int kx = -kernel_size; kx <= kernel_size; ++kx)
        {
            /* math::gaussian_2d((float)kx, (float)ky, sigma, sigma) */
            float const fx = static_cast<float>(kx), fy = static_cast<float>(ky);
            float const ex = -(fx * fx) / (2.0f * sigma * sigma)
                - (fy * fy) / (2.0f * sigma * sigma);
            a.spatial[(ky + kernel_size) * side + (kx + kernel_size)]
                = std::exp(ex);
        }
    fill_exp_table(a.exp_tab);
    dim3 const block(128, 1), grid((w + 127) / 128, h);
    bilateral_kernel<<<grid, block, 0, c->stream>>>(a, ci_dev, dm_dev,
        out_dev);
    CUDA_CHECK(cudaGetLastError());
    count_launches(c, 1);
}

/* Host twin of the device expf (tests pin it to libm). */
float
host_expf_like_glibc (float x)
{
    unsigned long long tab[32];
    fill_exp_table(tab);
    return expf_like_glibc(x, tab);
}

} /* namespace smvsb */
