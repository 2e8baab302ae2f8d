/*
 * sgm.cu -- SGMStereo::run_sgm on the GPU (reference: lib/sgm_stereo.cc).
 *
 *   K6  create_cost_volume (:192-244): u8_to_float_kernel (float copy of the
 *       neighbour image), sgm_warp_volume_kernel (plane sweep of the
 *       neighbour luminance at num_steps inverse-depth planes,
 *       warped_neighbors_for_depth :150-190: fp32, byte bilinear with +0.5
 *       rounding, into a uint8 volume), sgm_cost_bits_kernel (9x7 census
 *       :126-148 of the main image and of every warped slice, Hamming
 *       distance; 255 where the warped pixel is 0). The census words never
 *       leave the SM (the reference's uint64 census volume is 2.1 GB at
 *       2 MP x 128).
 *   K7  aggregate_sgm_costs (:429-667), SSE branch (constant P2, uint16
 *       arithmetic): sgm_paths_kernel<L>, L = D / 8 lanes per scan line.
 *       All 8 directions in one launch, warps on scan lines, disparities
 *       across the lanes, L_r carried in registers, min over disparities by
 *       warp shuffles. Diagonals wrap around at the image
 *       border, where the reference restarts the path (:515-534). Each
 *       direction writes L_r - C (a byte) to its own volume.
 *   K8  S = 8 C + sum_r (L_r - C) (+ the reference's corner extras) and
 *       depth_from_sgm_volume (:274-306) in one pass: sgm_sum_wta_kernel<G>,
 *       G = D / 16 lanes per pixel; S is only materialised when the caller
 *       asks for the volume.
 *
 * When the volumes of a run do not fit the device budget (smvsb_sgm_ex), the
 * same kernels run on bands of image rows in two sweeps with the paths' state
 * carried across bands (run_banded); the depth is the same, bitwise.
 *
 * Layouts: cost C[pixel][disp] uint8, sum S[pixel][disp] uint16 (pixel-major,
 * disparity contiguous, like the reference's sse_*_volume), so a warp's
 * access to one pixel is one coalesced 128 B / 256 B segment.
 */
#include <algorithm>
#include <mutex>

#include <cuda_fp16.h>

#include "common.cuh"

namespace smvsb {

namespace {

struct SgmParams
{
    int w, h, nw, nh, D;
    float M[9];
    float t[3];
};

/*
 * Cost volume, in three launches: the neighbour image as floats, the warped
 * volume (sgm_warp_volume_kernel), then census + Hamming distance
 * (sgm_cost_bits_kernel), four depth planes per iteration.
 *  - The warp restates the reference's fp32 steps with explicit
 *    round-to-nearest ops, so it is bit-identical to the CPU; M * (x, y, 1)
 *    does not depend on the plane and is kept in registers. Integer <-> float
 *    conversions run on the quarter-rate XU pipe: the neighbour image is read
 *    from a float copy, floor() is taken with the 1.5 * 2^23 trick.
 * Semantics restated from census_filter / create_cost_volume
 * (lib/sgm_stereo.cc:126-148, 192-244): census only for pixels with
 * 4 <= x < w-5, 3 <= y < h-4 and a non-zero centre; cost 255 where the
 * warped pixel is 0.
 */
constexpr int PLANES = 4;                        /* planes per iteration */

/* floor of 0 <= x < 2^22 as a float and as an int, without F2I / I2F */
__device__ __forceinline__ void
floor_pos (float x, float& fl, int& n)
{
    float const magic = 12582912.0f;              /* 1.5 * 2^23 */
    float const t = __fadd_rn(x, magic);          /* nearest integer */
    fl = __fsub_rn(t, magic);
    n = __float_as_int(t) - 0x4B400000;
    if (fl > x)
    {
        fl = __fsub_rn(fl, 1.0f);
        n -= 1;
    }
}

/* warped_neighbors_for_depth (lib/sgm_stereo.cc:150-190) for one pixel and
 * plane: the neighbour's luminance as the byte value the reference stores
 * (0 = no sample). neigh: float copy of the byte image. */
__device__ __forceinline__ unsigned
warp_from_tp (SgmParams const& p, float const* __restrict__ neigh,
    float const* tp, float depth, float nw1, float nh1)
{
    float q0 = __fadd_rn(__fmul_rn(tp[0], depth), p.t[0]);
    float q1 = __fadd_rn(__fmul_rn(tp[1], depth), p.t[1]);
    float const q2 = __fadd_rn(__fmul_rn(tp[2], depth), p.t[2]);
    if (q2 < 0)
        return 0u;
    q0 = __fsub_rn(__fdiv_rn(q0, q2), 0.5f);
    q1 = __fsub_rn(__fdiv_rn(q1, q2), 0.5f);
    /* written so that NaN coordinates pass like in the reference's test
     * (all comparisons false) and are then clamped by fmaxf / fminf */
    if (q0 < 0 || q1 < 0 || q0 > nw1 || q1 > nh1)
        return 0u;
    /* mve::Image<uint8_t>::linear_at */
    float const xx = fmaxf(0.0f, fminf(nw1, q0));
    float const yy = fmaxf(0.0f, fminf(nh1, q1));
    float fxf, fyf;
    int fx, fy;
    floor_pos(xx, fxf, fx);
    floor_pos(yy, fyf, fy);
    int const fx1 = min(fx + 1, p.nw - 1), fy1 = min(fy + 1, p.nh - 1);
    float const w1 = __fsub_rn(xx, fxf);
    float const w0 = __fsub_rn(1.0f, w1);
    float const w3 = __fsub_rn(yy, fyf);
    float const w2 = __fsub_rn(1.0f, w3);
    float const v00 = __ldg(neigh + fy * p.nw + fx);
    float const v10 = __ldg(neigh + fy * p.nw + fx1);
    float const v01 = __ldg(neigh + fy1 * p.nw + fx);
    float const v11 = __ldg(neigh + fy1 * p.nw + fx1);
    float s = __fmul_rn(v00, __fmul_rn(w0, w2));
    s = __fadd_rn(s, __fmul_rn(v10, __fmul_rn(w1, w2)));
    s = __fadd_rn(s, __fmul_rn(v01, __fmul_rn(w0, w3)));
    s = __fadd_rn(s, __fmul_rn(v11, __fmul_rn(w1, w3)));
    s = __fadd_rn(s, 0.5f);
    /* static_cast<uint8_t>(s): truncation, 0 <= s < 256. One conversion
     * instruction on the otherwise idle XU pipe instead of six on the
     * ALU / FMA pipes the kernel is bound by */
    return __float2uint_rz(s);
}

__device__ __forceinline__ __half2
as_half2 (unsigned v)
{
    return *reinterpret_cast<__half2*>(&v);
}

__device__ __forceinline__ unsigned
as_word (__half2 v)
{
    return *reinterpret_cast<unsigned*>(&v);
}

__global__ void
u8_to_float_kernel (size_t n, uint8_t const* __restrict__ in,
    float* __restrict__ out)
{
    size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x
        + threadIdx.x;
    if (i < n)
        out[i] = static_cast<float>(in[i]);
}

/*
 * Warped neighbour volume: W[plane][row][col] = the byte
 * warped_neighbors_for_depth (:150-190) gives main pixel
 * (col - 4, row0 + row - 3) at that plane, 0 outside the image (row0 > 0: a
 * band of rows, see run_banded) -- a margin of the census window's halo
 * (4 columns, 3 rows, rounded up to the cost kernel's tiles) is part of the
 * volume, so the cost kernel loads its tiles without bounds tests. One thread
 * warps four neighbouring pixels through all planes (M * (x, y, 1) stays in
 * registers) and stores one word per plane; every voxel is warped ONCE
 * (warping inside the cost kernel would repeat it wherever the tiles' halos
 * overlap, 1.7 times per voxel).
 */
constexpr int WV_BX = 32, WV_BY = 4;

__global__ void __launch_bounds__(WV_BX * WV_BY)
sgm_warp_volume_kernel (SgmParams const p, float const* __restrict__ neigh,
    float const* __restrict__ depths, uint8_t* __restrict__ Wv, int pitch,
    int rows, int row0)
{
    __shared__ float s_depths[256];
    int const tid = threadIdx.y * WV_BX + threadIdx.x;
    for (int i = tid; i < p.D; i += WV_BX * WV_BY)
        s_depths[i] = depths[i];
    __syncthreads();
    int const col = (blockIdx.x * WV_BX + threadIdx.x) * 4;   /* padded */
    int const row = blockIdx.y * WV_BY + threadIdx.y;
    if (col >= pitch || row >= rows)
        return;
    int const gy = row0 + row - 3;
    float const nw1 = static_cast<float>(p.nw - 1);
    float const nh1 = static_cast<float>(p.nh - 1);
    float tp[4][3];
    bool in_img[4];
    bool any = false;
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
        int const gx = col - 4 + k;
        in_img[k] = (gx >= 0 && gx < p.w && gy >= 0 && gy < p.h);
        any = any || in_img[k];
        float const fx = 0.5f + static_cast<float>(gx);
        float const fy = 0.5f + static_cast<float>(gy);
#pragma unroll
        for (int r = 0; r < 3; ++r)
        {
            float s = __fmul_rn(p.M[3 * r], fx);
            s = __fadd_rn(s, __fmul_rn(p.M[3 * r + 1], fy));
            tp[k][r] = __fadd_rn(s, p.M[3 * r + 2]);      /* * 1.f */
        }
    }
    size_t const plane_stride = static_cast<size_t>(pitch) * rows;
    unsigned* dst = reinterpret_cast<unsigned*>(Wv
        + static_cast<size_t>(row) * pitch + col);
    if (!any)
    {
        for (int d = 0; d < p.D; ++d)
            dst[d * (plane_stride / 4)] = 0u;
        return;
    }
#pragma unroll 2
    for (int d = 0; d < p.D; ++d)
    {
        float const depth = s_depths[d];
        unsigned word = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
            unsigned v = 0;
            if (in_img[k])
                v = warp_from_tp(p, neigh, tp[k], depth, nw1, nh1);
            word |= v << (8 * k);
        }
        dst[d * (plane_stride / 4)] = word;
    }
}

/*
 * Census + Hamming distance from the warped volume. Pixels enter the fp16
 * comparisons as 1024 + byte (0x6400 | byte: one PRMT turns two bytes into a
 * half2; the order of the values is the bytes'). A thread owns four
 * neighbouring pixels (two half2 pairs); per offset and plane a pair costs
 * one HSET2 (1.0 where centre < neighbour) and one HFMA2 that adds
 * 2^e to the accumulator of the window row: an accumulator starts at 1024.0
 * and the nine offsets of a row add distinct powers of two below 512, so its
 * fp16 bit pattern is 0x6400 | (the row's nine comparison bits) -- exact, no
 * conversion. The main image's bits are built the same way once per block
 * and stay in fourteen REGISTERS; distance = popcount of the XOR (two rows
 * per POPC after a byte permute).
 * Why bits: a signed-sum formulation reads 63 sign words per pair and
 * iteration from shared memory and is bound by the shared-memory queue.
 * The per-offset work is split between the ALU pipe (HSET2) and the FMA
 * pipe (HFMA2), and the odd-offset windows come from a second copy of the
 * tile shifted by one pixel (an LDS instead of a funnel shift). Tiles are
 * 64 x 16 pixels (halo redundancy 1.55; 1.72 at 32 x 16), loaded as
 * aligned words one iteration ahead into the other half of a double buffer.
 */
constexpr int C2_W = 64, C2_H = 16;
constexpr int C2_THREADS = (C2_W / 4) * C2_H;            /* 256 */
constexpr int C2_HALO_W = C2_W + 8, C2_HALO_H = C2_H + 6;  /* 72 x 22 */
constexpr int C2_ROW_WORDS = C2_HALO_W / 2;              /* 36 half2 words */
constexpr int C2_LOAD_WORDS = PLANES * C2_HALO_H * (C2_HALO_W / 4);  /* 1584 */
constexpr int C2_LOADS = (C2_LOAD_WORDS + C2_THREADS - 1) / C2_THREADS; /* 7 */

/* one window row: ev[0..5] = elements (0,1) .. (10,11) of the row counted from
 * the thread's first pixel's column - 4, od[0..4] = (1,2) .. (9,10) */
#define SMVSB_ROW_BITS(A0, A1, ev, od, acc0, acc1)                          \
    do {                                                                    \
        _Pragma("unroll")                                                   \
        for (int e_ = 0; e_ < 9; ++e_)                                      \
        {                                                                   \
            __half2 const wgt_ = __float2half2_rn(static_cast<float>(       \
                1 << e_));                                                  \
            unsigned const n0_ = (e_ & 1) ? (od)[e_ >> 1] : (ev)[e_ >> 1];  \
            unsigned const n1_ = (e_ & 1) ? (od)[(e_ >> 1) + 1]             \
                : (ev)[(e_ >> 1) + 1];                                      \
            acc0 = __hfma2(__hlt2(A0, as_half2(n0_)), wgt_, acc0);          \
            acc1 = __hfma2(__hlt2(A1, as_half2(n1_)), wgt_, acc1);          \
        }                                                                   \
    } while (0)

__global__ void __launch_bounds__(C2_THREADS, 2)
sgm_cost_bits_kernel (SgmParams const p, uint8_t const* __restrict__ main_img,
    uint8_t const* __restrict__ Wv, int pitch, int rows, int row0,
    uint8_t* __restrict__ cost)
{
    /* [buffer][0 = pairs at even, 1 = at odd columns][plane][row][word],
     * 50 KB: dynamic */
    extern __shared__ __align__(16) unsigned s_bits_dyn[];
    unsigned (*s_tile)[2][PLANES][C2_HALO_H][C2_ROW_WORDS] =
        reinterpret_cast<unsigned (*)[2][PLANES][C2_HALO_H][C2_ROW_WORDS]>(
            s_bits_dyn);

    int const tid = threadIdx.x;
    int const tx = tid % (C2_W / 4), ty = tid / (C2_W / 4);
    int const x0 = blockIdx.x * C2_W, y0 = blockIdx.y * C2_H;
    int const px = x0 + 4 * tx, py = y0 + ty;      /* first of four pixels */
    /* y0, py: rows of the volume and of `cost`, which start at image row
     * row0; gpy: the image row */
    int const gpy = row0 + py;

    /* main image tile (0x6400 | byte, like the warped tiles), both copies */
    {
        unsigned short* t0 = reinterpret_cast<unsigned short*>(
            &s_tile[0][0][0][0][0]);
        unsigned short* t1 = reinterpret_cast<unsigned short*>(
            &s_tile[0][1][0][0][0]);
        for (int i = tid; i < C2_HALO_W * C2_HALO_H; i += C2_THREADS)
        {
            int const c = i % C2_HALO_W, r = i / C2_HALO_W;
            int const gx = x0 - 4 + c, gy = row0 + y0 - 3 + r;
            bool const in = (gx >= 0 && gx < p.w && gy >= 0 && gy < p.h);
            unsigned short const v = static_cast<unsigned short>(0x6400u
                | (in ? main_img[gy * p.w + gx] : 0));
            t0[i] = v;
            if (c > 0)
                t1[i - 1] = v;
        }
    }
    __syncthreads();
    bool in_px[4], int_px[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        in_px[i] = (px + i < p.w && gpy < p.h);
        int_px[i] = in_px[i] && px + i >= 4 && px + i < p.w - 5 && gpy >= 3
            && gpy < p.h - 4;
    }
    __half2 const bias = as_half2(0x64006400u);          /* 1024.0 */
    /* census bits of the main pixels per window row (with the 0x6400 bias);
     * pixels without a census (border, zero centre) have all bits 0
     * (lib/sgm_stereo.cc:131-147) */
    unsigned mb0[7], mb1[7];
    {
        __half2 const A0 = as_half2(s_tile[0][0][0][ty + 3][2 * tx + 2]);
        __half2 const A1 = as_half2(s_tile[0][0][0][ty + 3][2 * tx + 3]);
        unsigned const a0 = as_word(A0), a1 = as_word(A1);
        unsigned const keep0 =
            ((int_px[0] && (a0 & 0xffffu) != 0x6400u) ? 0x01ffu : 0u)
            | ((int_px[1] && (a0 >> 16) != 0x6400u) ? 0x01ff0000u : 0u);
        unsigned const keep1 =
            ((int_px[2] && (a1 & 0xffffu) != 0x6400u) ? 0x01ffu : 0u)
            | ((int_px[3] && (a1 >> 16) != 0x6400u) ? 0x01ff0000u : 0u);
#pragma unroll
        for (int j = 0; j < 7; ++j)
        {
            unsigned ev[6], od[6];
#pragma unroll
            for (int q = 0; q < 6; ++q)
            {
                ev[q] = s_tile[0][0][0][ty + j][2 * tx + q];
                od[q] = s_tile[0][1][0][ty + j][2 * tx + q];
            }
            __half2 m0 = bias, m1 = bias;
            SMVSB_ROW_BITS(A0, A1, ev, od, m0, m1);
            mb0[j] = (as_word(m0) & keep0) | 0x64006400u;
            mb1[j] = (as_word(m1) & keep1) | 0x64006400u;
        }
    }
    __syncthreads();

    size_t const plane_stride = static_cast<size_t>(pitch) * rows;
    constexpr int RW = C2_HALO_W / 4;                        /* 18 words */
    /* a tile word and the word after it (the shifted copy needs its first
     * byte; the volume's margin keeps the read inside the row) */
    auto fetch = [&] (int d0, unsigned* nb, unsigned* nx)
    {
#pragma unroll
        for (int k = 0; k < C2_LOADS; ++k)
        {
            int const i = tid + k * C2_THREADS;
            nb[k] = 0u; nx[k] = 0u;
            if (i < C2_LOAD_WORDS)
            {
                int const pl = i / (C2_HALO_H * RW);
                int const rem = i % (C2_HALO_H * RW);
                int const r = rem / RW, q = rem % RW;
                unsigned const* src = reinterpret_cast<unsigned const*>(Wv
                    + (d0 + pl) * plane_stride
                    + static_cast<size_t>(y0 + r) * pitch + x0) + q;
                nb[k] = __ldg(src);
                nx[k] = __ldg(src + 1);
            }
        }
    };
    auto stash = [&] (int buf, unsigned const* nb, unsigned const* nx)
    {
#pragma unroll
        for (int k = 0; k < C2_LOADS; ++k)
        {
            int const i = tid + k * C2_THREADS;
            if (i < C2_LOAD_WORDS)
            {
                int const pl = i / (C2_HALO_H * RW);
                int const rem = i % (C2_HALO_H * RW);
                int const r = rem / RW, q = rem % RW;
                unsigned const b = nb[k];
                *reinterpret_cast<uint2*>(&s_tile[buf][0][pl][r][2 * q])
                    = make_uint2(__byte_perm(b, 0x64646464u, 0x4140),
                        __byte_perm(b, 0x64646464u, 0x4342));
                *reinterpret_cast<uint2*>(&s_tile[buf][1][pl][r][2 * q])
                    = make_uint2(__byte_perm(b, 0x64646464u, 0x4241),
                        (__byte_perm(b, nx[k], 0x4443) & 0x00ff00ffu)
                            | 0x64006400u);
            }
        }
    };

    unsigned nb[C2_LOADS], nx[C2_LOADS];
    fetch(0, nb, nx);
    stash(0, nb, nx);
    __syncthreads();
    int cur = 0;
    for (int d0 = 0; d0 < p.D; d0 += PLANES)
    {
        bool const more = d0 + PLANES < p.D;
        if (more)
            fetch(d0 + PLANES, nb, nx);

        unsigned out[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int pl = 0; pl < PLANES; ++pl)
        {
            __half2 const A0 = as_half2(s_tile[cur][0][pl][ty + 3][2 * tx + 2]);
            __half2 const A1 = as_half2(s_tile[cur][0][pl][ty + 3][2 * tx + 3]);
            unsigned x0w[7], x1w[7];
#pragma unroll
            for (int j = 0; j < 7; ++j)
            {
                unsigned ev[6], od[6];
#pragma unroll
                for (int q = 0; q < 6; q += 2)
                {
                    uint2 const e2 = *reinterpret_cast<uint2 const*>(
                        &s_tile[cur][0][pl][ty + j][2 * tx + q]);
                    uint2 const o2 = *reinterpret_cast<uint2 const*>(
                        &s_tile[cur][1][pl][ty + j][2 * tx + q]);
                    ev[q] = e2.x; ev[q + 1] = e2.y;
                    od[q] = o2.x; od[q + 1] = o2.y;
                }
                __half2 b0 = bias, b1 = bias;
                SMVSB_ROW_BITS(A0, A1, ev, od, b0, b1);
                x0w[j] = as_word(b0) ^ mb0[j];
                x1w[j] = as_word(b1) ^ mb1[j];
            }
            /* Hamming distances: low halves = even pixel, high = odd */
            unsigned c[4];
            c[0] = __popc(__byte_perm(x0w[0], x0w[1], 0x5410))
                + __popc(__byte_perm(x0w[2], x0w[3], 0x5410))
                + __popc(__byte_perm(x0w[4], x0w[5], 0x5410))
                + __popc(x0w[6] & 0xffffu);
            c[1] = __popc(__byte_perm(x0w[0], x0w[1], 0x7632))
                + __popc(__byte_perm(x0w[2], x0w[3], 0x7632))
                + __popc(__byte_perm(x0w[4], x0w[5], 0x7632))
                + __popc(x0w[6] >> 16);
            c[2] = __popc(__byte_perm(x1w[0], x1w[1], 0x5410))
                + __popc(__byte_perm(x1w[2], x1w[3], 0x5410))
                + __popc(__byte_perm(x1w[4], x1w[5], 0x5410))
                + __popc(x1w[6] & 0xffffu);
            c[3] = __popc(__byte_perm(x1w[0], x1w[1], 0x7632))
                + __popc(__byte_perm(x1w[2], x1w[3], 0x7632))
                + __popc(__byte_perm(x1w[4], x1w[5], 0x7632))
                + __popc(x1w[6] >> 16);
            unsigned const a0 = as_word(A0), a1 = as_word(A1);
            bool const zero[4] = { (a0 & 0xffffu) == 0x6400u,
                (a0 >> 16) == 0x6400u, (a1 & 0xffffu) == 0x6400u,
                (a1 >> 16) == 0x6400u };
#pragma unroll
            for (int i = 0; i < 4; ++i)
            {
                /* border pixels have no census on either side: distance 0;
                 * warped pixel 0: no sample, 255 */
                unsigned v = int_px[i] ? c[i] : 0u;
                if (zero[i]) v = 255u;
                out[i] |= v << (8 * pl);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (in_px[i])
                *reinterpret_cast<unsigned*>(cost + (static_cast<size_t>(py)
                    * p.w + px + i) * p.D + d0) = out[i];
        if (more)
            stash(cur ^ 1, nb, nx);
        __syncthreads();
        cur ^= 1;
    }
}
#undef SMVSB_ROW_BITS

/* ------------------------------------------------------------------ */

enum PathKind
{
    PATH_L2R = 0, PATH_R2L, PATH_T2B, PATH_T2B_D1, PATH_T2B_D2,
    PATH_B2T, PATH_B2T_D1, PATH_B2T_D2
};

__host__ __device__ constexpr int
ilog2 (int n)
{
    return n > 1 ? 1 + ilog2(n / 2) : 0;
}

/*
 * All eight path directions in ONE launch: warp -> (direction, scan lines),
 * 2h + 6w scan lines in flight (13 680 at 1920x1080) instead of h or w per
 * sequential launch.
 * fill_path_cost_sse (:361-406):
 *   L(p,i) = C(p,i) + min(L(q,i), L(q,i-1)+P1, L(q,i+1)+P1, min_k L(q,k)+P2)
 *            - min_k L(q,k)            (all uint16, wrap-around)
 * and copy_cost_and_add_to_sgm (:408-426) where a path starts (L = C).
 * The directions cannot share one read-modify-write sum volume without
 * racing, so each writes its own byte volume of L - C, which lies in [0, P2]
 * (P2 <= 255): 1 B/voxel/direction. The sum / WTA kernel adds them up.
 *
 * L lanes own a scan line (D = 8 L) and a warp 32 / L lines; a lane owns
 * eight disparities (four registers of 16-bit pairs; the minima are DPX
 * instructions, and L_r <= C + P2 <= 510 never overflows a half, so packed
 * adds / subtracts are plain 32-bit ones). The kernel is bound by
 * instruction issue, and the per-step bookkeeping (position, pointers, the
 * shuffle tree of min_k, the loop) costs the same per warp whatever D is,
 * so every warp carries 256 voxels per step. A step moves both pointers by
 * a constant (plus or minus one image row where a diagonal wraps around),
 * and the next step's costs are fetched one step ahead. The lines of a warp
 * are neighbours of the same direction, so they take the same number of
 * steps; a diagonal restarts at different steps on each, hence no branch
 * around the shuffles: the recurrence is always evaluated and a restarting
 * line overrides it.
 *
 * BANDED: one band of image rows [band.y0, band.y0 + band.rows) of a
 * top-to-bottom sweep (band.sweep 0: L2R, R2L, T2B, T2B_D1, T2B_D2) or a
 * bottom-to-top one (band.sweep 1: B2T, B2T_D1, B2T_D2); `cost` and `Dvol`
 * hold the band's rows only. A vertical or diagonal line advances exactly one
 * image row per step (the diagonals' wrap-around included), so a band is a
 * range of its steps: the line's position after the steps of the bands before
 * follows from its start, and its lanes' Pa..Pd are saved to band.state at the
 * end of a band and reloaded at the start of the next.
 */
struct PathBand
{
    int y0, rows, sweep;
    uint4* state;      /* [vertical direction][column][lane]: Pa, Pb, Pc, Pd */
};

template <int L, bool BANDED>
__global__ void __launch_bounds__(128)
sgm_paths_kernel (int w, int h, unsigned P1, unsigned P2,
    uint8_t const* __restrict__ cost, uint8_t* __restrict__ Dvol,
    PathBand const band)
{
    constexpr int D = 8 * L;
    constexpr int LPW = 32 / L;                 /* lines per warp */
    int const grp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    int const sl = lane & (L - 1);              /* lane within the line */
    bool const up_sweep = BANDED && band.sweep != 0;
    int const rows = BANDED ? band.rows : h;    /* rows of cost and Dvol */
    int const n_horiz = up_sweep ? 0 : 2;       /* kinds of each group */
    int const n_vert = BANDED ? 3 : 6;
    int const first_vert = up_sweep ? PATH_B2T : PATH_T2B;
    int const hp = (rows + LPW - 1) / LPW, wp = (w + LPW - 1) / LPW;
    int kind, line, count;
    if (grp < n_horiz * hp)
    {
        kind = grp / hp;                        /* PATH_L2R, PATH_R2L */
        line = LPW * (grp % hp) + (lane >> ilog2(L));
        count = rows;
    }
    else
    {
        int const q = grp - n_horiz * hp;
        if (q >= n_vert * wp)
            return;
        kind = first_vert + q / wp;             /* PATH_T2B .. PATH_B2T_D2 */
        line = LPW * (q % wp) + (lane >> ilog2(L));
        count = w;
    }
    /* line count not a multiple of LPW: the leftover lines of the last warp
     * repeat its last real line (they take part in the shuffles) and store
     * nothing */
    bool const live = line < count;
    if (!live)
        line = count - 1;
    bool const horizontal = (kind < 2);
    int const steps = horizontal ? w : rows;
    size_t const nvox = static_cast<size_t>(w) * rows * D;
    uint8_t* __restrict__ Dr = Dvol + static_cast<size_t>(kind
        - (up_sweep ? PATH_B2T : 0)) * nvox;

    int x, y, dx, dy;
    switch (kind)
    {
    case PATH_L2R: x = 0; y = line; dx = 1; dy = 0; break;
    case PATH_R2L: x = w - 1; y = line; dx = -1; dy = 0; break;
    case PATH_T2B: x = line; y = 0; dx = 0; dy = 1; break;
    case PATH_T2B_D1: x = line; y = 0; dx = 1; dy = 1; break;
    case PATH_T2B_D2: x = line; y = 0; dx = -1; dy = 1; break;
    case PATH_B2T: x = line; y = rows - 1; dx = 0; dy = -1; break;
    case PATH_B2T_D1: x = line; y = rows - 1; dx = 1; dy = -1; break;
    default: x = line; y = rows - 1; dx = -1; dy = -1; break;   /* B2T_D2 */
    }
    int const restart_x = (dx > 0) ? 0 : w - 1;   /* diagonals only */
    bool const diagonal = (!horizontal && dx != 0);

    unsigned const P1x2 = P1 | (P1 << 16), P2x2 = P2 | (P2 << 16);
    unsigned const BIG = 0x7000u;          /* "no neighbour" sentinel */
    unsigned Pa = 0, Pb = 0, Pc = 0, Pd = 0;
    bool start = true;
    uint4* saved = nullptr;
    if (BANDED && !horizontal)
    {
        /* steps this line took in the sweep's earlier bands */
        int const done = (dy > 0) ? band.y0 : h - band.y0 - rows;
        x = ((line + dx * (done % w)) % w + w) % w;
        saved = band.state + (static_cast<size_t>(kind - PATH_T2B) * w
            + line) * L + sl;
        if (done > 0)
        {
            start = diagonal && x == restart_x;
            uint4 const v = *saved;
            Pa = v.x; Pb = v.y; Pc = v.z; Pd = v.w;
        }
    }
    long long const row_bytes = static_cast<long long>(w) * D;
    long long const step_bytes = dy * row_bytes + dx * D;
    uint8_t const* pc = cost + (static_cast<size_t>(y) * w + x) * D + sl * 8;
    uint8_t* pd = Dr + (static_cast<size_t>(y) * w + x) * D + sl * 8;
    uint2 c8 = *reinterpret_cast<uint2 const*>(pc);
    for (int s = 0; s < steps; ++s)
    {
        int xn = x + dx;
        long long adv = step_bytes;
        if (xn < 0) { xn = w - 1; adv += row_bytes; }
        if (xn >= w) { xn = 0; adv -= row_bytes; }
        uint2 c8n = make_uint2(0u, 0u);
        if (s + 1 < steps)
            c8n = *reinterpret_cast<uint2 const*>(pc + adv);

        unsigned const Ca = __byte_perm(c8.x, 0, 0x4140);
        unsigned const Cb = __byte_perm(c8.x, 0, 0x4342);
        unsigned const Cc = __byte_perm(c8.y, 0, 0x4140);
        unsigned const Cd = __byte_perm(c8.y, 0, 0x4342);

        unsigned const m2 = __vminu2(__vminu2(Pa, Pb), __vminu2(Pc, Pd));
        unsigned mn = min(m2 & 0xffffu, m2 >> 16);
#pragma unroll
        for (int off = L / 2; off > 0; off >>= 1)
            mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        unsigned below = __shfl_up_sync(0xffffffffu, Pd, 1) >> 16;
        unsigned above = __shfl_down_sync(0xffffffffu, Pa, 1) & 0xffffu;
        if (sl == 0) below = BIG;
        if (sl == L - 1) above = BIG;
        unsigned const lo_a = below | (Pa << 16);               /* -, L0 */
        unsigned const ab = __funnelshift_r(Pa, Pb, 16);         /* L1, L2 */
        unsigned const bc = __funnelshift_r(Pb, Pc, 16);         /* L3, L4 */
        unsigned const cd = __funnelshift_r(Pc, Pd, 16);         /* L5, L6 */
        unsigned const hi_d = (Pd >> 16) | (above << 16);        /* L7, - */
        unsigned const mn2 = mn * 0x10001u;
        unsigned const far2 = mn2 + P2x2;
        unsigned const ba = __vimin3_u16x2(Pa, far2,
            __viaddmin_u16x2(ab, P1x2, lo_a + P1x2));
        unsigned const bb = __vimin3_u16x2(Pb, far2,
            __viaddmin_u16x2(bc, P1x2, ab + P1x2));
        unsigned const bcv = __vimin3_u16x2(Pc, far2,
            __viaddmin_u16x2(cd, P1x2, bc + P1x2));
        unsigned const bd = __vimin3_u16x2(Pd, far2,
            __viaddmin_u16x2(hi_d, P1x2, cd + P1x2));
        /* L - C, in [0, P2] per half; zero where the path (re)starts */
        unsigned const Da = start ? 0u : ba - mn2;
        unsigned const Db = start ? 0u : bb - mn2;
        unsigned const Dc = start ? 0u : bcv - mn2;
        unsigned const Dd = start ? 0u : bd - mn2;
        Pa = Ca + Da; Pb = Cb + Db; Pc = Cc + Dc; Pd = Cd + Dd;
        if (live)
            *reinterpret_cast<uint2*>(pd) = make_uint2(
                __byte_perm(Da, Db, 0x6420), __byte_perm(Dc, Dd, 0x6420));
        c8 = c8n;
        x = xn; pc += adv; pd += adv;
        start = diagonal && (xn == restart_x);
    }
    if (BANDED && saved != nullptr && live)
        *saved = make_uint4(Pa, Pb, Pc, Pd);
}

/*
 * S(p,i) = sum over the 8 directions of L_r(p,i) = 8 C + sum_r (L_r - C),
 * plus C once more at the four image corners: column 0 of the d1 volume and
 * column w-1 of the d2 volume are (re)initialised for ALL y after row 0 /
 * row h-1 already were (:521-534, :600-613). Then depth_from_sgm_volume
 * (:274-306): first minimum over the planes.
 * G = D / 16 lanes per pixel: a lane owns 16 consecutive disparities and
 * reads them as ONE 16-byte word per volume (nine 128-bit loads per lane
 * instead of 144 byte loads; with byte loads the kernel spends its time in
 * the load/store unit, lg_throttle and mio_throttle stalls), adds them as
 * pairs of 16-bit fields (S <= 9 * 255 + 8 * 255: no carry between the
 * fields), and the argmin -- lowest value, then lowest index, like the
 * reference's first minimum -- runs over the lane's 16 values and then over
 * the pixel's G lanes.
 *
 * The same kernel serves the banded path (rows [y0, y0 + rows) of the image;
 * cost, Dvol, part_in and S_out hold those rows only): NV byte volumes,
 * optionally a uint16 partial sum `part_in` in S's layout, and WTA = false
 * writes the sum to S_out without the cost term or the winner. The current
 * path is NV = 8, no partial sum, WTA, y0 = 0, rows = h.
 */
__device__ __forceinline__ void
wta_add16 (uint4 const v, unsigned mult, unsigned (&even)[4], unsigned (&odd)[4])
{
    unsigned const x[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
        even[k] += (x[k] & 0x00ff00ffu) * mult;          /* bytes 0, 2 */
        odd[k] += ((x[k] >> 8) & 0x00ff00ffu) * mult;    /* bytes 1, 3 */
    }
}

template <int G, int NV, bool PART, bool WTA>
__global__ void __launch_bounds__(256)
sgm_sum_wta_kernel (int w, int h, int y0, int rows,
    uint8_t const* __restrict__ cost, uint8_t const* __restrict__ Dvol,
    uint16_t const* __restrict__ part_in, uint8_t const* __restrict__ main_img,
    float const* __restrict__ depths, uint16_t* __restrict__ S_out,
    float* __restrict__ out)
{
    constexpr int D = 16 * G;
    int const npix = w * rows;
    int const t = blockIdx.x * blockDim.x + threadIdx.x;
    int const p = t >> ilog2(G), sub = threadIdx.x & (G - 1);
    bool const on = p < npix;
    size_t const nvox = static_cast<size_t>(npix) * D;
    size_t const base = static_cast<size_t>(on ? p : 0) * D + sub * 16;
    int const px = p % w, py = y0 + p / w;
    unsigned const mult = 8u + (((px == 0 || px == w - 1)
        && (py == 0 || py == h - 1)) ? 1u : 0u);
    unsigned even[4] = { 0u, 0u, 0u, 0u }, odd[4] = { 0u, 0u, 0u, 0u };
    uint4 v[NV + 1];
    if (WTA)
        v[0] = __ldg(reinterpret_cast<uint4 const*>(cost + base));
#pragma unroll
    for (int r = 0; r < NV; ++r)
        v[r + 1] = __ldg(reinterpret_cast<uint4 const*>(Dvol + r * nvox + base));
    if (WTA)
        wta_add16(v[0], mult, even, odd);
#pragma unroll
    for (int r = 0; r < NV; ++r)
        wta_add16(v[r + 1], 1u, even, odd);
    if (PART)
    {
        /* S's layout: word j of the 32 bytes = disparities (2j, 2j + 1) */
        uint4 const* src = reinterpret_cast<uint4 const*>(part_in + base);
        uint4 const lo = __ldg(src), hi = __ldg(src + 1);
        unsigned const q[8] = { lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z,
            hi.w };
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
            even[k] += __byte_perm(q[2 * k], q[2 * k + 1], 0x5410);
            odd[k] += __byte_perm(q[2 * k], q[2 * k + 1], 0x7632);
        }
    }
    if (S_out != nullptr && on)
    {
        /* disparities 4k .. 4k+3 of word k: even = (d0, d2), odd = (d1, d3) */
        uint4 lo, hi;
        lo.x = __byte_perm(even[0], odd[0], 0x5410);
        lo.y = __byte_perm(even[0], odd[0], 0x7632);
        lo.z = __byte_perm(even[1], odd[1], 0x5410);
        lo.w = __byte_perm(even[1], odd[1], 0x7632);
        hi.x = __byte_perm(even[2], odd[2], 0x5410);
        hi.y = __byte_perm(even[2], odd[2], 0x7632);
        hi.z = __byte_perm(even[3], odd[3], 0x5410);
        hi.w = __byte_perm(even[3], odd[3], 0x7632);
        uint4* dst = reinterpret_cast<uint4*>(S_out + base);
        dst[0] = lo;
        dst[1] = hi;
    }
    if (!WTA)
        return;
    /* key = value << 16 | index; 0xffff is "no minimum found" (the reference
     * starts from numeric_limits<uint16_t>::max() and compares with <) */
    unsigned key = 0xffffffffu;
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
        unsigned const val[4] = { even[k] & 0xffffu, odd[k] & 0xffffu,
            even[k] >> 16, odd[k] >> 16 };
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (val[i] != 0xffffu)
                key = min(key, (val[i] << 16)
                    | static_cast<unsigned>(sub * 16 + k * 4 + i));
    }
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1)
        key = min(key, __shfl_xor_sync(0xffffffffu, key, off));
    if (sub == 0 && on)
    {
        int const idx = (key == 0xffffffffu) ? 0 : static_cast<int>(
            key & 0xffffu);
        int const gp = y0 * w + p;
        out[gp] = (idx < 2 || main_img[gp] < 25) ? 0.0f : depths[idx];
    }
}

__global__ void
u8_to_u16_kernel (size_t n, uint8_t const* __restrict__ in,
    uint16_t* __restrict__ out)
{
    size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x
        + threadIdx.x;
    if (i < n)
        out[i] = in[i];
}

/* K7 and K8 for D planes; mid is recorded between the two launches */
template <int D>
void
run_paths_wta (int w, int h, unsigned P1, unsigned P2, uint8_t const* cost,
    uint8_t* Dvol, uint8_t const* main_img, float const* depths,
    uint16_t* S_out, float* out, cudaEvent_t mid, cudaStream_t st)
{
    constexpr int L = D / 8, G = D / 16;        /* lanes per line / pixel */
    constexpr int LPW = 32 / L;                 /* lines per warp */
    int const warps = 2 * ((h + LPW - 1) / LPW) + 6 * ((w + LPW - 1) / LPW);
    sgm_paths_kernel<L, false><<<(warps * 32 + 127) / 128, 128, 0, st>>>(w,
        h, P1, P2, cost, Dvol, PathBand{});
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaEventRecord(mid, st));
    sgm_sum_wta_kernel<G, 8, false, true><<<(w * h * G + 255) / 256, 256, 0,
        st>>>(w, h, 0, h, cost, Dvol, nullptr, main_img, depths, S_out, out);
    CUDA_CHECK(cudaGetLastError());
}

/*
 * SGMStereo::reconstruct's consistency check (lib/sgm_stereo.cc:64-91): every
 * main-view depth is reprojected into the neighbour (Correspondence::update /
 * fill, lib/correspondence.cc:20-51, in double with the fp32 reprojection
 * widened, pixel coordinates WITHOUT the half-pixel offset) and dropped when
 * it lands inside the 3 % border, on a neighbour pixel without depth, or when
 * the two depths differ by more than 20 %. Arithmetic in the reference's
 * order, no contraction: decisions are the CPU's.
 */
struct ConsistencyParams
{
    int w, h, nw, nh, cut;
    double M[9], t[3];
};

__global__ void
sgm_consistency_kernel (ConsistencyParams const p,
    float* __restrict__ d_main, float const* __restrict__ d_neig)
{
    int const x = blockIdx.x * blockDim.x + threadIdx.x;
    int const y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= p.w || y >= p.h)
        return;
    size_t const i = static_cast<size_t>(y) * p.w + x;
    float const dm = d_main[i];
    if (dm == 0.0f)
        return;
    double const u = x, v = y, wd = dm;
    double const pp = __dadd_rn(__dadd_rn(__dmul_rn(p.M[0], u),
        __dmul_rn(p.M[1], v)), p.M[2]);
    double const qq = __dadd_rn(__dadd_rn(__dmul_rn(p.M[3], u),
        __dmul_rn(p.M[4], v)), p.M[5]);
    double const rr = __dadd_rn(__dadd_rn(__dmul_rn(p.M[6], u),
        __dmul_rn(p.M[7], v)), p.M[8]);
    double const a = __dadd_rn(__dmul_rn(wd, pp), p.t[0]);
    double const b = __dadd_rn(__dmul_rn(wd, qq), p.t[1]);
    double const d = __dadd_rn(__dmul_rn(wd, rr), p.t[2]);
    double const cx = __ddiv_rn(a, d), cy = __ddiv_rn(b, d);
    /* written as the negation of "inside" so that NaN coordinates (d == 0)
     * behave like the reference's comparisons: all false -> not rejected
     * here, then indexed with whatever (int)NaN is -- not reproduced: the
     * reference's behaviour is undefined there; such a pixel is dropped */
    if (!(cx == cx) || !(cy == cy))
    {
        d_main[i] = 0.0f;
        return;
    }
    if (cx < p.cut || cx >= p.nw - p.cut || cy < p.cut || cy >= p.nh - p.cut)
    {
        d_main[i] = 0.0f;
        return;
    }
    float const cdepth = static_cast<float>(d);
    float const ndepth = d_neig[static_cast<size_t>(static_cast<int>(cy))
        * p.nw + static_cast<int>(cx)];
    float const ratio = __fdiv_rn(fminf(cdepth, ndepth),
        fmaxf(cdepth, ndepth));
    if (ndepth == 0.0f || ratio < 0.8f)
        d_main[i] = 0.0f;
}

/* app/smvsrecon.cc:362-377: the mean of two SGM results where both have a
 * depth, otherwise the one that has. */
__global__ void
sgm_merge_kernel (size_t n, float const* __restrict__ first,
    float* __restrict__ second_inout)
{
    size_t const i = static_cast<size_t>(blockIdx.x) * blockDim.x
        + threadIdx.x;
    if (i >= n)
        return;
    float const d1 = first[i], d2 = second_inout[i];
    float out = d1;
    if (d2 != 0.0f)
        out = (d1 == 0.0f) ? d2 : __fmul_rn(__fadd_rn(d1, d2), 0.5f);
    second_inout[i] = out;
}

/* One workspace per device, shared by all host threads (calls on a device
 * serialise: the volumes of one 2 MP x 128 run take 2.4 GB). After a call it
 * holds at most that call's budget (fit_workspace). */
struct SgmWorkspace
{
    std::mutex lock;
    bool ready = false;
    int device = 0;
    size_t card_bytes = 0;
    cudaStream_t st = nullptr;
    cudaStream_t copy = nullptr;     /* partial sums to and from the host */
    cudaEvent_t ev[8] = {};
    cudaEvent_t band_ev[8] = {};     /* 4 per partial-sum slot, see run_banded */
    DevBuf<uint8_t> d_main, d_neigh, d_cost, d_D, d_warp;
    DevBuf<uint16_t> d_S, d_part;
    DevBuf<uint4> d_state;
    DevBuf<float> d_depths, d_out, d_out2, d_prev, d_neigh_f;
};

SgmWorkspace g_sgm_ws[SMVSB_MAX_DEVICES];

void
check_sgm_args (int w, int h, int nw, int nh, void const* a, void const* b,
    void const* M, void const* t, void const* out, int num_steps,
    uint16_t penalty1, uint16_t penalty2)
{
    if (!(w > 9 && h > 7 && nw > 1 && nh > 1 && a && b && M && t && out))
        throw Error(SMVSB_ERR_INVALID, "smvsb_sgm: bad image arguments");
    if (num_steps < 32 || num_steps > 256 || num_steps % 32 != 0
        || (num_steps / 32 != 1 && num_steps / 32 != 2
            && num_steps / 32 != 4 && num_steps / 32 != 8))
        throw Error(SMVSB_ERR_INVALID,
            "smvsb_sgm: num_steps must be 32, 64, 128 or 256");
    /* the O(D) recurrence equals the reference's O(D^2) minimum only
     * for P1 <= P2 and without uint16 wrap-around */
    if (penalty1 > penalty2 || penalty2 > 255)
        throw Error(SMVSB_ERR_INVALID,
            "smvsb_sgm: need penalty1 <= penalty2 <= 255");
}

/* The start of sgm_run and sgm_reconstruct: the workspace of `device`, held
 * by `hold` for the call, with its streams ready. */
SgmWorkspace&
open_workspace (std::unique_lock<std::mutex>& hold, int device)
{
    check_device(device);
    if (device >= SMVSB_MAX_DEVICES)
        throw Error(SMVSB_ERR_INVALID, "device index out of range");
    SgmWorkspace& ws = g_sgm_ws[device];
    hold = std::unique_lock<std::mutex>(ws.lock);
    CUDA_CHECK(cudaSetDevice(device));
    if (!ws.ready)
    {
        CUDA_CHECK(cudaStreamCreateWithFlags(&ws.st, cudaStreamNonBlocking));
        CUDA_CHECK(cudaStreamCreateWithFlags(&ws.copy,
            cudaStreamNonBlocking));
        for (int i = 0; i < 8; ++i)
        {
            CUDA_CHECK(cudaEventCreate(&ws.ev[i]));
            CUDA_CHECK(cudaEventCreateWithFlags(&ws.band_ev[i],
                cudaEventDisableTiming));
        }
        usable_device_bytes(&ws.card_bytes);
        ws.device = device;
        ws.ready = true;
    }
    return ws;
}

/* The two byte images on their way to the device. */
void
upload_images (SgmWorkspace& ws, int w, int h, uint8_t const* main_lum,
    int nw, int nh, uint8_t const* neigh_lum)
{
    CUDA_CHECK(cudaMemcpyAsync(ws.d_main.p, main_lum,
        static_cast<size_t>(w) * h, cudaMemcpyHostToDevice, ws.st));
    CUDA_CHECK(cudaMemcpyAsync(ws.d_neigh.p, neigh_lum,
        static_cast<size_t>(nw) * nh, cudaMemcpyHostToDevice, ws.st));
}

/*
 * What one run_sgm of a w x h image at D planes keeps on the device besides
 * the images and depth maps, in elements of the workspace's buffers.
 *  - The volume path: cost (1 B/voxel), eight L - C volumes (8 B) and the
 *    warped volume with its margin (~1 B), for the whole image.
 *  - The banded path, per band of band_rows rows: cost, five L - C volumes
 *    (the most one sweep writes) and the warped volume with the census halo;
 *    the uint16 partial sums, for the whole image on the device or two band
 *    slots staged through the host; the carried state of the six vertical
 *    directions (D / 8 uint4 per column).
 */
struct PairPlan
{
    bool banded = false, host_part = false;
    int band_rows = 0, bands = 1;
    size_t cost = 0, dvol = 0, warp = 0, S = 0, part = 0, state = 0;

    size_t bytes (void) const
    {
        return cost + dvol + warp + (S + part) * sizeof(uint16_t)
            + state * sizeof(uint4);
    }
};

int
warp_pitch (int w)
{
    return (w + C2_W - 1) / C2_W * C2_W + 16;
}

int
warp_rows (int rows)
{
    return (rows + C2_H - 1) / C2_H * C2_H + 6;
}

PairPlan
pair_plan (int w, int h, int D, int band_rows, bool host_part)
{
    PairPlan q;
    q.banded = band_rows > 0;
    q.host_part = q.banded && host_part;
    int const r = q.banded ? band_rows : h;
    q.band_rows = r;
    q.bands = (h + r - 1) / r;
    size_t const row_vox = static_cast<size_t>(w) * D;
    q.cost = row_vox * r;
    q.dvol = q.cost * (q.banded ? 5 : 8);
    q.warp = static_cast<size_t>(warp_pitch(w)) * warp_rows(r) * D;
    if (q.banded)
    {
        q.part = q.host_part ? 2 * q.cost : row_vox * h;
        q.state = static_cast<size_t>(6) * w * (D / 8);
    }
    return q;
}

/* The bands on the banded path (they start at multiples of C2_H, so every
 * band but the last fills whole cost tiles). Partial sums stay on the device
 * when that still leaves bands of 64 rows or more (or as tall as host staging
 * would give); band_rows 0: not even 16 rows fit `avail`. */
PairPlan
banded_plan (int w, int h, int D, size_t avail)
{
    auto most_rows = [&] (bool host) {
        for (int r = (h + C2_H - 1) / C2_H * C2_H; r >= C2_H; r -= C2_H)
            if (pair_plan(w, h, D, r, host).bytes() <= avail)
                return r;
        return 0;
    };
    int const on_device = most_rows(false), on_host = most_rows(true);
    if (on_device > 0 && on_device >= std::min(on_host, 64))
        return pair_plan(w, h, D, on_device, false);
    PairPlan q = pair_plan(w, h, D, C2_H, true);
    if (on_host > 0)
        q = pair_plan(w, h, D, on_host, true);
    else
        q.band_rows = 0;
    return q;
}

/* The volume path when it fits `avail` (or the dumps ask for the volumes),
 * otherwise bands; throws when the budget does not hold one band. */
PairPlan
choose_plan (int w, int h, int D, bool dumps, size_t avail, size_t fixed,
    size_t budget, bool default_budget)
{
    PairPlan q = pair_plan(w, h, D, 0, false);
    if (dumps)
        q.S = static_cast<size_t>(w) * h * D;
    if (dumps || q.bytes() <= avail)
        return q;
    q = banded_plan(w, h, D, avail);
    if (q.band_rows == 0)
    {
        /* the smaller of one 16-row band's needs with the partial sums on
         * the device and with them staged (the device wins below 32 rows) */
        size_t const least = fixed + std::min(
            pair_plan(w, h, D, C2_H, false).bytes(),
            pair_plan(w, h, D, C2_H, true).bytes());
        throw Error(default_budget ? SMVSB_ERR_ALLOC : SMVSB_ERR_INVALID,
            "smvsb_sgm: a device budget of " + std::to_string(budget)
            + " bytes is below the minimum of " + std::to_string(least)
            + " bytes for " + std::to_string(w) + "x"
            + std::to_string(h) + " at " + std::to_string(D) + " planes "
            "(one band of 16 rows and the carried state)");
    }
    return q;
}

/* The device bytes of the images, depths and depth maps a call keeps for
 * its whole length. */
struct Fixed
{
    size_t main = 0, neigh = 0, neigh_f = 0, out = 0, out2 = 0, prev = 0;

    size_t bytes (void) const
    {
        return main + neigh + (neigh_f + out + out2 + prev + 512)
            * sizeof(float);
    }
};

/* fn(buffer, elements needed) over the buffers of the call's fixed data and
 * over those of one run's volumes. */
template <typename Fn>
void
each_fixed (SgmWorkspace& ws, Fixed const& f, Fn&& fn)
{
    fn(ws.d_main, f.main); fn(ws.d_neigh, f.neigh);
    fn(ws.d_neigh_f, f.neigh_f); fn(ws.d_out, f.out);
    fn(ws.d_out2, f.out2); fn(ws.d_prev, f.prev);
    fn(ws.d_depths, size_t(512));
}

template <typename Fn>
void
each_volume (SgmWorkspace& ws, PairPlan const& q, Fn&& fn)
{
    fn(ws.d_cost, q.cost); fn(ws.d_D, q.dvol); fn(ws.d_warp, q.warp);
    fn(ws.d_S, q.S); fn(ws.d_part, q.part); fn(ws.d_state, q.state);
}

/*
 * Sizes the workspace for one run: the call's fixed buffers (fixed_live:
 * already sized and holding data) and the run's volumes. When keeping every
 * buffer at least as large as it is would exceed the budget -- or would not
 * leave `later` bytes for a later run of the call -- the buffers larger than
 * needed are released first, so the workspace never holds more than the
 * budget (unless the volume dumps alone exceed it). Returns the bytes held.
 */
size_t
fit_workspace (SgmWorkspace& ws, Fixed const& f, bool fixed_live,
    PairPlan const& q, size_t budget, size_t later)
{
    size_t kept_fixed = 0, kept_vol = 0;
    each_fixed(ws, f, [&] (auto& b, size_t n) {
        kept_fixed += std::max(b.cap, n) * sizeof(*b.p); });
    each_volume(ws, q, [&] (auto& b, size_t n) {
        kept_vol += std::max(b.cap, n) * sizeof(*b.p); });
    auto shrink = [] (auto& b, size_t n) { if (b.cap > n) b.release(); };
    if (kept_fixed + std::max(kept_vol, later) > budget)
    {
        if (!fixed_live)
            each_fixed(ws, f, shrink);
        each_volume(ws, q, shrink);
    }
    size_t held = 0;
    auto grow = [&] (auto& b, size_t n) {
        b.reserve(n);
        held += b.bytes();
    };
    each_fixed(ws, f, grow);
    each_volume(ws, q, grow);
    return held;
}

void
release_workspace (SgmWorkspace& ws)
{
    auto drop = [] (auto& b, size_t) { b.release(); };
    each_fixed(ws, Fixed{}, drop);
    each_volume(ws, PairPlan{}, drop);
}

size_t
held_bytes (SgmWorkspace& ws)
{
    size_t held = 0;
    auto add = [&] (auto& b, size_t) { held += b.bytes(); };
    each_fixed(ws, Fixed{}, add);
    each_volume(ws, PairPlan{}, add);
    return held;
}

void
check_sgm_options (smvsb_sgm_options const* opts)
{
    if (opts != nullptr && (opts->reserved[0] != 0 || opts->reserved[1] != 0
        || opts->reserved[2] != 0))
        throw Error(SMVSB_ERR_INVALID,
            "smvsb_sgm_options: reserved fields must be 0");
}

/* True when the run's buffers are larger than what the workspace holds. */
bool
grows (SgmWorkspace& ws, Fixed const& f, PairPlan const& q)
{
    bool more = false;
    auto check = [&] (auto& b, size_t n) { more = more || n > b.cap; };
    each_fixed(ws, f, check);
    each_volume(ws, q, check);
    return more;
}

/*
 * The call's budget and the plans of its runs (plan(budget) returns them):
 * opts->device_bytes, or the smaller of a quarter of the card and what is
 * free (counting the workspace, which can be released) less the margin. The
 * free memory is only asked for (a slow runtime query) when the plans within
 * a quarter of the card need more than the workspace holds.
 */
template <typename Plan, typename Grows>
size_t
sgm_budget (SgmWorkspace& ws, smvsb_sgm_options const* opts, Plan&& plan,
    Grows&& needs_more)
{
    if (opts != nullptr && opts->device_bytes != 0)
    {
        plan(opts->device_bytes);
        return opts->device_bytes;
    }
    size_t budget = ws.card_bytes / 4;
    plan(budget);
    if (needs_more())
    {
        budget = std::min(budget, usable_device_bytes() + held_bytes(ws));
        plan(budget);
    }
    return budget;
}

/* Pinned host memory for the partial sums of one call. */
struct PinnedPart
{
    uint16_t* p = nullptr;
    size_t cap = 0;

    ~PinnedPart (void) { if (p) cudaFreeHost(p); }

    void reserve (size_t n)
    {
        if (n <= cap)
            return;
        if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
        cudaError_t const e = cudaHostAlloc(&p, n * sizeof(uint16_t),
            cudaHostAllocDefault);
        if (e != cudaSuccess)
        {
            p = nullptr;
            throw Error(SMVSB_ERR_ALLOC, std::string("cudaHostAlloc of ")
                + std::to_string(n * sizeof(uint16_t)) + " bytes: "
                + cudaGetErrorString(e));
        }
        cap = n;
    }
};

/* Warped volume and census cost of image rows [y0, y0 + rows) into d_cost
 * (the whole image: y0 = 0, rows = h). */
void
launch_cost (SgmWorkspace& ws, SgmParams const& p, uint8_t const* main_dev,
    float const* depths_dev, int y0, int rows)
{
    cudaStream_t st = ws.st;
    /* warped volume with the cost tiles' halo as margin (zeros, written by
     * the kernel itself) */
    int const pitch = warp_pitch(p.w);
    int const vrows = warp_rows(rows);
    dim3 const wb(WV_BX, WV_BY);
    dim3 const wg((pitch / 4 + WV_BX - 1) / WV_BX, (vrows + WV_BY - 1) / WV_BY);
    sgm_warp_volume_kernel<<<wg, wb, 0, st>>>(p, ws.d_neigh_f.p, depths_dev,
        ws.d_warp.p, pitch, vrows, y0);
    CUDA_CHECK(cudaGetLastError());
    dim3 const cg((p.w + C2_W - 1) / C2_W, (rows + C2_H - 1) / C2_H);
    size_t const tile_bytes = sizeof(unsigned) * 2 * 2 * PLANES
        * C2_HALO_H * C2_ROW_WORDS;
    CUDA_CHECK(cudaFuncSetAttribute(sgm_cost_bits_kernel,
        cudaFuncAttributeMaxDynamicSharedMemorySize,
        static_cast<int>(tile_bytes)));
    sgm_cost_bits_kernel<<<cg, C2_THREADS, tile_bytes, st>>>(p, main_dev,
        ws.d_warp.p, pitch, vrows, y0, ws.d_cost.p);
    CUDA_CHECK(cudaGetLastError());
}

/*
 * run_sgm in bands of q.band_rows rows. Sweep 0, top to bottom: cost, the
 * paths L2R, R2L, T2B, T2B_D1, T2B_D2 and their sum as uint16 partial sums
 * (at most 5 * 255). Sweep 1, bottom to top: cost again, the paths B2T,
 * B2T_D1, B2T_D2, and S = 8 C (+ the corner extra) + the three + the partial
 * sum with the winner, as sgm_sum_wta_kernel does for the whole volume. The
 * sums are integers: the depth is the volume path's.
 * Host staging: band b's partial sums go through device slot b % 2. Sweep 0
 * copies each slot to the host on the copy stream once it is written
 * (band_ev[s]: written, [2 + s]: copied out); sweep 1 loads band b - 1 into
 * its slot while band b runs (band_ev[4 + s]: loaded, [6 + s]: read). The
 * last band's sums are still in their slot when sweep 1 starts.
 * Returns the kernel launches.
 */
template <int D>
int
run_banded (SgmWorkspace& ws, SgmParams const& p, PairPlan const& q,
    unsigned P1, unsigned P2, uint8_t const* main_dev, float const* depths_dev,
    uint16_t* host_part, float* out_dev)
{
    constexpr int L = D / 8, G = D / 16;        /* lanes per line / pixel */
    constexpr int LPW = 32 / L;                 /* lines per warp */
    cudaStream_t st = ws.st, cp = ws.copy;
    cudaEvent_t* const ev = ws.band_ev;
    int const w = p.w, h = p.h, R = q.band_rows, nb = q.bands;
    size_t const row_vox = static_cast<size_t>(w) * D;
    size_t const band_vox = row_vox * R;
    auto rows_of = [&] (int b) { return std::min(R, h - b * R); };
    auto slot = [&] (int b) {
        return ws.d_part.p + (q.host_part ? (b & 1) : b) * band_vox;
    };
    auto band_bytes = [&] (int b) {
        return row_vox * rows_of(b) * sizeof(uint16_t);
    };
    int launches = 0;
    for (int sweep = 0; sweep < 2; ++sweep)
    {
        for (int i = 0; i < nb; ++i)
        {
            int const b = (sweep == 0) ? i : nb - 1 - i;
            int const y0 = b * R, rows = rows_of(b), s = b & 1;
            if (sweep == 1 && q.host_part && b > 0)
            {
                /* load band b - 1 once band b + 1 has read its slot */
                int const n = b - 1, sn = n & 1;
                if (n + 2 <= nb - 1)
                    CUDA_CHECK(cudaStreamWaitEvent(cp, ev[6 + sn], 0));
                CUDA_CHECK(cudaMemcpyAsync(slot(n), host_part
                    + static_cast<size_t>(n) * band_vox, band_bytes(n),
                    cudaMemcpyHostToDevice, cp));
                CUDA_CHECK(cudaEventRecord(ev[4 + sn], cp));
            }
            launch_cost(ws, p, main_dev, depths_dev, y0, rows);
            int const n_horiz = (sweep == 0) ? 2 : 0;
            int const warps = n_horiz * ((rows + LPW - 1) / LPW)
                + 3 * ((w + LPW - 1) / LPW);
            sgm_paths_kernel<L, true><<<(warps * 32 + 127) / 128, 128, 0,
                st>>>(w, h, P1, P2, ws.d_cost.p, ws.d_D.p,
                PathBand{ y0, rows, sweep, ws.d_state.p });
            CUDA_CHECK(cudaGetLastError());
            unsigned const blocks = static_cast<unsigned>(
                (static_cast<size_t>(w) * rows * G + 255) / 256);
            if (sweep == 0)
            {
                if (q.host_part && b >= 2)
                    CUDA_CHECK(cudaStreamWaitEvent(st, ev[2 + s], 0));
                sgm_sum_wta_kernel<G, 5, false, false><<<blocks, 256, 0,
                    st>>>(w, h, y0, rows, nullptr, ws.d_D.p, nullptr,
                    nullptr, nullptr, slot(b), nullptr);
                CUDA_CHECK(cudaGetLastError());
                if (q.host_part)
                {
                    CUDA_CHECK(cudaEventRecord(ev[s], st));
                    CUDA_CHECK(cudaStreamWaitEvent(cp, ev[s], 0));
                    CUDA_CHECK(cudaMemcpyAsync(host_part
                        + static_cast<size_t>(b) * band_vox, slot(b),
                        band_bytes(b), cudaMemcpyDeviceToHost, cp));
                    CUDA_CHECK(cudaEventRecord(ev[2 + s], cp));
                }
            }
            else
            {
                if (q.host_part && b < nb - 1)
                    CUDA_CHECK(cudaStreamWaitEvent(st, ev[4 + s], 0));
                sgm_sum_wta_kernel<G, 3, true, true><<<blocks, 256, 0,
                    st>>>(w, h, y0, rows, ws.d_cost.p, ws.d_D.p, slot(b),
                    main_dev, depths_dev, nullptr, out_dev);
                CUDA_CHECK(cudaGetLastError());
                if (q.host_part)
                    CUDA_CHECK(cudaEventRecord(ev[6 + s], st));
            }
            launches += 4;
        }
    }
    if (q.host_part)
    {
        /* nothing of the copy stream outlives the run */
        CUDA_CHECK(cudaEventRecord(ev[0], cp));
        CUDA_CHECK(cudaStreamWaitEvent(st, ev[0], 0));
    }
    return launches;
}

/* create_cost_volume + aggregate_sgm_costs + depth_from_sgm_volume for the
 * image pair already on the device, in the workspace fit_workspace sized for
 * plan q; ev[e0 .. e0+3] bracket the three stages (on the banded path they
 * interleave: ev[e0 + 1] and ev[e0 + 2] are recorded at the end). */
void
sgm_pair (SgmWorkspace& ws, PairPlan const& q, int w, int h,
    uint8_t const* main_dev, int nw, int nh, uint8_t const* neigh_dev,
    float const* M, float const* t, float min_depth, float max_depth,
    int num_steps, unsigned P1, unsigned P2, bool want_S, float* out_dev,
    int e0, PinnedPart& pinned)
{
    cudaStream_t st = ws.st;
    /* plane depths, lib/sgm_stereo.cc:195-203 (fp32 recurrence) */
    std::vector<float> depths(num_steps);
    {
        float inv_depth = 1.0f / max_depth;
        float const increment = (1.0f / min_depth - inv_depth)
            / (num_steps - 1);
        for (int i = 0; i < num_steps; ++i)
        {
            depths[i] = 1.0f / inv_depth;
            inv_depth += increment;
        }
    }
    /* two slots: the first pair of a reconstruct call may still be reading
     * its depths when the second pair's are copied */
    float* const depths_dev = ws.d_depths.p + (e0 != 0 ? 256 : 0);
    CUDA_CHECK(cudaMemcpyAsync(depths_dev, depths.data(),
        num_steps * sizeof(float), cudaMemcpyHostToDevice, st));
    /* pageable source: staged before the call returns */

    SgmParams p;
    p.w = w; p.h = h; p.nw = nw; p.nh = nh; p.D = num_steps;
    std::copy(M, M + 9, p.M);
    std::copy(t, t + 3, p.t);
    /* page-locking the host's partial sums takes the host a while: before
     * the events, so that they time the device (a no-op in a reconstruct,
     * which sizes the buffer for both runs) */
    if (q.host_part)
        pinned.reserve(static_cast<size_t>(w) * h * num_steps);

    CUDA_CHECK(cudaEventRecord(ws.ev[e0], st));
    /* float copy of the neighbour's byte image (part of the cost stage) */
    size_t const nnpix = static_cast<size_t>(nw) * nh;
    u8_to_float_kernel<<<static_cast<unsigned>((nnpix + 255) / 256), 256, 0,
        st>>>(nnpix, neigh_dev, ws.d_neigh_f.p);
    CUDA_CHECK(cudaGetLastError());

    if (q.banded)
    {
        uint16_t* const host_part = q.host_part ? pinned.p : nullptr;
        int launches = 0;
        switch (num_steps)
        {
        case 32: launches = run_banded<32>(ws, p, q, P1, P2, main_dev, depths_dev, host_part, out_dev); break;
        case 64: launches = run_banded<64>(ws, p, q, P1, P2, main_dev, depths_dev, host_part, out_dev); break;
        case 128: launches = run_banded<128>(ws, p, q, P1, P2, main_dev, depths_dev, host_part, out_dev); break;
        default: launches = run_banded<256>(ws, p, q, P1, P2, main_dev, depths_dev, host_part, out_dev); break;
        }
        count_device_launches(ws.device, 1 + launches);
        for (int k = 1; k <= 3; ++k)
            CUDA_CHECK(cudaEventRecord(ws.ev[e0 + k], st));
        return;
    }

    launch_cost(ws, p, main_dev, depths_dev, 0, h);
    CUDA_CHECK(cudaEventRecord(ws.ev[e0 + 1], st));

    uint16_t* const S_dev = want_S ? ws.d_S.p : nullptr;
    switch (num_steps)
    {
    case 32: run_paths_wta<32>(w, h, P1, P2, ws.d_cost.p, ws.d_D.p, main_dev, depths_dev, S_dev, out_dev, ws.ev[e0 + 2], st); break;
    case 64: run_paths_wta<64>(w, h, P1, P2, ws.d_cost.p, ws.d_D.p, main_dev, depths_dev, S_dev, out_dev, ws.ev[e0 + 2], st); break;
    case 128: run_paths_wta<128>(w, h, P1, P2, ws.d_cost.p, ws.d_D.p, main_dev, depths_dev, S_dev, out_dev, ws.ev[e0 + 2], st); break;
    default: run_paths_wta<256>(w, h, P1, P2, ws.d_cost.p, ws.d_D.p, main_dev, depths_dev, S_dev, out_dev, ws.ev[e0 + 2], st); break;
    }
    /* u8_to_float, warp volume, cost bits, paths, sum + WTA */
    count_device_launches(ws.device, 5);
    CUDA_CHECK(cudaEventRecord(ws.ev[e0 + 3], st));
}

void
note_pair (smvsb_sgm_stats* stats, PairPlan const& q, size_t held, int w,
    int h, int D)
{
    if (stats == nullptr)
        return;
    stats->banded |= q.banded ? 1 : 0;
    stats->bands = std::max(stats->bands, q.bands);
    stats->peak_device_bytes = std::max<uint64_t>(stats->peak_device_bytes,
        held);
    if (q.host_part)
        stats->host_bytes += static_cast<uint64_t>(w) * h * D
            * sizeof(uint16_t);
}

} /* namespace */

void
sgm_run (int device, int w, int h, uint8_t const* main_lum, int nw, int nh,
    uint8_t const* neigh_lum, float const* M, float const* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out, smvsb_sgm_options const* opts,
    smvsb_sgm_stats* stats)
{
    check_sgm_args(w, h, nw, nh, main_lum, neigh_lum, M, t, depth_out,
        num_steps, penalty1, penalty2);
    check_sgm_options(opts);
    if (stats != nullptr)
        *stats = smvsb_sgm_stats{};
    std::unique_lock<std::mutex> hold;
    SgmWorkspace& ws = open_workspace(hold, device);
    cudaStream_t st = ws.st;
    size_t const npix = static_cast<size_t>(w) * h;
    size_t const nvox = npix * num_steps;
    bool const dumps = (cost_out != nullptr || sgm_out != nullptr);
    Fixed f;
    f.main = npix; f.neigh = static_cast<size_t>(nw) * nh;
    f.neigh_f = f.neigh; f.out = npix;
    PairPlan q;
    size_t const budget = sgm_budget(ws, opts, [&] (size_t b) {
        size_t const avail = b > f.bytes() ? b - f.bytes() : 0;
        q = choose_plan(w, h, num_steps, dumps, avail, f.bytes(), b,
            opts == nullptr || opts->device_bytes == 0);
    }, [&] { return grows(ws, f, q); });
    size_t const held = fit_workspace(ws, f, false, q, budget, 0);
    note_pair(stats, q, held, w, h, num_steps);
    upload_images(ws, w, h, main_lum, nw, nh, neigh_lum);
    PinnedPart pinned;
    sgm_pair(ws, q, w, h, ws.d_main.p, nw, nh, ws.d_neigh.p, M, t, min_depth,
        max_depth, num_steps, penalty1, penalty2, sgm_out != nullptr,
        ws.d_out.p, 0, pinned);
    CUDA_CHECK(cudaMemcpyAsync(depth_out, ws.d_out.p, npix * sizeof(float),
        cudaMemcpyDeviceToHost, st));
    if (sgm_out)
        CUDA_CHECK(cudaMemcpyAsync(sgm_out, ws.d_S.p,
            nvox * sizeof(uint16_t), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (cost_out)
    {
        /* widen through the (now free) S buffer */
        u8_to_u16_kernel<<<static_cast<unsigned>((nvox + 255) / 256), 256,
            0, st>>>(nvox, ws.d_cost.p, ws.d_S.p);
        CUDA_CHECK(cudaGetLastError());
        count_device_launches(device, 1);
        CUDA_CHECK(cudaMemcpyAsync(cost_out, ws.d_S.p,
            nvox * sizeof(uint16_t), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    }
    /* the volume dumps are the one way past the budget: not kept */
    if (held > budget)
        release_workspace(ws);
    float ms[3];
    for (int i = 0; i < 3; ++i)
        CUDA_CHECK(cudaEventElapsedTime(&ms[i], ws.ev[i], ws.ev[i + 1]));
    if (ms_out)
        for (int i = 0; i < 3; ++i)
            ms_out[i] = q.banded ? (i == 0 ? ms[0] + ms[1] + ms[2] : 0.0)
                : ms[i];
    if (stats != nullptr)
        stats->ms_device = ms[0] + ms[1] + ms[2];
}

/* SGMStereo::reconstruct (lib/sgm_stereo.cc:45-96) for an image pair at SGM
 * working resolution, optionally followed by the merge of
 * app/smvsrecon.cc:362-377 with an earlier result. */
void
sgm_reconstruct (int device, int w, int h, uint8_t const* main_lum, int nw,
    int nh, uint8_t const* neigh_lum, float const* M_mn, float const* t_mn,
    float const* M_nm, float const* t_nm, float const* depth_range_main,
    float const* depth_range_neigh, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float const* merge_with, float* depth_out,
    double* ms_out, smvsb_sgm_options const* opts, smvsb_sgm_stats* stats)
{
    check_sgm_args(w, h, nw, nh, main_lum, neigh_lum, M_mn, t_mn, depth_out,
        num_steps, penalty1, penalty2);
    check_sgm_options(opts);
    if (!(nw > 9 && nh > 7 && M_nm && t_nm && depth_range_main
        && depth_range_neigh))
        throw Error(SMVSB_ERR_INVALID, "smvsb_sgm_reconstruct: bad arguments");
    if (stats != nullptr)
        *stats = smvsb_sgm_stats{};
    std::unique_lock<std::mutex> hold;
    SgmWorkspace& ws = open_workspace(hold, device);
    cudaStream_t st = ws.st;
    size_t const npix = static_cast<size_t>(w) * h;
    size_t const nnpix = static_cast<size_t>(nw) * nh;
    bool const default_budget = opts == nullptr || opts->device_bytes == 0;
    Fixed f;
    f.main = npix; f.neigh = nnpix;
    f.neigh_f = std::max(npix, nnpix);
    f.out = npix; f.out2 = nnpix;
    f.prev = (merge_with != nullptr) ? npix : 0;
    /* sgm1: main against neighbour; sgm2: the roles swapped (:56-62) */
    PairPlan q1, q2;
    size_t const budget = sgm_budget(ws, opts, [&] (size_t b) {
        size_t const avail = b > f.bytes() ? b - f.bytes() : 0;
        q1 = choose_plan(w, h, num_steps, false, avail, f.bytes(), b,
            default_budget);
        q2 = choose_plan(nw, nh, num_steps, false, avail, f.bytes(), b,
            default_budget);
    }, [&] { return grows(ws, f, q1) || grows(ws, f, q2); });
    size_t held = fit_workspace(ws, f, false, q1, budget, q2.bytes());
    note_pair(stats, q1, held, w, h, num_steps);
    upload_images(ws, w, h, main_lum, nw, nh, neigh_lum);
    if (merge_with != nullptr)
        CUDA_CHECK(cudaMemcpyAsync(ws.d_prev.p, merge_with,
            npix * sizeof(float), cudaMemcpyHostToDevice, st));
    /* sized for both runs before the first: growing it between them would
     * free memory the first run's copies may still use */
    PinnedPart pinned;
    pinned.reserve(std::max(q1.host_part ? npix * num_steps : 0,
        q2.host_part ? nnpix * num_steps : 0));
    sgm_pair(ws, q1, w, h, ws.d_main.p, nw, nh, ws.d_neigh.p, M_mn, t_mn,
        depth_range_main[0], depth_range_main[1], num_steps, penalty1,
        penalty2, false, ws.d_out.p, 0, pinned);
    held = fit_workspace(ws, f, true, q2, budget, 0);
    note_pair(stats, q2, held, nw, nh, num_steps);
    sgm_pair(ws, q2, nw, nh, ws.d_neigh.p, w, h, ws.d_main.p, M_nm, t_nm,
        depth_range_neigh[0], depth_range_neigh[1], num_steps, penalty1,
        penalty2, false, ws.d_out2.p, 4, pinned);

    ConsistencyParams cp;
    cp.w = w; cp.h = h; cp.nw = nw; cp.nh = nh;
    cp.cut = static_cast<int>(0.03 * std::max(nw, nh));
    for (int i = 0; i < 9; ++i) cp.M[i] = M_mn[i];
    for (int i = 0; i < 3; ++i) cp.t[i] = t_mn[i];
    dim3 const block(32, 8);
    dim3 const grid((w + 31) / 32, (h + 7) / 8);
    sgm_consistency_kernel<<<grid, block, 0, st>>>(cp, ws.d_out.p,
        ws.d_out2.p);
    CUDA_CHECK(cudaGetLastError());
    count_device_launches(device, 1);
    if (merge_with != nullptr)
    {
        sgm_merge_kernel<<<static_cast<unsigned>((npix + 255) / 256), 256,
            0, st>>>(npix, ws.d_prev.p, ws.d_out.p);
        CUDA_CHECK(cudaGetLastError());
        count_device_launches(device, 1);
    }
    CUDA_CHECK(cudaMemcpyAsync(depth_out, ws.d_out.p, npix * sizeof(float),
        cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    float ms[2];
    CUDA_CHECK(cudaEventElapsedTime(&ms[0], ws.ev[0], ws.ev[3]));
    CUDA_CHECK(cudaEventElapsedTime(&ms[1], ws.ev[4], ws.ev[7]));
    if (ms_out)
    {
        ms_out[0] = ms[0];
        ms_out[1] = ms[1];
    }
    if (stats != nullptr)
        stats->ms_device = ms[0] + ms[1];
}

} /* namespace smvsb */
