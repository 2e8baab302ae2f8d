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
 * warped_neighbors_for_depth (:150-190) gives main pixel (col - 4, row - 3)
 * at that plane, 0 outside the image -- a margin of the census window's halo
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
    int rows)
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
    int const gy = row - 3;
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
    uint8_t const* __restrict__ Wv, int pitch, int rows,
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

    /* main image tile (0x6400 | byte, like the warped tiles), both copies */
    {
        unsigned short* t0 = reinterpret_cast<unsigned short*>(
            &s_tile[0][0][0][0][0]);
        unsigned short* t1 = reinterpret_cast<unsigned short*>(
            &s_tile[0][1][0][0][0]);
        for (int i = tid; i < C2_HALO_W * C2_HALO_H; i += C2_THREADS)
        {
            int const c = i % C2_HALO_W, r = i / C2_HALO_W;
            int const gx = x0 - 4 + c, gy = y0 - 3 + r;
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
        in_px[i] = (px + i < p.w && py < p.h);
        int_px[i] = in_px[i] && px + i >= 4 && px + i < p.w - 5 && py >= 3
            && py < p.h - 4;
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
 */
template <int L>
__global__ void __launch_bounds__(128)
sgm_paths_kernel (int w, int h, unsigned P1, unsigned P2,
    uint8_t const* __restrict__ cost, uint8_t* __restrict__ Dvol)
{
    constexpr int D = 8 * L;
    constexpr int LPW = 32 / L;                 /* lines per warp */
    int const grp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    int const sl = lane & (L - 1);              /* lane within the line */
    int const hp = (h + LPW - 1) / LPW, wp = (w + LPW - 1) / LPW;
    int kind, line, count;
    if (grp < 2 * hp)
    {
        kind = grp / hp;                        /* PATH_L2R, PATH_R2L */
        line = LPW * (grp % hp) + (lane >> ilog2(L));
        count = h;
    }
    else
    {
        int const q = grp - 2 * hp;
        if (q >= 6 * wp)
            return;
        kind = 2 + q / wp;                      /* PATH_T2B .. PATH_B2T_D2 */
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
    int const steps = horizontal ? w : h;
    size_t const nvox = static_cast<size_t>(w) * h * D;
    uint8_t* __restrict__ Dr = Dvol + static_cast<size_t>(kind) * nvox;

    int x, y, dx, dy;
    switch (kind)
    {
    case PATH_L2R: x = 0; y = line; dx = 1; dy = 0; break;
    case PATH_R2L: x = w - 1; y = line; dx = -1; dy = 0; break;
    case PATH_T2B: x = line; y = 0; dx = 0; dy = 1; break;
    case PATH_T2B_D1: x = line; y = 0; dx = 1; dy = 1; break;
    case PATH_T2B_D2: x = line; y = 0; dx = -1; dy = 1; break;
    case PATH_B2T: x = line; y = h - 1; dx = 0; dy = -1; break;
    case PATH_B2T_D1: x = line; y = h - 1; dx = 1; dy = -1; break;
    default: x = line; y = h - 1; dx = -1; dy = -1; break;   /* B2T_D2 */
    }
    int const restart_x = (dx > 0) ? 0 : w - 1;   /* diagonals only */
    bool const diagonal = (!horizontal && dx != 0);

    unsigned const P1x2 = P1 | (P1 << 16), P2x2 = P2 | (P2 << 16);
    unsigned const BIG = 0x7000u;          /* "no neighbour" sentinel */
    unsigned Pa = 0, Pb = 0, Pc = 0, Pd = 0;
    long long const row_bytes = static_cast<long long>(w) * D;
    long long const step_bytes = dy * row_bytes + dx * D;
    uint8_t const* pc = cost + (static_cast<size_t>(y) * w + x) * D + sl * 8;
    uint8_t* pd = Dr + (static_cast<size_t>(y) * w + x) * D + sl * 8;
    uint2 c8 = *reinterpret_cast<uint2 const*>(pc);
    bool start = true;
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

template <int G>
__global__ void __launch_bounds__(256)
sgm_sum_wta_kernel (int w, int h, uint8_t const* __restrict__ cost,
    uint8_t const* __restrict__ Dvol, uint8_t const* __restrict__ main_img,
    float const* __restrict__ depths, uint16_t* __restrict__ S_out,
    float* __restrict__ out)
{
    constexpr int D = 16 * G;
    int const npix = w * h;
    int const t = blockIdx.x * blockDim.x + threadIdx.x;
    int const p = t >> ilog2(G), sub = threadIdx.x & (G - 1);
    bool const on = p < npix;
    size_t const nvox = static_cast<size_t>(npix) * D;
    size_t const base = static_cast<size_t>(on ? p : 0) * D + sub * 16;
    int const px = p % w, py = p / w;
    unsigned const mult = 8u + (((px == 0 || px == w - 1)
        && (py == 0 || py == h - 1)) ? 1u : 0u);
    unsigned even[4] = { 0u, 0u, 0u, 0u }, odd[4] = { 0u, 0u, 0u, 0u };
    uint4 v[9];
    v[0] = __ldg(reinterpret_cast<uint4 const*>(cost + base));
#pragma unroll
    for (int r = 0; r < 8; ++r)
        v[r + 1] = __ldg(reinterpret_cast<uint4 const*>(Dvol + r * nvox + base));
    wta_add16(v[0], mult, even, odd);
#pragma unroll
    for (int r = 0; r < 8; ++r)
        wta_add16(v[r + 1], 1u, even, odd);
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
        out[p] = (idx < 2 || main_img[p] < 25) ? 0.0f : depths[idx];
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
    sgm_paths_kernel<L><<<(warps * 32 + 127) / 128, 128, 0, st>>>(w, h, P1,
        P2, cost, Dvol);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaEventRecord(mid, st));
    sgm_sum_wta_kernel<G><<<(w * h * G + 255) / 256, 256, 0, st>>>(w, h,
        cost, Dvol, main_img, depths, S_out, out);
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
 * serialise: the volumes of one 2 MP x 128 run take 2.4 GB). */
struct SgmWorkspace
{
    std::mutex lock;
    bool ready = false;
    int device = 0;
    cudaStream_t st = nullptr;
    cudaEvent_t ev[8] = {};
    DevBuf<uint8_t> d_main, d_neigh, d_cost, d_D, d_warp;
    DevBuf<uint16_t> d_S;
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
 * by `hold` for the call, its stream ready and the two byte images on their
 * way to the device. */
SgmWorkspace&
open_workspace (std::unique_lock<std::mutex>& hold, int device, int w, int h,
    uint8_t const* main_lum, int nw, int nh, uint8_t const* neigh_lum)
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
        for (int i = 0; i < 8; ++i)
            CUDA_CHECK(cudaEventCreate(&ws.ev[i]));
        ws.device = device;
        ws.ready = true;
    }
    size_t const npix = static_cast<size_t>(w) * h;
    size_t const nnpix = static_cast<size_t>(nw) * nh;
    ws.d_main.reserve(npix);
    ws.d_neigh.reserve(nnpix);
    CUDA_CHECK(cudaMemcpyAsync(ws.d_main.p, main_lum, npix,
        cudaMemcpyHostToDevice, ws.st));
    CUDA_CHECK(cudaMemcpyAsync(ws.d_neigh.p, neigh_lum, nnpix,
        cudaMemcpyHostToDevice, ws.st));
    return ws;
}

/* create_cost_volume + aggregate_sgm_costs + depth_from_sgm_volume for the
 * image pair already on the device; ev[e0 .. e0+3] bracket the three stages. */
void
sgm_pair (SgmWorkspace& ws, int w, int h, uint8_t const* main_dev, int nw,
    int nh, uint8_t const* neigh_dev, float const* M, float const* t,
    float min_depth, float max_depth, int num_steps, unsigned P1, unsigned P2,
    bool want_S, float* out_dev, int e0)
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
    size_t const npix = static_cast<size_t>(w) * h;
    size_t const nvox = npix * num_steps;
    ws.d_cost.reserve(nvox);
    ws.d_D.reserve(nvox * 8);                 /* L - C per direction */
    if (want_S)
        ws.d_S.reserve(nvox);
    /* two slots: the first pair of a reconstruct call may still be reading
     * its depths when the second pair's are copied */
    ws.d_depths.reserve(512);
    float* const depths_dev = ws.d_depths.p + (e0 != 0 ? 256 : 0);
    CUDA_CHECK(cudaMemcpyAsync(depths_dev, depths.data(),
        num_steps * sizeof(float), cudaMemcpyHostToDevice, st));
    /* pageable source: staged before the call returns */

    SgmParams p;
    p.w = w; p.h = h; p.nw = nw; p.nh = nh; p.D = num_steps;
    std::copy(M, M + 9, p.M);
    std::copy(t, t + 3, p.t);

    CUDA_CHECK(cudaEventRecord(ws.ev[e0], st));
    /* float copy of the neighbour's byte image (part of the cost stage) */
    size_t const nnpix = static_cast<size_t>(nw) * nh;
    ws.d_neigh_f.reserve(nnpix);
    u8_to_float_kernel<<<static_cast<unsigned>((nnpix + 255) / 256), 256, 0,
        st>>>(nnpix, neigh_dev, ws.d_neigh_f.p);
    CUDA_CHECK(cudaGetLastError());
    /* warped volume with the cost tiles' halo as margin (zeros, written by
     * the kernel itself) */
    int const pitch = (w + C2_W - 1) / C2_W * C2_W + 16;
    int const rows = (h + C2_H - 1) / C2_H * C2_H + 6;
    ws.d_warp.reserve(static_cast<size_t>(pitch) * rows * num_steps);
    dim3 const wb(WV_BX, WV_BY);
    dim3 const wg((pitch / 4 + WV_BX - 1) / WV_BX, (rows + WV_BY - 1) / WV_BY);
    sgm_warp_volume_kernel<<<wg, wb, 0, st>>>(p, ws.d_neigh_f.p, depths_dev,
        ws.d_warp.p, pitch, rows);
    CUDA_CHECK(cudaGetLastError());
    dim3 const cg((w + C2_W - 1) / C2_W, (h + C2_H - 1) / C2_H);
    size_t const tile_bytes = sizeof(unsigned) * 2 * 2 * PLANES
        * C2_HALO_H * C2_ROW_WORDS;
    CUDA_CHECK(cudaFuncSetAttribute(sgm_cost_bits_kernel,
        cudaFuncAttributeMaxDynamicSharedMemorySize,
        static_cast<int>(tile_bytes)));
    sgm_cost_bits_kernel<<<cg, C2_THREADS, tile_bytes, st>>>(p, main_dev,
        ws.d_warp.p, pitch, rows, ws.d_cost.p);
    CUDA_CHECK(cudaGetLastError());
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

} /* namespace */

void
sgm_run (int device, int w, int h, uint8_t const* main_lum, int nw, int nh,
    uint8_t const* neigh_lum, float const* M, float const* t,
    float min_depth, float max_depth, int num_steps, uint16_t penalty1,
    uint16_t penalty2, float* depth_out, uint16_t* cost_out,
    uint16_t* sgm_out, double* ms_out)
{
    check_sgm_args(w, h, nw, nh, main_lum, neigh_lum, M, t, depth_out,
        num_steps, penalty1, penalty2);
    std::unique_lock<std::mutex> hold;
    SgmWorkspace& ws = open_workspace(hold, device, w, h, main_lum, nw, nh,
        neigh_lum);
    cudaStream_t st = ws.st;
    size_t const npix = static_cast<size_t>(w) * h;
    size_t const nvox = npix * num_steps;
    ws.d_out.reserve(npix);
    if (cost_out)
        ws.d_S.reserve(nvox);
    sgm_pair(ws, w, h, ws.d_main.p, nw, nh, ws.d_neigh.p, M, t, min_depth,
        max_depth, num_steps, penalty1, penalty2, sgm_out != nullptr,
        ws.d_out.p, 0);
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
    if (ms_out)
    {
        float ms;
        for (int i = 0; i < 3; ++i)
        {
            CUDA_CHECK(cudaEventElapsedTime(&ms, ws.ev[i], ws.ev[i + 1]));
            ms_out[i] = ms;
        }
    }
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
    double* ms_out)
{
    check_sgm_args(w, h, nw, nh, main_lum, neigh_lum, M_mn, t_mn, depth_out,
        num_steps, penalty1, penalty2);
    if (!(nw > 9 && nh > 7 && M_nm && t_nm && depth_range_main
        && depth_range_neigh))
        throw Error(SMVSB_ERR_INVALID, "smvsb_sgm_reconstruct: bad arguments");
    std::unique_lock<std::mutex> hold;
    SgmWorkspace& ws = open_workspace(hold, device, w, h, main_lum, nw, nh,
        neigh_lum);
    cudaStream_t st = ws.st;
    size_t const npix = static_cast<size_t>(w) * h;
    ws.d_out.reserve(npix);
    ws.d_out2.reserve(static_cast<size_t>(nw) * nh);
    if (merge_with != nullptr)
    {
        ws.d_prev.reserve(npix);
        CUDA_CHECK(cudaMemcpyAsync(ws.d_prev.p, merge_with,
            npix * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    /* sgm1: main against neighbour; sgm2: the roles swapped (:56-62) */
    sgm_pair(ws, w, h, ws.d_main.p, nw, nh, ws.d_neigh.p, M_mn, t_mn,
        depth_range_main[0], depth_range_main[1], num_steps, penalty1,
        penalty2, false, ws.d_out.p, 0);
    sgm_pair(ws, nw, nh, ws.d_neigh.p, w, h, ws.d_main.p, M_nm, t_nm,
        depth_range_neigh[0], depth_range_neigh[1], num_steps, penalty1,
        penalty2, false, ws.d_out2.p, 4);

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
    if (ms_out)
    {
        float ms;
        CUDA_CHECK(cudaEventElapsedTime(&ms, ws.ev[0], ws.ev[3]));
        ms_out[0] = ms;
        CUDA_CHECK(cudaEventElapsedTime(&ms, ws.ev[4], ws.ev[7]));
        ms_out[1] = ms;
    }
}

} /* namespace smvsb */
