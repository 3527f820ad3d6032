// mlp_wgmma.cu -- tensor-core Linear layers for the policy / value nets (SURVEY.md a13/a14): rollout-time forward and the whole autograd of the PPO update.
//   y[M][N] = act(x[M][Kp] W[N][Kp]^T + b),  bf16 operands (K-major, zero padded to Kp % 64 == 0), fp32 accumulation in registers.  sm_90a (Hopper wgmma).
//   k_linear_tc   one CTA per 128 x 128 tile: TMA (cp.async.bulk.tensor) -> 5-stage smem ring (mbarrier full / empty pairs) -> two consumer warpgroups, each
//                 issuing wgmma.mma_async m64n128k16 for its 64 rows with one k-block of MMAs kept in flight; warp 8 is the TMA producer.  Split-K work
//                 (gridDim.z slices of the reduction) for plain fp32 products with few output tiles: the TMA engine adds the partial tiles into the output.
// Epilogue: the accumulator fragments are handed through shared memory to a row-per-lane layout (warp = 32 rows x 64 columns); bias + activation; outputs
// staged in swizzled shared-memory tiles and stored by the TMA engine (fp32 pre-activation z, bf16 / fp32 y, the TRANSPOSED bf16 y for the backward pass'
// dW GEMM); DACT variant = the backward pass' dX GEMM with the previous layer's activation backward fused in (z tile fetched by TMA, dz / dz^T stored by
// TMA, bias gradient by a warp transpose-reduce).  Host entry points at the end of the file (C ABI: include/uhc_nn.h).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <string>
#include "../../include/uhc_nn.h"
#include "errors.h"
#include "group_core.h"

namespace {
constexpr int BM = 128, BN = 128, BK = 64, UK = 16, STAGES = 5;   // 5 stages x 32 KB in flight: one CTA per SM (up to 227 KB of shared memory per block)
constexpr int STAGE_BYTES = (BM * BK + BN * BK) * 2;             // 32 KB
constexpr int NTHREADS = 288;                                    // warps 0..7: two consumer warpgroups (MMA, then epilogue), warp 8: TMA producer
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;    // + alignment slack + barriers
// epilogue staging inside the (then idle) operand ring, one block per epilogue warp: [fp32 32x32 tile A | fp32 32x32 tile B | bf16 32x32 tile | bias row]
constexpr int EPI_F32_A = 0, EPI_F32_B = 4096, EPI_BF16 = 8192, EPI_BIAS = 10240, EPI_BLOCK = 11264;
// behind the staging blocks: the 128 x 128 fp32 accumulator tile in which the wgmma fragments change hands to the row-per-lane epilogue layout
// (pitch 132 floats: the fragment stores and the 16-byte row reads of a quarter warp touch distinct banks)
constexpr int ACC_OFF = 8 * EPI_BLOCK, ACC_LD = 132;
static_assert(ACC_OFF + BM * ACC_LD * 4 <= STAGES * STAGE_BYTES, "epilogue staging must fit the operand ring");
#ifndef UHC_TC_TMA_STORE
#define UHC_TC_TMA_STORE 1       /* outputs leave through the TMA engine (cp.async.bulk.tensor shared -> global) where their row pitch allows it */
#endif

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t cnt) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(cnt)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.b32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) { while (!mbar_try_wait(bar, parity)) {} }
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// one 32 x 32 tile, shared -> global, clipped at the tensor's bounds by the TMA engine
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap *map, uint32_t src, int c0, int c1) {      // global[tile] += shared tile (element type from the map: fp32)
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
// this thread's row of 32 fp32 values into a 32 x 128 B tile laid out for a SWIZZLE_128B tensor map (16-byte chunk j of row r sits at chunk j ^ (r & 7))
__device__ __forceinline__ void stage_row_f32_sw128(uint32_t tile, int r, const float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile + r * 128 + ((j ^ (r & 7)) << 4)), "f"(v[4 * j]), "f"(v[4 * j + 1]), "f"(v[4 * j + 2]), "f"(v[4 * j + 3]) : "memory");
}
// the same as bf16 into a 32 x 64 B tile for a SWIZZLE_64B map (chunk j of row r sits at chunk j ^ ((r >> 1) & 3))
__device__ __forceinline__ void stage_row_bf16_sw64(uint32_t tile, int r, const float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 p0 = __floats2bfloat162_rn(v[8 * j], v[8 * j + 1]), p1 = __floats2bfloat162_rn(v[8 * j + 2], v[8 * j + 3]);
        __nv_bfloat162 p2 = __floats2bfloat162_rn(v[8 * j + 4], v[8 * j + 5]), p3 = __floats2bfloat162_rn(v[8 * j + 6], v[8 * j + 7]);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(tile + r * 64 + ((j ^ ((r >> 1) & 3)) << 4)), "r"(*(uint32_t *)&p0), "r"(*(uint32_t *)&p1),
                     "r"(*(uint32_t *)&p2), "r"(*(uint32_t *)&p3) : "memory");
    }
}
// this thread's row m (= lane) of 32 values as COLUMN m of the transposed 32 x 64 B bf16 tile (row j = output column nb + j), SWIZZLE_64B layout
__device__ __forceinline__ void stage_col_bf16_sw64(uint32_t tile, int m, const float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const unsigned short h = __bfloat16_as_ushort(__float2bfloat16_rn(v[j]));
        asm volatile("st.shared.b16 [%0], %1;" ::"r"(tile + j * 64 + ((((m >> 3) ^ ((j >> 1) & 3))) << 4) + ((m & 7) << 1)), "h"(h) : "memory");
    }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// K-major, 128B-swizzled operand tile: 8-row groups 1024 B apart (wgmma matrix descriptor: start >> 4, leading byte offset (unused for swizzled K-major),
// stride byte offset >> 4, layout type 1 = SWIZZLE_128B in bits 62-63)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// D[64][128] (+)= A[64][16] B[128][16]^T, both operands K-major in shared memory; the warpgroup's accumulator fragment: warp w, lane l holds for column block
// j = 0..15 d[4j], d[4j+1] at row 16w + l / 4, columns 8j + 2 (l % 4) + {0, 1}, and d[4j+2], d[4j+3] at row 16w + l / 4 + 8
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]),
                   "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]),
                   "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
                   "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc), "r"(accum) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// erf by Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7, i.e. below the bf16 / fp32 noise of this path) on the fast exp / rcp units:
// the epilogue is instruction-latency bound, and erff() alone costs more than the tile's tensor-core time
__device__ __forceinline__ float gelu_fast(float z) {
    const float x = fabsf(z) * 0.70710678118654752f;
    const float t = __fdividef(1.0f, fmaf(0.3275911f, x, 1.0f));
    const float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
    const float e = 1.0f - poly * __expf(-x * x);            // erf(|z| / sqrt 2)
    return 0.5f * z + 0.5f * fabsf(z) * e;                  // 0.5 z (1 + sign(z) e)
}
__device__ __forceinline__ float act_f(float z, int act) {
    switch (act) {
    case UHC_ACT_GELU: return gelu_fast(z);
    case UHC_ACT_TANH: return tanhf(z);
    case UHC_ACT_RELU: return z > 0.f ? z : 0.f;
    case UHC_ACT_SIGMOID: return 1.0f / (1.0f + expf(-z));
    }
    return z;
}

// act'(z) for the fused activation backward; GELU through the same erf approximation (one exp shared by the erf tail and the density)
__device__ __forceinline__ float act_b_fast(float z, int act) {
    switch (act) {
    case UHC_ACT_GELU: {
        const float x = fabsf(z) * 0.70710678118654752f;
        const float t = __fdividef(1.0f, fmaf(0.3275911f, x, 1.0f));
        const float E = __expf(-x * x);                                   // exp(-z^2 / 2)
        const float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
        const float e = 1.0f - poly * E;                                  // erf(|z| / sqrt 2)
        return 0.5f + copysignf(0.5f * e, z) + z * E * 0.3989422804014327f;
    }
    case UHC_ACT_TANH: { const float th = tanhf(z); return 1.0f - th * th; }
    case UHC_ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case UHC_ACT_SIGMOID: { const float sg = 1.0f / (1.0f + __expf(-z)); return sg * (1.0f - sg); }
    }
    return 1.f;
}
// one warp writes its 32 x 32 block (thread = row, vals = that row's 32 columns) to dst[row0 + rr][col0 + lane], rows in order
__device__ __forceinline__ void stage_store(float *stg, float *__restrict__ dst, const float (&vals)[32], int row0, int col0, int M, int N, int lane, bool atomic) {
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 32; ++j) stg[lane * 33 + j] = vals[j];
    __syncwarp();
    const int n = col0 + lane;
    if (n < N) {
#pragma unroll 8
        for (int rr = 0; rr < 32; ++rr) {
            const int grow = row0 + rr;
            if (grow < M) {
                const float x = stg[rr * 33 + lane];
                if (atomic) atomicAdd(dst + (size_t)grow * N + n, x); else dst[(size_t)grow * N + n] = x;
            }
        }
    }
}

// this lane's 32 accumulator values of row lr, columns c0 .. c0 + 31, from the hand-off tile
__device__ __forceinline__ void load_acc_row(const float *acc_s, int lr, int c0, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 t = *reinterpret_cast<const float4 *>(acc_s + lr * ACC_LD + c0 + 4 * j);
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
}

// DACT =the backward pass' dX GEMM with the activation backward fused into its epilogue: the accumulator (dh of the previous layer) is multiplied by act'(z_prev)
// (z tile fetched by TMA through mapZ) and leaves as bf16 dz (mapYb), its transpose (mapYT) and 32-row partial column sums added to dbias (the bias gradient);
// no fp32 dh is ever written.
template <bool DACT>
__global__ void __launch_bounds__(NTHREADS, 1)
k_linear_tc(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const float *__restrict__ bias,
            __nv_bfloat16 *__restrict__ ybf, float *__restrict__ yf, float *__restrict__ zf, int M, int N, int Kp, int ldy, int act, int ksplit,
            const __grid_constant__ CUtensorMap mapZ, const __grid_constant__ CUtensorMap mapYf, const __grid_constant__ CUtensorMap mapYb, int tma_mask,
            const __grid_constant__ CUtensorMap mapYT, float *__restrict__ dbias) {
    // tma_mask: bit 0 = zf, bit 1 = yf, bit 2 = ybf leave through their tensor map (32 x 32 boxes from swizzled staging tiles) instead of per-thread stores;
    // bit 3 = the TRANSPOSE of the bf16 activation ([N][M pitch], what the backward pass' dW = dz^T h GEMM reads as its K-major operand) is emitted as well
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = (uint64_t *)(smem + STAGES * STAGE_BYTES);   // full[STAGES], empty[STAGES]
    uint64_t *zbars = bars + 16;                                   // DACT: one barrier per epilogue warp for its z tiles
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    // split-K (gridDim.z slices of the reduction, partial tiles added into the zeroed yf): used for dW = dZ^T X whose output has few tiles
    const int nkb_all = Kp / BK, kb0 = (int)(((long)nkb_all * blockIdx.z) / ksplit), nkb = (int)(((long)nkb_all * (blockIdx.z + 1)) / ksplit) - kb0;
    const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA));
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB));
        for (int s = 0; s < STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }     // empty: one arrive per consumer warp
        if (DACT) for (int w = 0; w < 8; w++) mbar_init(smem_u32(zbars + w), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % STAGES; const uint32_t ph = (kb / STAGES) & 1;
                mbar_wait(empty0 + 8 * s, ph ^ 1);
                mbar_expect_tx(full0 + 8 * s, STAGE_BYTES);
                const uint32_t a = smem_u32(smem + s * STAGE_BYTES), b = a + BM * BK * 2;
                tma_load_2d(a, &mapA, full0 + 8 * s, (kb0 + kb) * BK, m0);
                tma_load_2d(b, &mapB, full0 + 8 * s, (kb0 + kb) * BK, n0);
            }
        }
    } else {
        const int g = warp >> 2, wl = warp & 3;          // consumer warpgroup (rows 64 g .. 64 g + 63 of the tile), warp within it
        {
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % STAGES; const uint32_t ph = (kb / STAGES) & 1;
                mbar_wait(full0 + 8 * s, ph);
                const uint32_t a = smem_u32(smem + s * STAGE_BYTES) + g * 64 * BK * 2, b = smem_u32(smem + s * STAGE_BYTES) + BM * BK * 2;
                const uint64_t ad = make_desc(a), bd = make_desc(b);
                fence_acc(acc);
                asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
                for (int k = 0; k < BK / UK; ++k) wgmma_m64n128k16(acc, ad + (uint64_t)(k * UK * 2 >> 4), bd + (uint64_t)(k * UK * 2 >> 4), (kb | k) != 0);
                asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");      // the previous k-block's MMAs have retired: its stage is free
                fence_acc(acc);
                if (kb > 0 && lane == 0) mbar_arrive(empty0 + 8 * ((kb - 1) % STAGES));
            }
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            fence_acc(acc);
            asm volatile("bar.sync 1, 256;" ::: "memory");       // both warpgroups are done with the operand ring: it now holds the epilogue staging
            float *acc_s = reinterpret_cast<float *>(smem + ACC_OFF) + g * 64 * ACC_LD;
            const int fr = 16 * wl + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                *reinterpret_cast<float2 *>(acc_s + fr * ACC_LD + 8 * j + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2 *>(acc_s + (fr + 8) * ACC_LD + 8 * j + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
            asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");     // the warpgroup's 64 rows are in the hand-off tile
        }
        // epilogue layout: warp = 32 rows (q = which 32 of the tile's 128) x 64 columns (half); its rows are rows lr0 .. lr0 + 31 of its warpgroup's tile
        const int q = 2 * g + (wl & 1), half = wl >> 1, lr = 32 * (wl & 1) + lane;
        const float *acc_s = reinterpret_cast<const float *>(smem + ACC_OFF) + g * 64 * ACC_LD;
        const int row = m0 + 32 * q + lane;
        if constexpr (DACT) {
            uint8_t *blk = smem + warp * EPI_BLOCK;
            const uint32_t blk_s = smem_u32(blk), zbar = smem_u32(zbars + warp);
            const int r0 = m0 + 32 * q, cfirst = half * (BN / 64);
            static_assert(BN / 64 == 2, "the z tiles of a warp's two chunks live in the two fp32 staging areas");
            const bool zl0 = r0 < M && n0 + cfirst * 32 < N, zl1 = r0 < M && n0 + cfirst * 32 + 32 < N;
            if (lane == 0 && zl0) {      // the operand ring is idle now: fetch this warp's z tiles while the accumulator is read from TMEM
                mbar_expect_tx(zbar, (zl1 ? 2u : 1u) * 4096u);
                tma_load_2d(blk_s + EPI_F32_A, &mapZ, zbar, n0 + cfirst * 32, r0);
                if (zl1) tma_load_2d(blk_s + EPI_F32_B, &mapZ, zbar, n0 + cfirst * 32 + 32, r0);
            }
#pragma unroll 1
            for (int cc = 0; cc < 2; ++cc) {
                float v[32];
                const int c = cfirst + cc, nb = n0 + c * 32;
                load_acc_row(acc_s, lr, c * 32, v);
                if (cc == 0 && zl0) mbar_wait(zbar, 0);
                if (cc == 1 && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");      // the bf16 tile of the first chunk has been read
                __syncwarp();
                const uint32_t zarea = blk_s + (cc ? EPI_F32_B : EPI_F32_A);
                if (cc ? zl1 : zl0) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {        // this thread's row of the 128B-swizzled z tile
                        float a, b, cq, d;
                        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(a), "=f"(b), "=f"(cq), "=f"(d) : "r"(zarea + lane * 128 + ((j ^ (lane & 7)) << 4)) : "memory");
                        v[4 * j] *= act_b_fast(a, act); v[4 * j + 1] *= act_b_fast(b, act); v[4 * j + 2] *= act_b_fast(cq, act); v[4 * j + 3] *= act_b_fast(d, act);
                    }
                }
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = (row < M && nb + j < N) ? v[j] : 0.f;
                __syncwarp();                             // every lane has read its z row: the area now stages the transposed tile
                if (nb < ldy) stage_row_bf16_sw64(blk_s + EPI_BF16, lane, v);
                if (nb < N) stage_col_bf16_sw64(zarea, lane, v);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) {
                    if (nb < ldy) tma_store_2d(&mapYb, blk_s + EPI_BF16, nb, r0);
                    if (nb < N) tma_store_2d(&mapYT, zarea, r0, nb);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                if (dbias && nb < N) {                    // column sums over the warp's 32 rows: transpose-reduce (31 shuffles), lane l ends with column l
#pragma unroll
                    for (int o = 16; o >= 1; o >>= 1) {
                        const bool up = (lane & o) != 0;
#pragma unroll
                        for (int k = 0; k < o; ++k) {
                            const float send = up ? v[k] : v[k + o], keep = up ? v[k + o] : v[k];
                            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                        }
                    }
                    if (nb + lane < N) atomicAdd(dbias + nb + lane, v[0]);
                }
            }
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the staging tiles have been read (the writes drain after the CTA)
        } else {
#pragma unroll 1
        for (int c = half * (BN / 64); c < (half + 1) * (BN / 64); ++c) {
            float v[32];
            load_acc_row(acc_s, lr, c * 32, v);
            // every output of this 32 x 32 chunk is staged in the warp's block of the (now idle) operand ring.  Where the output's row pitch allows a tensor map
            // (tma_mask) the tile is written in the map's swizzled layout and ONE elected lane hands it to the TMA engine (bounds are clipped by the hardware);
            // otherwise fp32 goes through a 32 x 33 tile so that every store instruction writes one full 128-byte row segment, bf16 as 16-byte stores of the row.
            const int nb = n0 + c * 32;
            uint8_t *blk = smem + warp * EPI_BLOCK;
            float *stg = reinterpret_cast<float *>(blk);                      // legacy 32 x 33 tile over the two fp32 areas
            float *sbias = reinterpret_cast<float *>(blk + EPI_BIAS);
            const uint32_t blk_s = smem_u32(blk);
            if (tma_mask) { if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }      // the previous chunk's tiles have been read
            __syncwarp();
            sbias[lane] = (bias && blockIdx.z == 0 && nb + lane < N) ? __ldg(bias + nb + lane) : 0.f;   // this chunk's 32 biases, read back as broadcasts
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = (row < M && nb + j < N) ? v[j] + sbias[j] : 0.f;
            if (zf) {                                                            // pre-activation (for the backward pass)
                if (tma_mask & 1) stage_row_f32_sw128(blk_s + EPI_F32_A, lane, v);
                else stage_store(stg, zf, v, m0 + 32 * q, nb, M, N, lane, false);
            }
            if (act == UHC_ACT_GELU) {        // act(0) = 0 for every supported activation except sigmoid, so padded entries stay 0
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = gelu_fast(v[j]);
            } else if (act != UHC_ACT_NONE) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = (row < M && nb + j < N) ? act_f(v[j], act) : 0.f;
            }
            if (yf) {
                if (tma_mask & 2) stage_row_f32_sw128(blk_s + EPI_F32_B, lane, v);
                else stage_store(stg, yf, v, m0 + 32 * q, nb, M, N, lane, ksplit > 1);
            }
            if ((tma_mask & 8) && nb < N) stage_col_bf16_sw64(blk_s + EPI_F32_B, lane, v);     // (the second fp32 area is free: a transposed copy is only asked for next to a bf16 y)
            if (ybf && nb < ldy) {
                if (tma_mask & 4) stage_row_bf16_sw64(blk_s + EPI_BF16, lane, v);
                else if (row < M) {
                    if (nb + 32 <= ldy) {
                        uint4 *dst = (uint4 *)(ybf + (size_t)row * ldy + nb);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            __nv_bfloat162 p0 = __floats2bfloat162_rn(v[8 * j], v[8 * j + 1]), p1 = __floats2bfloat162_rn(v[8 * j + 2], v[8 * j + 3]);
                            __nv_bfloat162 p2 = __floats2bfloat162_rn(v[8 * j + 4], v[8 * j + 5]), p3 = __floats2bfloat162_rn(v[8 * j + 6], v[8 * j + 7]);
                            uint4 u; u.x = *(uint32_t *)&p0; u.y = *(uint32_t *)&p1; u.z = *(uint32_t *)&p2; u.w = *(uint32_t *)&p3;
                            dst[j] = u;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (nb + j < ldy) ybf[(size_t)row * ldy + nb + j] = __float2bfloat16_rn(v[j]);      // (static indices: v stays in registers)
                    }
                }
            }
            if (tma_mask) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // this lane's tile rows -> visible to the async proxy
                __syncwarp();
                if (lane == 0) {
                    const int r0 = m0 + 32 * q;
                    if (zf && (tma_mask & 1)) tma_store_2d(&mapZ, blk_s + EPI_F32_A, nb, r0);
                    if (yf && (tma_mask & 2)) { if (ksplit > 1) tma_reduce_add_2d(&mapYf, blk_s + EPI_F32_B, nb, r0); else tma_store_2d(&mapYf, blk_s + EPI_F32_B, nb, r0); }
                    if (ybf && (tma_mask & 4) && nb < ldy) tma_store_2d(&mapYb, blk_s + EPI_BF16, nb, r0);
                    if ((tma_mask & 8) && nb < N) tma_store_2d(&mapYT, blk_s + EPI_F32_B, r0, nb);          // box = 32 rows (n) x 32 m-values
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (tma_mask && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the staging tiles have been read before the CTA's shared memory goes away (the global writes drain on their own)
        }
    }
}

// Grouped forward: G weight sets in one launch (the policy forward of several checkpoints side by side, eval.cu).  Row tile blockIdx.y
// belongs to one group (group_core.h): it loads 128 rows of x from the group's first row on, multiplies them by that group's weights
// (its tensor map in ga.mapB) and stores only the group's rows.  Main loop and epilogue arithmetic are k_linear_tc's without split-K, so
// a row's output is bit-identical to uhc_linear_forward_tc on that row; the outputs leave through per-thread stores bounded by the group.
struct GroupedArgs {
    CUtensorMap mapB[uhc::grp::MAX_GROUPS];
    const float *bias[uhc::grp::MAX_GROUPS];
    uhc::grp::TilePlan plan;
};
static_assert(sizeof(GroupedArgs) + sizeof(CUtensorMap) + 64 <= 32764, "the grouped kernel's parameters must fit the 32 KB parameter space");

__global__ void __launch_bounds__(NTHREADS, 1)
k_linear_tc_grouped(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ GroupedArgs ga, __nv_bfloat16 *__restrict__ ybf, float *__restrict__ yf,
                    int N, int Kp, int ldy, int act) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = (uint64_t *)(smem + STAGES * STAGE_BYTES);   // full[STAGES], empty[STAGES]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int m0, row_end;
    const int grp = uhc::grp::tile_rows(ga.plan, blockIdx.y, &m0, &row_end);
    const int n0 = blockIdx.x * BN, nkb = Kp / BK;
    const CUtensorMap *mapB = &ga.mapB[grp];
    const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA));
        asm volatile("prefetch.tensormap [%0];" ::"l"(mapB));
        for (int s = 0; s < STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % STAGES; const uint32_t ph = (kb / STAGES) & 1;
                mbar_wait(empty0 + 8 * s, ph ^ 1);
                mbar_expect_tx(full0 + 8 * s, STAGE_BYTES);
                const uint32_t a = smem_u32(smem + s * STAGE_BYTES), b = a + BM * BK * 2;
                tma_load_2d(a, &mapA, full0 + 8 * s, kb * BK, m0);       // rows past M read as zeros; rows of a later group are loaded, never stored
                tma_load_2d(b, mapB, full0 + 8 * s, kb * BK, n0);
            }
        }
        return;
    }
    const int g = warp >> 2, wl = warp & 3;
    {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < nkb; ++kb) {
            const int s = kb % STAGES; const uint32_t ph = (kb / STAGES) & 1;
            mbar_wait(full0 + 8 * s, ph);
            const uint32_t a = smem_u32(smem + s * STAGE_BYTES) + g * 64 * BK * 2, b = smem_u32(smem + s * STAGE_BYTES) + BM * BK * 2;
            const uint64_t ad = make_desc(a), bd = make_desc(b);
            fence_acc(acc);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int k = 0; k < BK / UK; ++k) wgmma_m64n128k16(acc, ad + (uint64_t)(k * UK * 2 >> 4), bd + (uint64_t)(k * UK * 2 >> 4), (kb | k) != 0);
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            fence_acc(acc);
            if (kb > 0 && lane == 0) mbar_arrive(empty0 + 8 * ((kb - 1) % STAGES));
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        fence_acc(acc);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        float *acc_s = reinterpret_cast<float *>(smem + ACC_OFF) + g * 64 * ACC_LD;
        const int fr = 16 * wl + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<float2 *>(acc_s + fr * ACC_LD + 8 * j + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2 *>(acc_s + (fr + 8) * ACC_LD + 8 * j + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
    }
    const int q = 2 * g + (wl & 1), half = wl >> 1, lr = 32 * (wl & 1) + lane;
    const float *acc_s = reinterpret_cast<const float *>(smem + ACC_OFF) + g * 64 * ACC_LD;
    const int row = m0 + 32 * q + lane;
    const float *bias = ga.bias[grp];
    uint8_t *blk = smem + warp * EPI_BLOCK;
    float *stg = reinterpret_cast<float *>(blk);
    float *sbias = reinterpret_cast<float *>(blk + EPI_BIAS);
#pragma unroll 1
    for (int c = half * (BN / 64); c < (half + 1) * (BN / 64); ++c) {
        float v[32];
        load_acc_row(acc_s, lr, c * 32, v);
        const int nb = n0 + c * 32;
        __syncwarp();
        sbias[lane] = (bias && nb + lane < N) ? __ldg(bias + nb + lane) : 0.f;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = (row < row_end && nb + j < N) ? v[j] + sbias[j] : 0.f;
        if (act == UHC_ACT_GELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = gelu_fast(v[j]);
        } else if (act != UHC_ACT_NONE) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = (row < row_end && nb + j < N) ? act_f(v[j], act) : 0.f;
        }
        if (yf) stage_store(stg, yf, v, m0 + 32 * q, nb, row_end, N, lane, false);
        if (ybf && nb < ldy && row < row_end) {       // ldy is a multiple of 8 and nb of 32: a chunk below ldy is whole or ends at ldy
            if (nb + 32 <= ldy) {
                uint4 *dst = (uint4 *)(ybf + (size_t)row * ldy + nb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    __nv_bfloat162 p0 = __floats2bfloat162_rn(v[8 * j], v[8 * j + 1]), p1 = __floats2bfloat162_rn(v[8 * j + 2], v[8 * j + 3]);
                    __nv_bfloat162 p2 = __floats2bfloat162_rn(v[8 * j + 4], v[8 * j + 5]), p3 = __floats2bfloat162_rn(v[8 * j + 6], v[8 * j + 7]);
                    uint4 u; u.x = *(uint32_t *)&p0; u.y = *(uint32_t *)&p1; u.z = *(uint32_t *)&p2; u.w = *(uint32_t *)&p3;
                    dst[j] = u;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (nb + j < ldy) ybf[(size_t)row * ldy + nb + j] = __float2bfloat16_rn(v[j]);
            }
        }
    }
}

__global__ void k_f32_to_bf16_padded(const float *__restrict__ x, __nv_bfloat16 *__restrict__ y, int M, int K, int Kp) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)M * Kp; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % Kp); const size_t r = i / Kp;
        y[i] = __float2bfloat16_rn(k < K ? x[r * K + k] : 0.f);
    }
}


// d/dz gelu(z) = Phi(z) + z phi(z), Phi through the same A&S erf as gelu_fast (shares the exp)
__device__ __forceinline__ float dgelu_fast(float z) {
    const float x = fabsf(z) * 0.70710678118654752f;
    const float t = __fdividef(1.0f, fmaf(0.3275911f, x, 1.0f));
    const float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
    const float ex = __expf(-x * x);                       // exp(-z^2 / 2)
    const float e = 1.0f - poly * ex;                      // erf(|z| / sqrt 2)
    return 0.5f + copysignf(0.5f * e, z) + z * 0.3989422804014327f * ex;
}
__device__ __forceinline__ float act_b(float z, int act) {
    switch (act) {
    case UHC_ACT_GELU: return dgelu_fast(z);
    case UHC_ACT_TANH: { float t = tanhf(z); return 1.0f - t * t; }
    case UHC_ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case UHC_ACT_SIGMOID: { float s = 1.0f / (1.0f + expf(-z)); return s * (1.0f - s); }
    }
    return 1.f;
}
// out[c][r] = in[r][c]  (bf16, 64x64 tiles through shared memory); rows r >= R of `in` read as zero so out is zero padded to ld_out
__global__ void k_transpose_bf16(const __nv_bfloat16 *__restrict__ in, __nv_bfloat16 *__restrict__ out, int R, int Cc, int ld_in, int ld_out) {
    __shared__ __nv_bfloat16 t[64][66];
    const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64;
    for (int i = threadIdx.y; i < 64; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        t[i][threadIdx.x] = (r < R && c < Cc) ? in[(size_t)r * ld_in + c] : __float2bfloat16_rn(0.f);
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 64; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (c < Cc && r < ld_out) out[(size_t)c * ld_out + r] = t[threadIdx.x][i];
    }
}
// vectorised variants (4 elements per thread along the contiguous dimension, all loads of a thread issued before use): used when the
// row lengths are multiples of 4
__device__ __forceinline__ uint2 pack_bf16x4(float a, float b, float c, float d) {
    __nv_bfloat162 p0 = __floats2bfloat162_rn(a, b), p1 = __floats2bfloat162_rn(c, d);
    uint2 u; u.x = *(uint32_t *)&p0; u.y = *(uint32_t *)&p1; return u;
}
__global__ void __launch_bounds__(256) k_transpose_bf16_v4(const __nv_bfloat16 *__restrict__ in, __nv_bfloat16 *__restrict__ out, int R, int Cc, int ld_in, int ld_out) {
    __shared__ float t[64][65];
    const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    uint2 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = r0 + ty + 16 * k, c = c0 + 4 * tx;
        v[k] = (r < R && c < Cc) ? *reinterpret_cast<const uint2 *>(in + (size_t)r * ld_in + c) : make_uint2(0u, 0u);   // Cc % 4 == 0: a group is all in or all out
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const __nv_bfloat162 a = *(__nv_bfloat162 *)&v[k].x, b = *(__nv_bfloat162 *)&v[k].y;
        float *row = t[ty + 16 * k] + 4 * tx;
        row[0] = __low2float(a); row[1] = __high2float(a); row[2] = __low2float(b); row[3] = __high2float(b);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + ty + 16 * k, r = r0 + 4 * tx;
        if (c < Cc && r < ld_out)
            *reinterpret_cast<uint2 *>(out + (size_t)c * ld_out + r) = pack_bf16x4(t[4 * tx][ty + 16 * k], t[4 * tx + 1][ty + 16 * k], t[4 * tx + 2][ty + 16 * k], t[4 * tx + 3][ty + 16 * k]);
    }
}
__global__ void __launch_bounds__(256) k_dact_bf16_v4(const float *__restrict__ dh, const float *__restrict__ z, __nv_bfloat16 *__restrict__ dz, __nv_bfloat16 *__restrict__ dzT,
                                                     float *__restrict__ db, int M, int N, int ld_dz, int ld_dzT, int act) {
    __shared__ float t[64][65];
    __shared__ float cs[64];
    const int n0 = blockIdx.x * 64, m0 = blockIdx.y * 64, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    if (threadIdx.x < 64) cs[threadIdx.x] = 0.f;
    float4 g[4], zz[4];
    const int n = n0 + 4 * tx;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int m = m0 + ty + 16 * k;
        const bool in = m < M && n < N;
        g[k] = in ? *reinterpret_cast<const float4 *>(dh + (size_t)m * N + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        zz[k] = (in && z) ? *reinterpret_cast<const float4 *>(z + (size_t)m * N + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int m = m0 + ty + 16 * k;
        float4 v = g[k];
        if (z) { v.x *= act_b(zz[k].x, act); v.y *= act_b(zz[k].y, act); v.z *= act_b(zz[k].z, act); v.w *= act_b(zz[k].w, act); }
        float *row = t[ty + 16 * k] + 4 * tx;
        row[0] = v.x; row[1] = v.y; row[2] = v.z; row[3] = v.w;
        c0 += v.x; c1 += v.y; c2 += v.z; c3 += v.w;
        if (dz && m < M && n < ld_dz) *reinterpret_cast<uint2 *>(dz + (size_t)m * ld_dz + n) = pack_bf16x4(v.x, v.y, v.z, v.w);
    }
    if (db) { atomicAdd(&cs[4 * tx], c0); atomicAdd(&cs[4 * tx + 1], c1); atomicAdd(&cs[4 * tx + 2], c2); atomicAdd(&cs[4 * tx + 3], c3); }
    __syncthreads();
    if (db && threadIdx.x < 64 && n0 + threadIdx.x < N) atomicAdd(db + n0 + threadIdx.x, cs[threadIdx.x]);
    if (dzT) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int nn = n0 + ty + 16 * k, m = m0 + 4 * tx;
            if (nn < N && m < ld_dzT)
                *reinterpret_cast<uint2 *>(dzT + (size_t)nn * ld_dzT + m) = pack_bf16x4(t[4 * tx][ty + 16 * k], t[4 * tx + 1][ty + 16 * k], t[4 * tx + 2][ty + 16 * k], t[4 * tx + 3][ty + 16 * k]);
        }
    }
}
// dz = dh * act'(z): writes dz (bf16, [M][ld_dz]) and its transpose ([N][ld_dzT], zero padded in M) and accumulates column sums (bias grads)
__global__ void k_dact_bf16(const float *__restrict__ dh, const float *__restrict__ z, __nv_bfloat16 *__restrict__ dz, __nv_bfloat16 *__restrict__ dzT,
                            float *__restrict__ db, int M, int N, int ld_dz, int ld_dzT, int act) {
    __shared__ float t[64][65];
    const int n0 = blockIdx.x * 64, m0 = blockIdx.y * 64;
    float colsum = 0.f;
    for (int i = threadIdx.y; i < 64; i += 8) {
        const int m = m0 + i, n = n0 + threadIdx.x;
        float v = 0.f;
        if (m < M && n < N) { v = dh[(size_t)m * N + n]; if (z) v *= act_b(z[(size_t)m * N + n], act); }
        t[i][threadIdx.x] = v;
        colsum += v;
        if (dz && m < M && n < ld_dz) dz[(size_t)m * ld_dz + n] = __float2bfloat16_rn(v);
    }
    if (db && n0 + threadIdx.x < N) atomicAdd(db + n0 + threadIdx.x, colsum);
    __syncthreads();
    if (dzT) for (int i = threadIdx.y; i < 64; i += 8) {
        const int n = n0 + i, m = m0 + threadIdx.x;
        if (n < N && m < ld_dzT) dzT[(size_t)n * ld_dzT + m] = __float2bfloat16_rn(t[threadIdx.x][i]);
    }
}

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                             const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn get_encode() {
    static const EncodeFn fn = [] {       // a function-local static: initialised once even when threads make their first GEMM calls at once
        void *p = nullptr; cudaDriverEntryPointQueryResult q;
        return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess ? (EncodeFn)p : (EncodeFn) nullptr;
    }();
    return fn;
}
int make_map(CUtensorMap *m, const void *base, int rows, int Kp, int box_rows = BM) {  // row-major [rows][Kp] bf16, box 64 x 128, 128B swizzle
    EncodeFn enc = get_encode();
    if (!enc) { uhc_err() = "cuTensorMapEncodeTiled unavailable"; return -1; }
    cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)Kp * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows}, estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { uhc_err() = "cuTensorMapEncodeTiled failed: " + std::to_string((int)r); return -1; }
    return 0;
}
// output tensor map: row-major [rows][cols] with a row pitch of `pitch` bytes, 32 x 32 boxes; the staging tiles use the 128-byte (fp32) / 64-byte (bf16) swizzle
int make_map_out(CUtensorMap *m, const void *base, int rows, int cols, size_t pitch, bool bf16) {
    EncodeFn enc = get_encode();
    if (!enc) { uhc_err() = "cuTensorMapEncodeTiled unavailable"; return -1; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)pitch};
    cuuint32_t box[2] = {32, 32}, estr[2] = {1, 1};
    CUresult r = enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     bf16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { uhc_err() = "cuTensorMapEncodeTiled (output) failed: " + std::to_string((int)r); return -1; }
    return 0;
}
bool tma_store_enabled() {
    static const bool on = [] { const char *e = getenv("UHC_TC_TMA_STORE"); return e ? (e[0] != '0') : (UHC_TC_TMA_STORE != 0); }();
    return on;
}
int sm_count(int dev) { int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); return sms; }
// per device: the kernels' shared-memory attribute belongs to the function on the CURRENT device.  Atomic flags: host threads may make their
// first GEMM calls at once (one per rank of an in-process group); setting the attribute twice is harmless, a torn flag is not.
int set_smem_attr(int dev) {
    static std::atomic<bool> attr_set[64] = {};
    if (dev >= 0 && dev < 64 && attr_set[dev]) return 0;
    if (cudaFuncSetAttribute(k_linear_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(k_linear_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) { uhc_err() = "cudaFuncSetAttribute failed"; return -1; }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
    return 0;
}
}  // namespace

extern "C" {
int uhc_f32_to_bf16_padded(const float *x, void *y_bf16, int M, int K, int Kp, void *stream) {
    k_f32_to_bf16_padded<<<1056, 256, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16 *)y_bf16, M, K, Kp);
    CK(cudaGetLastError()); return 0;
}

static int linear_tc_impl(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16_or_null, float *y_f32_or_null, float *z_f32_or_null,
                          int M, int N, int Kp, int ldy_bf16, int act, void *stream, void *yT_bf16_or_null = nullptr, int ld_yT = 0, int ld_yf = 0) {
    if (ld_yf <= 0) ld_yf = N;      // row pitch of the fp32 y in floats (only a plain fp32 product through the TMA engine takes a pitch other than N)
    if (Kp % BK != 0 || M <= 0 || N <= 0) { uhc_err() = "uhc_linear_forward_tc: Kp must be a positive multiple of 64"; return -2; }
    if (y_bf16_or_null && (ldy_bf16 % 8 != 0)) { uhc_err() = "uhc_linear_forward_tc: ldy must be a multiple of 8"; return -2; }
    // the per-thread epilogue writes bf16 rows as 16-byte vectors, and a pitch below N would drop the columns past it
    if (y_bf16_or_null && ((uintptr_t)y_bf16_or_null & 15)) { uhc_err() = "uhc_linear_forward_tc: the bf16 y must be 16-byte aligned"; return -2; }
    if (y_bf16_or_null && ldy_bf16 < N) { uhc_err() = "uhc_linear_forward_tc: ldy must be >= N"; return -2; }
    int dev = 0; cudaGetDevice(&dev);
    if (set_smem_attr(dev)) return -1;
    CUtensorMap ma, mb;
    if (make_map(&ma, x_bf16, M, Kp, BM) || make_map(&mb, W_bf16, N, Kp, BN)) return -1;
    const int tiles = ((N + BN - 1) / BN) * ((M + BM - 1) / BM), nkb = Kp / BK;
    // a plain fp32 product with a long reduction (dW = dz^T h, few output tiles): the reduction is split into as many slices as fill the SMs evenly
    // (one CTA per SM), the partial tiles are added into the zeroed output
    int ksplit = 1;
    if (!y_bf16_or_null && !z_f32_or_null && !yT_bf16_or_null && act == UHC_ACT_NONE && y_f32_or_null && nkb >= 32) {
        const int sms = sm_count(dev);
        double best = 0.0;
        for (int c = 1; c <= 16 && c <= nkb / 8; ++c) {
            const int items = tiles * c; const double eff = (double)items / (double)(((items + sms - 1) / sms) * sms);
            if (eff > best + 0.02) { best = eff; ksplit = c; }
        }
    }
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, ksplit);
    // outputs through the TMA engine: a tensor map needs a 16-byte aligned base and row pitch.  The fp32 outputs share one staging decision (their legacy
    // 32 x 33 tile spans both fp32 areas of the warp's block); without a map split-K accumulates with fp32 atomics.
    CUtensorMap mz = ma, myf = ma, myb = ma;
    int tma_mask = 0;
    if (tma_store_enabled()) {
        auto ok = [](const void *p, size_t pitch) { return p && ((uintptr_t)p & 15) == 0 && pitch % 16 == 0; };
        const size_t pf = (size_t)N * sizeof(float), pb = (size_t)ldy_bf16 * 2;
        const bool f32_ok = (z_f32_or_null || y_f32_or_null) && (!z_f32_or_null || ok(z_f32_or_null, pf)) && (!y_f32_or_null || ok(y_f32_or_null, (size_t)ld_yf * sizeof(float)));
        if (f32_ok) {
            if (z_f32_or_null) { if (make_map_out(&mz, z_f32_or_null, M, N, pf, false)) return -1; tma_mask |= 1; }
            if (y_f32_or_null) { if (make_map_out(&myf, y_f32_or_null, M, N, (size_t)ld_yf * sizeof(float), false)) return -1; tma_mask |= 2; }
        }
        if (y_bf16_or_null && ok(y_bf16_or_null, pb)) { if (make_map_out(&myb, y_bf16_or_null, M, ldy_bf16, pb, true)) return -1; tma_mask |= 4; }
    }
    if (ld_yf != N && !(tma_mask & 2)) { uhc_err() = "uhc_linear_forward_tc_f32_pitched: a padded pitch needs the TMA store path and a 16-byte aligned output"; return -2; }
    if ((ksplit > 1 || ld_yf != N) && cudaMemsetAsync(y_f32_or_null, 0, (size_t)M * ld_yf * sizeof(float), (cudaStream_t)stream) != cudaSuccess) { uhc_err() = "memset failed"; return -1; }   // (a padded pitch: the padding columns read as zeros)
    CUtensorMap myt = ma;
    if (yT_bf16_or_null) {      // transposed activation [N][ld_yT] (ld_yT >= M rounded up to 64, the padding columns receive the tile's zero rows)
        if (!tma_store_enabled() || y_f32_or_null || ((uintptr_t)yT_bf16_or_null & 15) || ld_yT % 8 != 0 || ld_yT < M) { uhc_err() = "uhc_linear_forward_tc_train_t: the transposed output needs the TMA store path, no fp32 y, and a pitch >= M that is a multiple of 8"; return -2; }
        if (make_map_out(&myt, yT_bf16_or_null, N, ld_yT, (size_t)ld_yT * 2, true)) return -1;
        tma_mask |= 8;
    }
    k_linear_tc<false><<<grid, NTHREADS, SMEM_BYTES, (cudaStream_t)stream>>>(ma, mb, b, (__nv_bfloat16 *)y_bf16_or_null, y_f32_or_null, z_f32_or_null, M, N, Kp, ldy_bf16, act, ksplit,
                                                                            mz, myf, myb, tma_mask, myt, nullptr);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { uhc_err() = cudaGetErrorString(e); return -1; }
    return 0;
}

int uhc_linear_forward_tc(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16_or_null, float *y_f32_or_null, int M, int N, int Kp,
                          int ldy_bf16, int act, void *stream) {
    return linear_tc_impl(x_bf16, W_bf16, b, y_bf16_or_null, y_f32_or_null, nullptr, M, N, Kp, ldy_bf16, act, stream);
}
int uhc_linear_forward_tc_train(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16_or_null, float *y_f32_or_null, float *z_f32,
                                int M, int N, int Kp, int ldy_bf16, int act, void *stream) {
    return linear_tc_impl(x_bf16, W_bf16, b, y_bf16_or_null, y_f32_or_null, z_f32, M, N, Kp, ldy_bf16, act, stream);
}
/* training forward that also emits the transpose of the bf16 activation, yT [N][ld_yT] (zero padded to ld_yT): the K-major operand of the backward pass' dW GEMM,
 * written by the same epilogue through the TMA engine instead of by a separate transpose kernel */
int uhc_linear_forward_tc_train_t(const void *x_bf16, const void *W_bf16, const float *b, void *y_bf16, void *yT_bf16, int ld_yT, float *z_f32_or_null,
                                  int M, int N, int Kp, int ldy_bf16, int act, void *stream) {
    if (!y_bf16 || !yT_bf16) { uhc_err() = "uhc_linear_forward_tc_train_t: y and yT are required"; return -2; }
    return linear_tc_impl(x_bf16, W_bf16, b, y_bf16, nullptr, z_f32_or_null, M, N, Kp, ldy_bf16, act, stream, yT_bf16, ld_yT);
}
/* plain fp32 product y[M][ld_y] = x W^T with a row pitch ld_y >= N (floats, multiple of 4): lets an output whose own pitch no tensor map accepts (N % 4 != 0) be
 * computed through the TMA engine (split-K included) into a padded scratch.  Returns -2 when the arguments do not qualify (then use uhc_linear_forward_tc). */
int uhc_linear_forward_tc_f32_pitched(const void *x_bf16, const void *W_bf16, float *y_f32, int ld_y, int M, int N, int Kp, void *stream) {
    if (!y_f32 || ld_y < N || ld_y % 4 != 0 || ((uintptr_t)y_f32 & 15) || !tma_store_enabled()) { uhc_err() = "uhc_linear_forward_tc_f32_pitched: arguments not eligible"; return -2; }
    return linear_tc_impl(x_bf16, W_bf16, nullptr, nullptr, y_f32, nullptr, M, N, Kp, 0, UHC_ACT_NONE, stream, nullptr, 0, ld_y);
}
int uhc_tc_tma_store_enabled(void) { return tma_store_enabled() ? 1 : 0; }
/* G weight sets in one launch: rows [row0[g], row0[g] + rows[g]) of x are multiplied by W[g] (+ b[g]) and written to the same rows of y;
 * every other row of y is left as it was.  One launch per layer for several policies side by side (uhc_eval_run_groups). */
int uhc_linear_forward_tc_grouped(int G, const int *row0_host, const int *rows_host, const void *x_bf16, const void *const *W_bf16_host,
                                  const float *const *b_host_or_null, void *y_bf16_or_null, float *y_f32_or_null, int M, int N, int Kp, int ldy_bf16,
                                  int act, void *stream) {
    if (!x_bf16 || !W_bf16_host || (!y_bf16_or_null && !y_f32_or_null)) { uhc_err() = "uhc_linear_forward_tc_grouped: null argument"; return -2; }
    if (Kp % BK != 0 || Kp <= 0 || M <= 0 || N <= 0) { uhc_err() = "uhc_linear_forward_tc_grouped: M, N > 0 and Kp a positive multiple of 64"; return -2; }
    if (y_bf16_or_null && (ldy_bf16 % 8 != 0 || ldy_bf16 < N)) { uhc_err() = "uhc_linear_forward_tc_grouped: ldy must be a multiple of 8 and >= N"; return -2; }
    if (y_bf16_or_null && ((uintptr_t)y_bf16_or_null & 15)) { uhc_err() = "uhc_linear_forward_tc_grouped: the bf16 y must be 16-byte aligned"; return -2; }
    GroupedArgs ga;
    memset(&ga, 0, sizeof ga);
    if (uhc::grp::plan_tiles(G, row0_host, rows_host, M, &ga.plan)) {
        uhc_err() = "uhc_linear_forward_tc_grouped: groups must be 1..64 ascending, disjoint, non-empty row ranges inside [0, M)"; return -2;
    }
    for (int g = 0; g < G; g++) if (!W_bf16_host[g]) { uhc_err() = "uhc_linear_forward_tc_grouped: null weights"; return -2; }
    int dev = 0; cudaGetDevice(&dev);
    static std::atomic<bool> attr_set[64] = {};
    if (!(dev >= 0 && dev < 64 && attr_set[dev])) {
        if (cudaFuncSetAttribute(k_linear_tc_grouped, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) { uhc_err() = "cudaFuncSetAttribute failed"; return -1; }
        if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    CUtensorMap ma;
    if (make_map(&ma, x_bf16, M, Kp, BM)) return -1;
    for (int g = 0; g < G; g++) {
        if (make_map(&ga.mapB[g], W_bf16_host[g], N, Kp, BN)) return -1;
        ga.bias[g] = b_host_or_null ? b_host_or_null[g] : nullptr;
    }
    dim3 grid((N + BN - 1) / BN, ga.plan.tile0[G], 1);
    k_linear_tc_grouped<<<grid, NTHREADS, SMEM_BYTES, (cudaStream_t)stream>>>(ma, ga, (__nv_bfloat16 *)y_bf16_or_null, y_f32_or_null, N, Kp, ldy_bf16, act);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { uhc_err() = cudaGetErrorString(e); return -1; }
    return 0;
}
/* backward through one Linear + the previous layer's activation in ONE kernel:  dz_prev = (dz W) * act'(z_prev)  as bf16 [M][ld_dz] and transposed [K][ld_dzT],
 * db_prev[k] += sum_m dz_prev[m][k].  dz [M][Np] and WT [K][Np] are the K-major bf16 operands (Np = N rounded up to 64).  Needs the TMA-store path, K % 4 == 0
 * and 16-byte aligned buffers (returns -2 otherwise: run uhc_linear_forward_tc + uhc_dact_bf16 instead). */
int uhc_linear_dx_dact_tc(const void *dz_bf16, const void *WT_bf16, const float *z_prev, void *dzp_bf16, void *dzpT_bf16, float *db_prev_or_null,
                          int M, int K, int Np, int ld_dz, int ld_dzT, int act, void *stream) {
    if (Np % BK != 0 || M <= 0 || K <= 0) { uhc_err() = "uhc_linear_dx_dact_tc: Np must be a positive multiple of 64"; return -2; }
    auto al = [](const void *p) { return p && ((uintptr_t)p & 15) == 0; };
    if (!tma_store_enabled() || K % 4 != 0 || ld_dz % 8 != 0 || ld_dzT % 8 != 0 || ld_dz < K || ld_dzT < M || !al(z_prev) || !al(dzp_bf16) || !al(dzpT_bf16)) {
        uhc_err() = "uhc_linear_dx_dact_tc: needs the TMA store path, K % 4 == 0, pitches that are multiples of 8 elements and 16-byte aligned buffers"; return -2;
    }
    int dev = 0; cudaGetDevice(&dev);
    if (set_smem_attr(dev)) return -1;
    CUtensorMap ma, mb, mz, mdz, mdzT;
    if (make_map(&ma, dz_bf16, M, Np, BM) || make_map(&mb, WT_bf16, K, Np, BN)) return -1;
    if (make_map_out(&mz, z_prev, M, K, (size_t)K * 4, false) || make_map_out(&mdz, dzp_bf16, M, ld_dz, (size_t)ld_dz * 2, true) ||
        make_map_out(&mdzT, dzpT_bf16, K, ld_dzT, (size_t)ld_dzT * 2, true)) return -1;
    if (db_prev_or_null && cudaMemsetAsync(db_prev_or_null, 0, (size_t)K * sizeof(float), (cudaStream_t)stream) != cudaSuccess) { uhc_err() = "uhc_linear_dx_dact_tc: memset failed"; return -1; }
    dim3 grid((K + BN - 1) / BN, (M + BM - 1) / BM, 1);
    k_linear_tc<true><<<grid, NTHREADS, SMEM_BYTES, (cudaStream_t)stream>>>(ma, mb, nullptr, nullptr, nullptr, nullptr, M, K, Np, ld_dz, act, 1, mz, mz, mdz, 0, mdzT, db_prev_or_null);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { uhc_err() = cudaGetErrorString(e); return -1; }
    return 0;
}
int uhc_transpose_bf16(const void *in, void *out, int R, int Cc, int ld_in, int ld_out, void *stream) {
    dim3 grid((Cc + 63) / 64, (R + 63) / 64);
    if (Cc % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0 && ((uintptr_t)in & 7) == 0 && ((uintptr_t)out & 7) == 0)
        k_transpose_bf16_v4<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)in, (__nv_bfloat16 *)out, R, Cc, ld_in, ld_out);
    else
        k_transpose_bf16<<<grid, dim3(64, 8), 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)in, (__nv_bfloat16 *)out, R, Cc, ld_in, ld_out);
    CK(cudaGetLastError()); return 0;
}
int uhc_dact_bf16(const float *dh, const float *z_or_null, void *dz_bf16, void *dzT_bf16, float *db_or_null, int M, int N, int ld_dz, int ld_dzT, int act,
                  void *stream) {
    if (db_or_null && cudaMemsetAsync(db_or_null, 0, N * sizeof(float), (cudaStream_t)stream) != cudaSuccess) { uhc_err() = "uhc_dact_bf16: memset failed"; return -1; }
    dim3 grid((N + 63) / 64, (M + 63) / 64);
    const bool v4 = N % 4 == 0 && (!dz_bf16 || (ld_dz % 4 == 0 && ((uintptr_t)dz_bf16 & 7) == 0)) && (!dzT_bf16 || (ld_dzT % 4 == 0 && ((uintptr_t)dzT_bf16 & 7) == 0)) &&
                    ((uintptr_t)dh & 15) == 0 && (!z_or_null || ((uintptr_t)z_or_null & 15) == 0);
    if (v4) k_dact_bf16_v4<<<grid, 256, 0, (cudaStream_t)stream>>>(dh, z_or_null, (__nv_bfloat16 *)dz_bf16, (__nv_bfloat16 *)dzT_bf16, db_or_null, M, N, ld_dz, ld_dzT, act);
    else k_dact_bf16<<<grid, dim3(64, 8), 0, (cudaStream_t)stream>>>(dh, z_or_null, (__nv_bfloat16 *)dz_bf16, (__nv_bfloat16 *)dzT_bf16, db_or_null, M, N, ld_dz, ld_dzT, act);
    CK(cudaGetLastError()); return 0;
}
}
