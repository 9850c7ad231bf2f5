// cz_net.cu -- hand-written sm_90a kernels for the two ends of the policy-value network
// (policy_value_network.py:45-74): the first convolution evaluated straight from board bytes, and the
// fused policy / value heads.  The batch-1024 residual tower in between stays on the library (cuDNN) path.
//
//   k_first_conv      : canonical board bytes -> conv3x3(14->128)+bias+ReLU output, fp16 NHWC [B][90][128].
//                       The 14-plane input is one-hot and <= 32 of its 1260 cells are set, so the convolution is a
//                       gather-add of weight rows: out[cell][:] = b + sum over the 3x3 neighbourhood of W[tap][piece][:].
//                       The [9][10][14] tensor (and the reference's rank*9+file indexing, main.py:550-555) is never
//                       materialised: image cell (r, f) reads canonical board byte r*9+f.
//   k_head_conv_mma   : conv1x1(128->3)+bias+ReLU (policy 2 ch + value 1 ch) as one streaming pass on mma.sync (hi+lo fp16
//                       weight split: fp32-weight accuracy); writes the policy features hp either row-major fp16 [B][192]
//                       (flatten order (h, w, c), zero padded) or directly as wgmma operand tiles.
//   k_value_mlp       : 90 -> 256 ReLU -> 1 tanh, 8 positions per CTA, all 90 weights of a hidden unit requested up front.
//   k_policy_fc_tc    : logits[B][2086] = hp . Wp^T + bp on wgmma; both operands arrive as 48 KB bulk async copies
//                       (cp.async.bulk) already in the operand layout; fp32 logits stored 128 B per warp and position.
//                       Batches of 128 rows or more (cz_net_heads_tc).
//   k_policy_fc       : the same on mma.sync m16n8k16 (smaller batches and the small-batch trunk, row-major hp).
//   k_epilogue_split  : the f32 epilogue of one convolution of the fp32-accurate plan (net.py: SplitTf32Plan) fused with the
//                       tf32 hi / lo operand split for the next one.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cchess_b200.h"
#include "cz_wgmma.cuh"

namespace {

using namespace cz_sm90;

// ------------------------------------------------------------------------------------------
// first convolution from board bytes: one CTA per position, a half-warp per output cell (128 channels, 8 per lane)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_first_conv(const uint8_t *__restrict__ boards, int B, const __half *__restrict__ w /* [9][14][128] */,
                                                     const float4 *__restrict__ bias /* [32] */, __half *__restrict__ out /* [B][90][128] */) {
    __shared__ uint8_t pb[11 * 12 + 12];   // zero-bordered image: pb[(r+1)*12 + f+1] = canonical board byte r*9+f (r < 9, f < 10)
    const int pos = blockIdx.x;
    const uint8_t *bd = boards + (size_t)pos * 96;
    if (threadIdx.x < 132) {
        const int r = threadIdx.x / 12 - 1, f = threadIdx.x % 12 - 1;
        pb[threadIdx.x] = (r >= 0 && r < 9 && f >= 0 && f < 10) ? bd[r * 9 + f] : (uint8_t)0;   // the reference's cell <- s[rank*9+file]
    }
    __syncthreads();
    const int hw = threadIdx.x >> 4, l16 = threadIdx.x & 15;   // 16 half-warps, lane owns channels 8*l16 .. 8*l16+7
    const float4 b0 = bias[l16 * 2], b1 = bias[l16 * 2 + 1];
    for (int cell = hw; cell < 90; cell += 16) {
        const int r = cell / 10, f = cell - r * 10;
        const uint8_t *c0 = pb + r * 12 + f;          // top-left of the 3x3 window
        int pc[9];
#pragma unroll
        for (int t = 0; t < 9; t++) pc[t] = c0[(t / 3) * 12 + (t % 3)];
        float acc[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int t = 0; t < 9; t++) {
            if (pc[t]) {
                const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(w + ((size_t)(t * 14 + pc[t] - 1) * 128 + l16 * 8)));
                const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float2 v = __half22float2(h2[k]);
                    acc[2 * k] += v.x;
                    acc[2 * k + 1] += v.y;
                }
            }
        }
        uint4 o;
        __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
        for (int k = 0; k < 4; k++) oh[k] = __floats2half2_rn(relu_nan(acc[2 * k]), relu_nan(acc[2 * k + 1]));
        *reinterpret_cast<uint4 *>(out + ((size_t)pos * 90 + cell) * 128 + l16 * 8) = o;
    }
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// heads, stage 2a: value MLP 90 -> 256 ReLU -> 1 tanh (policy_value_network.py:73-74), 8 positions per CTA.
// Thread t owns hidden unit t: its 90 first-layer weights are requested up front (90 independent coalesced loads, one L2 round trip
// instead of nine), the positions' features are broadcast from shared memory.
constexpr int VM_POS = 8;
__global__ void __launch_bounds__(256) k_value_mlp(const float *__restrict__ hv /* [B][96] */, int B, const float *__restrict__ w1t /* [90][256] */,
                                                    const float *__restrict__ b1, const float *__restrict__ w2, const float *__restrict__ b2, float *__restrict__ value) {
    __shared__ float sh[VM_POS][96];
    __shared__ float red[VM_POS][8];
    const int p0 = blockIdx.x * VM_POS, t = threadIdx.x, warp = t >> 5, lane = t & 31;
    float wv[90];
#pragma unroll
    for (int k = 0; k < 90; k++) wv[k] = __ldg(w1t + k * 256 + t);
    for (int i = t; i < VM_POS * 96; i += 256) {
        const int p = i / 96;
        sh[p][i - p * 96] = p0 + p < B ? hv[(size_t)(p0 + p) * 96 + (i - p * 96)] : 0.f;
    }
    const float bb = b1[t], w2v = w2[t];
    __syncthreads();
    float a[VM_POS];
#pragma unroll
    for (int p = 0; p < VM_POS; p++) a[p] = bb;
#pragma unroll
    for (int k = 0; k < 90; k++)
#pragma unroll
        for (int p = 0; p < VM_POS; p++) a[p] += wv[k] * sh[p][k];
#pragma unroll
    for (int p = 0; p < VM_POS; p++) {
        float s = relu_nan(a[p]) * w2v;
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[p][warp] = s;
    }
    __syncthreads();
    if (t < VM_POS && p0 + t < B) {
        float s = __ldg(b2);
#pragma unroll
        for (int wq = 0; wq < 8; wq++) s += red[t][wq];
        value[p0 + t] = tanhf(s);
    }
}

// ------------------------------------------------------------------------------------------
// heads, stage 1: conv1x1 (128 -> 3) + bias + ReLU as one streaming pass.
// A CTA (one position, 6 warps) stages its 90 x 128 fp16 cells in shared memory with cp.async (rows padded to 272 B: conflict-free
// ldmatrix), each warp multiplies its 16 cells with mma.sync m16n8k16 against the head weights held in registers as B fragments
// (N = 8: policy 2 + value 1 + 5 zero columns).  The f32 weights enter as hi + lo fp16 pairs (two MMAs per k-step), so the result
// equals the fp32-weight dot product to ~1e-7 relative: no precision is traded for the speed.  ~2 instructions per cell.
// ------------------------------------------------------------------------------------------
constexpr int HC_ROW = 136;   // halves per staged row (128 + 8 pad = 272 B)
// TILED: hp is written in the operand layout k_policy_fc_tc consumes: [position tile of 128][k-chunk 24][128 positions][8 halves].
template <bool TILED>
__global__ void __launch_bounds__(192) k_head_conv_mma(const __half *__restrict__ x /* [B][90][128] */, int B, const float *__restrict__ wh /* [3][128] */,
                                                        const float *__restrict__ bh /* [3] */, __half *__restrict__ hp /* [B][192] or tiled */,
                                                        float *__restrict__ hv /* [B][96] */) {
    __shared__ __align__(16) __half sx[96 * HC_ROW];
    const int pos = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const __half *src = x + (size_t)pos * 90 * 128;
    for (int i = tid; i < 96 * 16; i += 192) {                   // 16-byte chunks: row i / 16, chunk i % 16
        const int r = i >> 4, c = i & 15;
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(sx + r * HC_ROW + c * 8);
        if (r < 90) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + r * 128 + c * 8) : "memory");
        else *reinterpret_cast<uint4 *>(sx + r * HC_ROW + c * 8) = make_uint4(0, 0, 0, 0);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    // B fragments (col-major K x N): lane (g = lane >> 2 -> output n, t = lane & 3) holds k = 16*ks + 2t, 2t+1 and + 8
    const int g = lane >> 2, t = lane & 3;
    uint32_t bhi[8][2], blo[8][2];
#pragma unroll
    for (int ks = 0; ks < 8; ks++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int k = ks * 16 + h * 8 + t * 2;
            const float w0 = g < 3 ? __ldg(wh + g * 128 + k) : 0.f, w1 = g < 3 ? __ldg(wh + g * 128 + k + 1) : 0.f;
            const __half h0 = __float2half_rn(w0), h1 = __float2half_rn(w1);
            const __half l0 = __float2half_rn(w0 - __half2float(h0)), l1 = __float2half_rn(w1 - __half2float(h1));
            __half2 hh = __halves2half2(h0, h1), ll = __halves2half2(l0, l1);
            bhi[ks][h] = *reinterpret_cast<uint32_t *>(&hh);
            blo[ks][h] = *reinterpret_cast<uint32_t *>(&ll);
        }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int row0 = warp * 16;
    // ldmatrix.x4: lanes 0-15 address rows row0 + (lane & 15) at k-offset 0, lanes 16-31 the same rows at k-offset 8
    const uint32_t abase = (uint32_t)__cvta_generic_to_shared(sx + (row0 + (lane & 15)) * HC_ROW + (lane >> 4) * 8);
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
        uint32_t a[4];
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(abase + ks * 32));
        mma16816(acc, a, bhi[ks]);
        mma16816(acc, a, blo[ks]);
    }
    // accumulator layout: rows row0 + g and row0 + g + 8, columns 2t, 2t + 1
    const float b0 = bh[0], b1 = bh[1], b2 = bh[2];
#pragma unroll
    for (int hlf = 0; hlf < 2; hlf++) {
        const int cell = row0 + g + hlf * 8;
        if (cell < 90) {
            // flatten order of tf.reshape on NHWC (policy_value_network.py:62, 72): index = cell*2 + c
            if (t == 0) {
                const __half2 v = __floats2half2_rn(relu_nan(acc[hlf * 2] + b0), relu_nan(acc[hlf * 2 + 1] + b1));
                const int k = cell * 2;                              // feature index (even): chunk k / 8, offset k % 8
                if (TILED) *reinterpret_cast<__half2 *>(hp + ((size_t)(pos >> 7) * 24 + (k >> 3)) * 1024 + (size_t)(pos & 127) * 8 + (k & 7)) = v;
                else *reinterpret_cast<__half2 *>(hp + (size_t)pos * 192 + k) = v;
            }
            if (t == 1) hv[(size_t)pos * 96 + cell] = relu_nan(acc[hlf * 2] + b2);
        }
    }
    if (tid < 12) {                                                  // K padding of the policy GEMM (features 180..191)
        const int k = 180 + tid;
        if (TILED) hp[((size_t)(pos >> 7) * 24 + (k >> 3)) * 1024 + (size_t)(pos & 127) * 8 + (k & 7)] = __float2half(0.f);
        else hp[(size_t)pos * 192 + k] = __float2half(0.f);
    }
}

// ------------------------------------------------------------------------------------------
// heads, stage 2b on the Hopper tensor cores: logits[pos][label] = hp[pos] . wp[label] + bp[label]   (wgmma)
//   D[128 labels][128 positions] (f32) = A[128][192] . B[192][128]: A = a 128-label tile of the FC weights, B = a 128-position
//   tile of the head features, both already in the canonical K-major no-swizzle layout in global memory (weights: prepared once
//   on the host; features: written that way by k_head_conv_mma<true>), so each operand is ONE 48 KB bulk async copy
//   (cp.async.bulk) signalling an mbarrier.  Two warpgroups, one per 64-label half, each issue 12 wgmma m64n128k16; the tile is then
//   staged transposed in the (dead) operand buffers so that every warp stores 128 contiguous bytes of logits per position.
//   136 CTAs for 1024 positions x 2086 labels, one tile each.
// ------------------------------------------------------------------------------------------
constexpr int FC_TILE_BYTES = 24 * 128 * 16;   // 49 152 B per operand tile
constexpr int FC_OUT_ROW = 132;                // floats per staged position row: 128 labels + 4 pad (conflict-free fragment stores)
__global__ void __launch_bounds__(256) k_policy_fc_tc(const uint4 *__restrict__ hp_tiled, int B, const uint4 *__restrict__ wp_tiled,
                                                       const float *__restrict__ bp /* [>= 2176] */, float *__restrict__ logits /* [B][2086] */) {
    extern __shared__ __align__(128) unsigned char smem_fc_tc[];
    unsigned char *sA = smem_fc_tc, *sB = smem_fc_tc + FC_TILE_BYTES;
    float *sOut = reinterpret_cast<float *>(smem_fc_tc);            // [128 positions][FC_OUT_ROW], once the MMAs are done
    __shared__ __align__(8) uint64_t bar_ld;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int mt = blockIdx.y, nt = blockIdx.x;                     // label tile, position tile
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&bar_ld)), "r"(1u));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar_ld)), "r"(2u * FC_TILE_BYTES) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(sA)), "l"(reinterpret_cast<const unsigned char *>(wp_tiled) + (size_t)mt * FC_TILE_BYTES), "r"(FC_TILE_BYTES), "r"(smem_u32(&bar_ld)) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(sB)), "l"(reinterpret_cast<const unsigned char *>(hp_tiled) + (size_t)nt * FC_TILE_BYTES), "r"(FC_TILE_BYTES), "r"(smem_u32(&bar_ld)) : "memory");
    }
    {   // operands landed
        const uint32_t bar = smem_u32(&bar_ld);
        asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                     ::"r"(bar), "r"(0u) : "memory");
    }
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; i++) d[i] = 0.f;
    const uint64_t da = gmma_desc(smem_u32(sA) + (uint32_t)(wg * 64 * 16), 2048), db = gmma_desc(smem_u32(sB), 2048);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 12; ks++)                                 // two k-chunks per MMA
        Wgmma<128>::mma(d, da + (uint64_t)((ks * 4096) >> 4), db + (uint64_t)((ks * 4096) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(d);
    __syncthreads();                                                // both warpgroups are done reading the operands: they become sOut
    {   // fragment -> sOut[position][label]: lane holds labels lr, lr + 8 and positions 8j + 2(lane%4) + {0, 1}
        const int lr = wg * 64 + (warp & 3) * 16 + (lane >> 2), q = lane & 3;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int p = 8 * j + 2 * q;
            sOut[p * FC_OUT_ROW + lr] = d[4 * j];
            sOut[(p + 1) * FC_OUT_ROW + lr] = d[4 * j + 1];
            sOut[p * FC_OUT_ROW + lr + 8] = d[4 * j + 2];
            sOut[(p + 1) * FC_OUT_ROW + lr + 8] = d[4 * j + 3];
        }
    }
    __syncthreads();
    float bias[4];
    bool lab_ok[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int label = mt * 128 + 32 * k + lane;
        bias[k] = bp[label];
        lab_ok[k] = label < CZ_NLABEL;
    }
#pragma unroll 1
    for (int p = warp; p < 128; p += 8) {
        const int pos = nt * 128 + p;
        if (pos >= B) break;
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (lab_ok[k]) logits[(size_t)pos * CZ_NLABEL + mt * 128 + 32 * k + lane] = sOut[p * FC_OUT_ROW + 32 * k + lane] + bias[k];
    }
}

constexpr int NPAD = 2112;   // 33 * 64 >= 2086
constexpr int LDS_ROW = 200; // halves per staged row (192 + 8 pad): fragment loads hit 32 distinct banks

// ------------------------------------------------------------------------------------------
// heads, stage 2b for smaller batches: the policy FC on mma.sync m16n8k16 (0.77 GFLOP at 1024 positions, bound by its 8.5 MB f32 output)
// grid (ceil(B/64), 33), 128 threads.  A tile (64 positions x 192) and B tile (64 labels x 192) are staged through shared
// memory with 16-byte coalesced loads, all in flight at once; warp w owns rows [16w, 16w+16) x 64 columns.
__global__ void __launch_bounds__(128) k_policy_fc(const __half *__restrict__ hp /* [B][192] */, int B, const __half *__restrict__ wp /* [NPAD][192] */,
                                                    const float *__restrict__ bp /* [NPAD] */, float *__restrict__ logits /* [B][2086] */) {
    extern __shared__ __align__(16) __half smem_fc[];
    __half *sA = smem_fc, *sB = smem_fc + 64 * LDS_ROW;
    const int row0 = blockIdx.x * 64, col0 = blockIdx.y * 64;
    for (int i = threadIdx.x; i < 64 * 24; i += 128) {          // 24 x 16-byte chunks per 192-half row
        const int r = i / 24, c = i - r * 24;
        const int ra = min(row0 + r, B - 1);                     // clamp: rows >= B are computed but never stored
        *reinterpret_cast<uint4 *>(sA + r * LDS_ROW + c * 8) = __ldg(reinterpret_cast<const uint4 *>(hp + (size_t)ra * 192 + c * 8));
        *reinterpret_cast<uint4 *>(sB + r * LDS_ROW + c * 8) = __ldg(reinterpret_cast<const uint4 *>(wp + (size_t)(col0 + r) * 192 + c * 8));
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    float acc[8][4];
#pragma unroll
    for (int n = 0; n < 8; n++)
#pragma unroll
        for (int k = 0; k < 4; k++) acc[n][k] = 0.f;
    const uint32_t *A0 = reinterpret_cast<const uint32_t *>(sA + (warp * 16 + g) * LDS_ROW);
    const uint32_t *A1 = reinterpret_cast<const uint32_t *>(sA + (warp * 16 + g + 8) * LDS_ROW);
#pragma unroll
    for (int ks = 0; ks < 12; ks++) {
        uint32_t a[4];
        a[0] = A0[ks * 8 + t];
        a[1] = A1[ks * 8 + t];
        a[2] = A0[ks * 8 + 4 + t];
        a[3] = A1[ks * 8 + 4 + t];
#pragma unroll
        for (int n = 0; n < 8; n++) {
            const uint32_t *Bp = reinterpret_cast<const uint32_t *>(sB + (n * 8 + g) * LDS_ROW);
            uint32_t b[2];
            b[0] = Bp[ks * 8 + t];
            b[1] = Bp[ks * 8 + 4 + t];
            mma16816(acc[n], a, b);
        }
    }
    const int r0 = row0 + warp * 16 + g;
#pragma unroll
    for (int n = 0; n < 8; n++) {
        const int col = col0 + n * 8 + t * 2;
        if (col >= CZ_NLABEL) continue;
        const float b0 = bp[col], b1 = bp[col + 1];
        if (r0 < B) *reinterpret_cast<float2 *>(logits + (size_t)r0 * CZ_NLABEL + col) = make_float2(acc[n][0] + b0, acc[n][1] + b1);
        if (r0 + 8 < B) *reinterpret_cast<float2 *>(logits + (size_t)(r0 + 8) * CZ_NLABEL + col) = make_float2(acc[n][2] + b0, acc[n][3] + b1);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Operand split for the fp32-accurate inference mode (net.py: SplitTf32Plan).  y f32 [P][128] (NHWC activations of one convolution)
//   -> hi f32 [P][128] = tf32(y): rounded to the 10-bit TF32 mantissa (nearest, ties away; the low 13 bits are zero, so whatever
//      conversion the tensor-core kernel applies to it is the identity), and
//   -> x2 fp16 [P][256] = { (y - hi) * 2^11 | hi }: both halves have <= 11 significant bits, i.e. they are EXACT in fp16 (up to
//      fp16's range: |hi| <= 65504, residues below 2^-24 * 2^11 flush).
// A TF32 convolution hi(x) * hi(w) (K = 1152: the only long accumulation chain of full-size terms) plus an fp16 convolution
// x2 * { hi(w) | lo(w) * 2^11 } (the two cross terms, 2^-11 smaller, scaled back by 2^-11 in the epilogue) give the product to
// O(2^-22): dropped are lo*lo and the 11-bit rounding of the two lo operands.
__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xFFFFE000u); }
#define SPLIT_SCALE 2048.0f

// One pass per convolution: v = ReLU(t + 2^-11 s + bias [+ skip]) from the two library convolutions' raw results, then the split of v
// for the NEXT convolution.  t f32 [P][128] (hi*hi), s fp16 [P][128] or null (cross terms, scaled), skip f32 or null; outputs (each
// optional): x f32 (the value itself: next block's skip / the heads' input; may alias skip), hi f32, x2 fp16 [P][256] = { lo 2^11 | hi }.
// Streaming: 32-80 B in, 64-96 B out per thread (8 channels).
__global__ void __launch_bounds__(256) k_epilogue_split(const float4 *__restrict__ t, const uint4 *__restrict__ s, const float4 *__restrict__ bias,
                                                        const float4 *skip, float4 *x, float4 *__restrict__ hi, uint4 *__restrict__ x2, long long n8) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        float4 a = __ldg(t + 2 * i), b = __ldg(t + 2 * i + 1);
        if (s) {
            const uint4 sv = __ldg(s + i);
            const float2 s0 = __half22float2(*reinterpret_cast<const __half2 *>(&sv.x)), s1 = __half22float2(*reinterpret_cast<const __half2 *>(&sv.y));
            const float2 s2 = __half22float2(*reinterpret_cast<const __half2 *>(&sv.z)), s3 = __half22float2(*reinterpret_cast<const __half2 *>(&sv.w));
            const float r = 1.0f / SPLIT_SCALE;
            a.x += s0.x * r; a.y += s0.y * r; a.z += s1.x * r; a.w += s1.y * r;
            b.x += s2.x * r; b.y += s2.y * r; b.z += s3.x * r; b.w += s3.y * r;
        }
        const float4 ba = __ldg(bias + 2 * (i & 15)), bb = __ldg(bias + 2 * (i & 15) + 1);
        a.x += ba.x; a.y += ba.y; a.z += ba.z; a.w += ba.w;
        b.x += bb.x; b.y += bb.y; b.z += bb.z; b.w += bb.w;
        if (skip) {
            const float4 ka = skip[2 * i], kb = skip[2 * i + 1];
            a.x += ka.x; a.y += ka.y; a.z += ka.z; a.w += ka.w;
            b.x += kb.x; b.y += kb.y; b.z += kb.z; b.w += kb.w;
        }
        a.x = relu_nan(a.x); a.y = relu_nan(a.y); a.z = relu_nan(a.z); a.w = relu_nan(a.w);
        b.x = relu_nan(b.x); b.y = relu_nan(b.y); b.z = relu_nan(b.z); b.w = relu_nan(b.w);
        if (x) { x[2 * i] = a; x[2 * i + 1] = b; }
        if (!hi) continue;
        const float4 ha = make_float4(tf32_hi(a.x), tf32_hi(a.y), tf32_hi(a.z), tf32_hi(a.w));
        const float4 hb = make_float4(tf32_hi(b.x), tf32_hi(b.y), tf32_hi(b.z), tf32_hi(b.w));
        hi[2 * i] = ha; hi[2 * i + 1] = hb;
        uint4 l, h;
        *reinterpret_cast<__half2 *>(&l.x) = __floats2half2_rn((a.x - ha.x) * SPLIT_SCALE, (a.y - ha.y) * SPLIT_SCALE);
        *reinterpret_cast<__half2 *>(&l.y) = __floats2half2_rn((a.z - ha.z) * SPLIT_SCALE, (a.w - ha.w) * SPLIT_SCALE);
        *reinterpret_cast<__half2 *>(&l.z) = __floats2half2_rn((b.x - hb.x) * SPLIT_SCALE, (b.y - hb.y) * SPLIT_SCALE);
        *reinterpret_cast<__half2 *>(&l.w) = __floats2half2_rn((b.z - hb.z) * SPLIT_SCALE, (b.w - hb.w) * SPLIT_SCALE);
        *reinterpret_cast<__half2 *>(&h.x) = __floats2half2_rn(ha.x, ha.y);
        *reinterpret_cast<__half2 *>(&h.y) = __floats2half2_rn(ha.z, ha.w);
        *reinterpret_cast<__half2 *>(&h.z) = __floats2half2_rn(hb.x, hb.y);
        *reinterpret_cast<__half2 *>(&h.w) = __floats2half2_rn(hb.z, hb.w);
        uint4 *o = x2 + (i >> 4) * 32 + (i & 15);
        o[0] = l; o[16] = h;
    }
}

// The value MLP and the policy FC are independent: fork the value MLP onto a side stream (event fork/join, which CUDA-graph
// capture records as two parallel branches) so that the two small kernels overlap.  launch_policy_fc(st) launches the policy FC
// on the caller's stream between the fork and the join.  The side stream and its events are created on the first (eager,
// warm-up) call of either heads entry point, never during capture.
template <class LaunchPolicyFc>
int value_mlp_beside(cudaStream_t st, const float *hv, int B, const float *w1t, const float *b1, const float *w2, const float *b2, float *value,
                     LaunchPolicyFc launch_policy_fc) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return CZ_ECUDA;
    static cudaStream_t side[64] = {nullptr};
    static cudaEvent_t ev_fork[64] = {nullptr}, ev_join[64] = {nullptr};
    if (!side[dev]) {
        if (cudaStreamCreateWithFlags(&side[dev], cudaStreamNonBlocking) != cudaSuccess) return CZ_ECUDA;
        if (cudaEventCreateWithFlags(&ev_fork[dev], cudaEventDisableTiming) != cudaSuccess) return CZ_ECUDA;
        if (cudaEventCreateWithFlags(&ev_join[dev], cudaEventDisableTiming) != cudaSuccess) return CZ_ECUDA;
    }
    if (cudaEventRecord(ev_fork[dev], st) != cudaSuccess) return CZ_ECUDA;
    if (cudaStreamWaitEvent(side[dev], ev_fork[dev], 0) != cudaSuccess) return CZ_ECUDA;
    k_value_mlp<<<(B + VM_POS - 1) / VM_POS, 256, 0, side[dev]>>>(hv, B, w1t, b1, w2, b2, value);
    if (cudaGetLastError() != cudaSuccess) return CZ_ECUDA;
    if (cudaEventRecord(ev_join[dev], side[dev]) != cudaSuccess) return CZ_ECUDA;
    launch_policy_fc(st);
    if (cudaGetLastError() != cudaSuccess) return CZ_ECUDA;
    if (cudaStreamWaitEvent(st, ev_join[dev], 0) != cudaSuccess) return CZ_ECUDA;
    return CZ_OK;
}

}  // namespace

extern "C" {

int cz_net_first_conv(const uint8_t *canon_boards, int B, const void *w1, const float *b1, void *out, void *stream) {
    if (!canon_boards || !w1 || !b1 || !out || B <= 0) return CZ_EINVAL;
    k_first_conv<<<B, 256, 0, (cudaStream_t)stream>>>(canon_boards, B, reinterpret_cast<const __half *>(w1), reinterpret_cast<const float4 *>(b1),
                                                      reinterpret_cast<__half *>(out));
    return cudaGetLastError() == cudaSuccess ? CZ_OK : CZ_ECUDA;
}

// value MLP (side stream) || policy FC on already computed head features hp / hv
int cz_net_heads_fc(const void *hp, const float *hv, int B, const float *w1t, const float *b1, const float *w2, const float *b2,
                    const void *wp, const float *bp, float *logits, float *value, void *stream) {
    if (!hp || !hv || !w1t || !b1 || !w2 || !b2 || !wp || !bp || !logits || !value || B <= 0) return CZ_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int smem = 2 * 64 * LDS_ROW * (int)sizeof(__half);   // 51200 B > the 48 KB default: opt in (per device, so every call)
    if (cudaFuncSetAttribute(k_policy_fc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return CZ_ECUDA;
    return value_mlp_beside(st, hv, B, w1t, b1, w2, b2, value, [&](cudaStream_t s) {
        k_policy_fc<<<dim3((B + 63) / 64, NPAD / 64), 128, smem, s>>>((const __half *)hp, B, (const __half *)wp, bp, logits);
    });
}

int cz_net_heads(const void *x, int B, const float *wh, const float *bh, const float *w1t, const float *b1, const float *w2, const float *b2,
                 const void *wp, const float *bp, void *hp_scratch, float *hv_scratch, float *logits, float *value, void *stream) {
    if (!x || !wh || !bh || !hp_scratch || !hv_scratch || B <= 0) return CZ_EINVAL;
    k_head_conv_mma<false><<<B, 192, 0, (cudaStream_t)stream>>>((const __half *)x, B, wh, bh, (__half *)hp_scratch, hv_scratch);
    if (cudaGetLastError() != cudaSuccess) return CZ_ECUDA;
    return cz_net_heads_fc(hp_scratch, hv_scratch, B, w1t, b1, w2, b2, wp, bp, logits, value, stream);
}

// The heads for large batches: conv1x1 on mma.sync writing the policy features in the wgmma-tiled layout, value MLP on a side stream,
// policy FC on wgmma (k_policy_fc_tc).  wp_tiled: dev fp16 [17 label tiles][24 k-chunks][128 labels][8] (labels >= 2086 zero),
// bp: dev f32 [2176]; hp_tiled scratch: fp16, ceil(B/128) * 49152 bytes, ZERO-INITIALISED by the caller (rows beyond B stay zero).
int cz_net_heads_tc(const void *x, int B, const float *wh, const float *bh, const float *w1t, const float *b1, const float *w2, const float *b2,
                    const void *wp_tiled, const float *bp, void *hp_tiled_scratch, float *hv_scratch, float *logits, float *value, void *stream) {
    if (!x || !wh || !bh || !w1t || !b1 || !w2 || !b2 || !wp_tiled || !bp || !hp_tiled_scratch || !hv_scratch || !logits || !value || B <= 0) return CZ_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int smem = 2 * FC_TILE_BYTES;
    if (cudaFuncSetAttribute(k_policy_fc_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return CZ_ECUDA;
    k_head_conv_mma<true><<<B, 192, 0, st>>>((const __half *)x, B, wh, bh, (__half *)hp_tiled_scratch, hv_scratch);
    if (cudaGetLastError() != cudaSuccess) return CZ_ECUDA;
    return value_mlp_beside(st, hv_scratch, B, w1t, b1, w2, b2, value, [&](cudaStream_t s) {
        k_policy_fc_tc<<<dim3((B + 127) / 128, 17), 256, smem, s>>>((const uint4 *)hp_tiled_scratch, B, (const uint4 *)wp_tiled, bp, logits);
    });
}

// The f32 epilogue of one three-product convolution fused with the operand split for the next one (k_epilogue_split):
//   v = ReLU(t + 2^-11 s + bias [+ skip]);  x (optional) = v;  hi / x2 (optional, both or neither) = split of v
//   (hi = tf32(v), x2 = { (v - hi) * 2^11 | hi }, see above).
// t dev f32 [n_pix][128]; s dev fp16 [n_pix][128] or NULL; bias dev f32 [128]; skip dev f32 [n_pix][128] or NULL (x may alias skip).
int cz_net_epilogue_split(const float *t, const void *s, const float *bias, const float *skip, float *x, float *hi, void *x2, long long n_pix, void *stream) {
    if (!t || !bias || n_pix <= 0 || (!x && !hi) || ((hi == nullptr) != (x2 == nullptr))) return CZ_EINVAL;
    const long long n8 = n_pix * 16;
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    long long blocks = (n8 + 255) / 256;
    if (blocks > 8LL * sms) blocks = 8LL * sms;
    k_epilogue_split<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(t), reinterpret_cast<const uint4 *>(s),
                                                                        reinterpret_cast<const float4 *>(bias), reinterpret_cast<const float4 *>(skip),
                                                                        reinterpret_cast<float4 *>(x), reinterpret_cast<float4 *>(hi),
                                                                        reinterpret_cast<uint4 *>(x2), n8);
    return cudaGetLastError() == cudaSuccess ? CZ_OK : CZ_ECUDA;
}

}  // extern "C"
