// cz_tower.cu -- the whole convolutional trunk of the policy-value network for a FEW positions (1..16) in ONE launch:
// first conv3x3(14->128) + res_block_nums x [conv3x3 -> ReLU -> conv3x3 -> +skip -> ReLU] + the two 1x1 head convolutions
// (policy_value_network.py:45-74, 151-162; batch norm folded into the weights), hand-written for sm_90a (H100).
//
// Why: play mode (BASELINE config 5) and any single-tree search evaluate one leaf (or a handful) per network call.  At batch 1
// the library path is 15+ launches of ~5 us each, every one re-reading its weights; here the activations of a position never
// leave the SMs and the weights stream from L2 under the tensor cores.
//
// Shape: one thread-block CLUSTER of CL = 4 CTAs per position; CTA r owns output channels [r*NC, (r+1)*NC), NC = 128/CL = 32.
// Per 3x3 convolution and CTA:
//     D[128 rows][NC ch] (f32, registers) = sum over 9 taps of  A_tap[128][128] . B_tap[128][NC]
//   as two warpgroups, each 72 wgmma.mma_async m64n32k16 over its 64 rows.
//   * A = the position's activation image, fp16, resident in shared memory in the canonical K-major NO-SWIZZLE layout
//     [16 k-chunks of 8 channels][152 rows][8 halves]: with SBO = 128 B consecutive rows are 16 bytes apart in every chunk, so a
//     3x3 tap is nothing but a START-ADDRESS OFFSET of (dr*11 + df) rows in the A descriptor -- no im2col, no copies.  Rows are
//     image cells in a padded raster: cell (r, f) of the reference's [9][10] image sits in row 12 + r*11 + f; the 11th column and
//     the rows above / below are zeros, which gives the convolution's zero padding for free (99 of the 128 MMA rows are cells).
//   * B = this CTA's slice of the layer's weights, streamed tap by tap from L2 by TMA (cp.async.bulk.tensor, SASS UTMALDG)
//     through a ring of shared-memory stages (full / empty mbarriers); the producer runs ahead across layers.
//   * epilogue: each math thread adds bias (+ the residual skip) to its accumulator fragment, applies ReLU, converts to fp16 and
//     writes its channel pairs of the NEXT layer's A image into the shared memory of ALL CL CTAs of the cluster (st.async DSMEM
//     stores that complete their byte count on the receiver's `act_ready` mbarrier); a CTA starts the next layer when all bytes of
//     the image have arrived.  No cluster-wide barrier on the critical path.
// Warp roles: 8 math warps (two warpgroups: MMA rows 0-63 and 64-127), then one TMA producer warp (one elected lane).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cchess_b200.h"
#include "cz_wgmma.cuh"

namespace {

using namespace cz_sm90;

constexpr int ROWS = 152;                 // rows per k-chunk of an activation image (12 pad + 128 MMA rows + 12 pad)
constexpr int P0 = 12;                    // row of image cell (0, 0)
constexpr int LBO_A = ROWS * 16;          // bytes between k-chunks of A
constexpr int A_BYTES = 16 * LBO_A;       // 38 912 B per activation image
constexpr int NMATH = 256;                // two warpgroups
constexpr int NMATH_WARPS = NMATH / 32;
constexpr int NTHREADS = NMATH + 32;      // + the TMA producer warp
constexpr int CL = 4;                     // CTAs per cluster (one position)
constexpr int NC = 128 / CL;              // output channels of one CTA (= wgmma N)
constexpr int STAGE_BYTES = NC * 256;     // one tap of a CTA's weight slice: [16 k-chunks][NC rows][8 halves]
constexpr int S = 16;                     // weight ring depth (stages)

// Byte offset of (8-channel chunk 0..15, raster row) inside an activation image: canonical K-major NO-SWIZZLE layout
// [16 chunks][ROWS rows][16 B] (LBO = ROWS*16, SBO = 128).  A tap shift is a start-address offset of whole rows.
__device__ __forceinline__ uint32_t img_off(int chunk, int row) { return (uint32_t)(chunk * LBO_A + row * 16); }

__device__ __forceinline__ void mbar_init(uint64_t *b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
// wait on a barrier whose arrivals all come from THIS CTA (threads, TMA): CTA-scope acquire
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity) {
    const uint32_t a = smem_u32(b);
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 ::"r"(a), "r"(parity) : "memory");
}
// wait on a barrier that peer CTAs arrive on after writing OUR shared memory: cluster-scope acquire.  ptxas turns that into an
// L1 invalidate per successful wait, so exactly one thread per CTA and layer waits this way; everybody else is ordered behind it
// with a CTA-scope named barrier.
__device__ __forceinline__ void mbar_wait_cluster(uint64_t *b, uint32_t parity) {
    const uint32_t a = smem_u32(b);
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 ::"r"(a), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// Async-proxy stores into CTA `rank`'s shared memory that complete their byte count on THAT CTA's mbarrier: the designed
// DSMEM producer -> consumer path.  The barrier completes by byte count: no arrive loop, no release fence on the critical path.
__device__ __forceinline__ void st_async_v4(uint32_t local_addr, uint32_t local_bar, uint32_t rank, uint4 v) {
    uint32_t ra, rb;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(local_bar), "r"(rank));
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(ra), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(rb) : "memory");
}
__device__ __forceinline__ void st_async_b32(uint32_t local_addr, uint32_t local_bar, uint32_t rank, uint32_t v) {
    uint32_t ra, rb;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(local_bar), "r"(rank));
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra), "r"(v), "r"(rb) : "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void math_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NMATH) : "memory"); }   // the math warps only

struct TowerArgs {
    const uint8_t *boards;     // [n][96] side-to-move canonical boards
    const __half *w1;          // [9][14][128] folded first conv
    const float *bias;         // [1 + 2*blocks][128] folded biases (layer 0 = first conv)
    const float *wh;           // [3][128] folded 1x1 head convs (policy 2 + value 1)
    const float *bh;           // [3]
    __half *hp;                // out [n][192]
    float *hv;                 // out [n][96]
    int n_pos;
    int n_conv;                // 2 * res_block_nums
};

__global__ void __launch_bounds__(NTHREADS, 1) k_tower_small(const __grid_constant__ CUtensorMap wmap, TowerArgs a) {
    constexpr uint32_t IMAGE_TX = 128u * 16u * 16u;        // bytes every CTA receives per image: 128 rows x 16 chunks x 16 B
    constexpr int W = NC / 2;                              // layer 0: channels per math thread (two column groups)
    static_assert(W % 8 == 0 && W >= 8, "layer-0 column groups");
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *bufX = smem, *bufY = smem + A_BYTES, *ring = smem + 2 * A_BYTES;
    float *s_bias = reinterpret_cast<float *>(ring + S * STAGE_BYTES);      // [n_layers][NC] this CTA's slice
    __shared__ __align__(8) uint64_t full[S], empty[S], act_ready[2];       // act_ready ping-pongs by layer parity: arrivals of consecutive layers never mix

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rank = cluster_rank();
    const int pos = blockIdx.x / CL;
    const int n_layers = 1 + a.n_conv;

    // ---- one-time setup ----
    for (int i = tid; i < 2 * A_BYTES / 16; i += NTHREADS) reinterpret_cast<uint4 *>(smem)[i] = make_uint4(0, 0, 0, 0);   // zero images (padding rows stay zero)
    for (int i = tid; i < n_layers * NC; i += NTHREADS) s_bias[i] = a.bias[(i / NC) * 128 + rank * NC + (i % NC)];
    if (tid == 0) {
        for (int s = 0; s < S; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], NMATH_WARPS); }
        mbar_init(&act_ready[0], 1);                     // one arrive.expect_tx by thread 0 + IMAGE_TX bytes
        mbar_init(&act_ready[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async;" ::: "memory");     // the zeroed images (generic proxy) are what the tensor cores will read as padding
    __syncthreads();
    cluster_sync_all();                                  // every CTA's barriers and zeroed images exist before anyone writes remotely

    if (warp == NMATH_WARPS) {
        // ===== TMA producer: taps of all layers, in order, as fast as the ring frees up =====
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int L = 0; L < a.n_conv; L++) {
                for (int t = 0; t < 9; t++) {
                    mbar_wait(&empty[stage], phase ^ 1u);
                    mbar_expect_tx(&full[stage], STAGE_BYTES);
                    const int row = ((L * 9 + t) * CL + (int)rank) * NC;          // 256-byte rows of the weight blob
                    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                                 ::"r"(smem_u32(ring + stage * STAGE_BYTES)), "l"(&wmap), "r"(0), "r"(row), "r"(smem_u32(&full[stage])) : "memory");
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        // ===== math warps: layer 0 by thread = (column group cg, MMA row j = raster row P0 + j) =====
        {
            const int j = tid & 127, cg = tid >> 7;          // row 0..127, column group 0..1: channels [cg*W, (cg+1)*W) of this CTA's NC
            const int rr = j / 11, ff = j - rr * 11;
            const bool cell = rr < 9 && ff < 10;             // a real image cell (else padding: must be written as zero)
            // conv3x3(14 -> 128) straight from the board bytes (one-hot input: a gather-add of weight rows)
            float acc[W];
#pragma unroll
            for (int c = 0; c < W; c++) acc[c] = s_bias[cg * W + c];
            if (cell) {
                const uint8_t *bd = a.boards + (size_t)pos * 96;
#pragma unroll 1
                for (int t = 0; t < 9; t++) {
                    const int r2 = rr + t / 3 - 1, f2 = ff + t % 3 - 1;
                    if (r2 < 0 || r2 >= 9 || f2 < 0 || f2 >= 10) continue;
                    const int pc = __ldg(bd + r2 * 9 + f2);                        // the reference's cell <- s[rank*9+file]
                    if (!pc) continue;
                    const __half *wr = a.w1 + ((size_t)(t * 14 + pc - 1) * 128 + rank * NC + cg * W);
#pragma unroll
                    for (int c8 = 0; c8 < W / 8; c8++) {
                        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(wr) + c8);
                        const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw);
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            const float2 v = __half22float2(h2[k]);
                            acc[c8 * 8 + 2 * k] += v.x;
                            acc[c8 * 8 + 2 * k + 1] += v.y;
                        }
                    }
                }
            }
#pragma unroll
            for (int c8 = 0; c8 < W / 8; c8++) {
                uint4 o;
                __half2 *oh = reinterpret_cast<__half2 *>(&o);
#pragma unroll
                for (int k = 0; k < 4; k++)
                    oh[k] = cell ? __floats2half2_rn(relu_nan(acc[c8 * 8 + 2 * k]), relu_nan(acc[c8 * 8 + 2 * k + 1])) : __floats2half2_rn(0.f, 0.f);
                const int chunk = (int)rank * (NC / 8) + cg * (W / 8) + c8;          // 8-channel chunk of the full image
                const uint32_t dst = smem_u32(bufX) + img_off(chunk, P0 + j);
#pragma unroll
                for (int qi = 0; qi < CL; qi++) {
                    const uint32_t q = (rank + 1u + (uint32_t)qi) & (uint32_t)(CL - 1);   // every CTA starts with a different receiver (ingress spread), itself last
                    st_async_v4(dst, smem_u32(&act_ready[0]), q, o);
                }
            }
        }
        // ===== residual tower: warpgroup wg multiplies MMA rows [64 wg, 64 wg + 64); this thread's accumulator rows are j0, j0 + 8 =====
        const int wg = tid >> 7, q = lane & 3;
        const int j0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        bool cell[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int j = j0 + 8 * h, rr = j / 11, ff = j - rr * 11;
            cell[h] = rr < 9 && ff < 10;
        }
        float d[NC / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int L = 0; L < a.n_conv; L++) {
            if (tid == 0) {
                mbar_expect_tx(&act_ready[L & 1], IMAGE_TX);                    // our arrival + the byte count of image L
                mbar_wait_cluster(&act_ready[L & 1], (uint32_t)((L >> 1) & 1));   // image L (this layer's input) is complete in OUR shared memory
            }
            math_sync();
            const uint32_t abase = smem_u32((L & 1) ? bufY : bufX) + (uint32_t)((P0 + wg * 64) * 16);   // conv1 of a block reads X, conv2 reads Y
            int prev = 0;
            for (int t = 0; t < 9; t++) {
                mbar_wait(&full[stage], phase);
                const int shift = (t / 3 - 1) * 11 + (t % 3 - 1);                // tap (dr, df) = a row offset in the padded raster
                // Descriptors of the 8 K16 steps differ only in the start-address field: one add each from the tap's base descriptor.
                const uint64_t da0 = gmma_desc(abase + (uint32_t)(shift * 16), LBO_A);
                const uint64_t db0 = gmma_desc(smem_u32(ring + stage * STAGE_BYTES), NC * 16);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 8; kk++)                                   // 128 input channels = 8 x K16
                    Wgmma<NC>::mma(d, da0 + (uint64_t)((kk * 2 * LBO_A) >> 4), db0 + (uint64_t)((kk * 2 * (NC * 16)) >> 4), (t | kk) ? 1u : 0u);
                wgmma_commit();
                if (t > 0) {                                                     // the previous tap's MMAs are done: free its stage
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty[prev]);
                }
                prev = stage;
                if (++stage == S) { stage = 0; phase ^= 1u; }
            }
            wgmma_wait<0>();
            fence_regs(d);
            if (lane == 0) mbar_arrive(&empty[prev]);
            // ---- epilogue: bias (+ skip), ReLU, fp16, this thread's channel pairs of image L + 1 into every CTA of the cluster ----
            const bool second = L & 1;                        // conv2 of a block: + skip (the block input, still in X), result back into X
            unsigned char *dstbuf = second ? bufX : bufY;
            const float *bl = s_bias + (1 + L) * NC;
#pragma unroll
            for (int c8 = 0; c8 < NC / 8; c8++) {
                const int chunk = (int)rank * (NC / 8) + c8;                     // 8-channel chunk of the full image
                const float b0 = bl[c8 * 8 + 2 * q], b1 = bl[c8 * 8 + 2 * q + 1];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint32_t off = img_off(chunk, P0 + j0 + 8 * h) + (uint32_t)(q * 4);
                    float f0 = d[4 * c8 + 2 * h] + b0, f1 = d[4 * c8 + 2 * h + 1] + b1;
                    if (second) {                                                // only this thread writes this word: it reads its own skip
                        const float2 s = __half22float2(*reinterpret_cast<const __half2 *>(bufX + off));
                        f0 += s.x; f1 += s.y;
                    }
                    const __half2 o = cell[h] ? __floats2half2_rn(relu_nan(f0), relu_nan(f1)) : __floats2half2_rn(0.f, 0.f);
                    const uint32_t ov = *reinterpret_cast<const uint32_t *>(&o);
#pragma unroll
                    for (int qi = 0; qi < CL; qi++)   // receivers in rotated order: at any moment the CL senders address CL different CTAs
                        st_async_b32(smem_u32(dstbuf) + off, smem_u32(&act_ready[(L + 1) & 1]), (rank + 1u + (uint32_t)qi) & (uint32_t)(CL - 1), ov);
                }
            }
        }
        // ---- heads: conv1x1 (128 -> 2 policy + 1 value) + bias + ReLU on the final image (in X), CTA 0 writes ----
        {
            if (tid == 0) {
                mbar_expect_tx(&act_ready[a.n_conv & 1], IMAGE_TX);
                mbar_wait_cluster(&act_ready[a.n_conv & 1], (uint32_t)((a.n_conv >> 1) & 1));                // the final image (index n_conv) is complete
            }
            math_sync();                                                           // ordered behind thread 0's cluster-scope acquire
            const int j = tid & 127, rr = j / 11, ff = j - rr * 11;
            if (rank == 0 && tid < 128 && rr < 9 && ff < 10) {
                float s0 = a.bh[0], s1 = a.bh[1], s2 = a.bh[2];
#pragma unroll 4
                for (int c8 = 0; c8 < 16; c8++) {
                    const uint4 raw = *reinterpret_cast<const uint4 *>(bufX + img_off(c8, P0 + j));
                    const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const float2 x = __half22float2(h2[k]);
                        const int c = c8 * 8 + 2 * k;
                        s0 += x.x * __ldg(a.wh + c) + x.y * __ldg(a.wh + c + 1);
                        s1 += x.x * __ldg(a.wh + 128 + c) + x.y * __ldg(a.wh + 128 + c + 1);
                        s2 += x.x * __ldg(a.wh + 256 + c) + x.y * __ldg(a.wh + 256 + c + 1);
                    }
                }
                const int ci = rr * 10 + ff;                                       // flatten order of tf.reshape on NHWC: cell*2 + c
                *reinterpret_cast<__half2 *>(a.hp + (size_t)pos * 192 + ci * 2) = __floats2half2_rn(relu_nan(s0), relu_nan(s1));
                a.hv[(size_t)pos * 96 + ci] = relu_nan(s2);
            }
            if (rank == 0 && tid < 12) a.hp[(size_t)pos * 192 + 180 + tid] = __float2half(0.f);   // K padding of the policy GEMM
        }
    }
    // ---- teardown: nobody leaves while a peer may still write into its shared memory ----
    __syncthreads();
    cluster_sync_all();
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

}  // namespace

extern "C" {

// Bytes of the weight blob cz_net_tower_small expects for `n_conv` 3x3 convolutions.
int64_t cz_net_tower_blob_bytes(int n_conv) { return (int64_t)n_conv * 9 * 128 * 256; }

int cz_net_tower_small(const uint8_t *canon_boards, int n_pos, int n_conv, const void *w1, const void *wblob, const float *bias,
                       const float *wh, const float *bh, void *hp, float *hv, void *stream) {
    if (!canon_boards || !w1 || !wblob || !bias || !wh || !bh || !hp || !hv || n_pos <= 0 || n_conv <= 0 || (n_conv & 1)) return CZ_EINVAL;
    EncodeTiledFn enc = encode_tiled();
    if (!enc) return CZ_ECUDA;
    // the blob as a 2-D tensor of 256-byte rows: [n_conv * 9 * 128 rows][128 halves]; one box = one tap of one CTA's slice
    CUtensorMap map;
    const cuuint64_t gdim[2] = {128, (cuuint64_t)n_conv * 9 * 128};
    const cuuint64_t gstride[1] = {256};
    const cuuint32_t box[2] = {128, (cuuint32_t)NC};
    const cuuint32_t estr[2] = {1, 1};
    if (enc(&map, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void *>(wblob), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return CZ_ECUDA;
    TowerArgs a;
    a.boards = canon_boards; a.w1 = (const __half *)w1; a.bias = bias; a.wh = wh; a.bh = bh; a.hp = (__half *)hp; a.hv = hv;
    a.n_pos = n_pos; a.n_conv = n_conv;
    const size_t smem = 2 * (size_t)A_BYTES + (size_t)S * STAGE_BYTES + (size_t)(1 + n_conv) * NC * 4;
    if (cudaFuncSetAttribute(k_tower_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return CZ_ECUDA;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(a.n_pos * CL));
    cfg.blockDim = dim3(NTHREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k_tower_small, map, a) == cudaSuccess ? CZ_OK : CZ_ECUDA;
}

}  // extern "C"

