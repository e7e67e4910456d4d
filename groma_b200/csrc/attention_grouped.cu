// Decode attention of prompt groups (generate() with n prompts per image; DESIGN.md sections 3 and 4): the n <= 64 rows of an
// image share the K/V of their common prefix (positions 0 .. P - 1), which is streamed once per image and head and multiplied
// on the tensor cores, and each row merges its own keys (positions P .. *pos) on CUDA cores.
//
// One cluster of SPLIT CTAs per (head, image); 4 consumer warps (one wgmma warpgroup) + 1 TMA producer warp per CTA.
//   prologue  rows jr = rank (mod SPLIT) are reduced from the qkv split-K partials, rounded to bf16 and rotated at *pos exactly
//             as groma_decode_rope_attention does; q goes to the Q tile of every CTA of the cluster (DSMEM, 128-byte swizzle),
//             the new K/V row to the row cache at index *pos - P.  A cluster barrier publishes both.
//   prefix    the CTA's slice of the prefix keys is staged by TMA in 64-key tiles (2-deep ring); S = Q K^T (wgmma m64n64k16, Q
//             and K in shared memory), fp32 online softmax on the fragment, O += P V (P as the register operand), as
//             attention_wgmma.cu.  Pad query rows (n .. 63) are zero and never stored.
//   own keys  every row's own keys g = rank, rank + SPLIT, ... <= *pos - P (a warp per row, a lane per 4 dims) are merged into
//             the row's softmax state, which the prefix pass left in shared memory.
//   merge     rank c combines the SPLIT partial states of rows jr = c (mod SPLIT) through DSMEM and writes out[row] in bf16.
#include "ptx.cuh"
#include "wgmma.cuh"
#include "decode_common.cuh"
#include "capi_common.h"
#include "groma_b200.h"
#include <cooperative_groups.h>
#include <cstring>

namespace gb {

constexpr int GA_D = 128;
constexpr int GA_M = 64;                       // query rows of the wgmma tile = the largest group
constexpr int GA_BN = 64;                      // prefix keys per tile
constexpr int GA_STAGES = 2;
constexpr int GA_THREADS = 160;                // warps 0-3: consumer warpgroup, warp 4: TMA producer
constexpr int GA_TILE = GA_BN * GA_D * 2;      // one K or V tile: 2 column blocks of [64 keys][128 B]
constexpr int GA_Q_BYTES = GA_M * GA_D * 2;
constexpr int GA_SMEM = GA_Q_BYTES + 2 * GA_STAGES * GA_TILE + 1024;

struct GroupAttnParams {
    CUtensorMap tma_k, tma_v;                  // prefix [B * H * P, 128] bf16, box {64, 64}, 128-byte swizzle
    const float* ws; int S;                    // qkv split-K partials [S][B * n][3 * H * D]
    __nv_bfloat16* rk; __nv_bfloat16* rv;      // row cache [B * n, H, rcap, D]
    long long rcap;
    const int* pos_ptr;
    const float* cos_t; const float* sin_t;
    __nv_bfloat16* out;                        // [B * n, H * D]
    int H, n, P;
    float scale_log2;
};

__device__ __forceinline__ uint64_t ga_desc_sw128(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    uint64_t desc = 0;
    desc |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    desc |= static_cast<uint64_t>((lbo >> 4) & 0x3FFF) << 16;
    desc |= static_cast<uint64_t>((sbo >> 4) & 0x3FFF) << 32;
    desc |= static_cast<uint64_t>(1) << 62;
    return desc;
}

// byte offset of element (row, d) in a [2][64 rows][128 B] tile with the 128-byte swizzle TMA writes (16-byte chunk ^= row % 8)
__device__ __forceinline__ uint32_t ga_sw128_off(int row, int d) {
    const uint32_t c = (uint32_t)(d & 63) * 2;
    return (uint32_t)(d >> 6) * (GA_M * 128) + (uint32_t)row * 128 + ((((c >> 4) ^ (uint32_t)(row & 7)) << 4) | (c & 15));
}

__device__ __forceinline__ float ga_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <int SPLIT>
__global__ void __launch_bounds__(GA_THREADS, 1) decode_attention_grouped_kernel(const __grid_constant__ GroupAttnParams p) {
    constexpr int D = GA_D, half = D / 2;
    extern __shared__ uint8_t smem_raw_ga[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw_ga) + 1023) & ~uintptr_t(1023));
    uint8_t* Qs = smem;                                     // [2][64][128 B], swizzled
    uint8_t* Ks = Qs + GA_Q_BYTES;                          // [stages][2][64][128 B]
    uint8_t* Vs = Ks + GA_STAGES * GA_TILE;
    float* part_acc = reinterpret_cast<float*>(Ks);         // [64][128] after the prefix pass (the K ring is drained by then)
    __shared__ __align__(8) uint64_t k_full[GA_STAGES], k_empty[GA_STAGES], v_full[GA_STAGES], v_empty[GA_STAGES];
    __shared__ float part_m[GA_M], part_l[GA_M];

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = (int)cluster.block_rank();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int H = p.H, n = p.n, P = p.P;
    const int h = blockIdx.x / SPLIT, b = blockIdx.y;
    const int R = (int)gridDim.y * n;
    // this CTA's slice of the prefix, in whole 64-key tiles except the last
    const int per = ((P + SPLIT - 1) / SPLIT + GA_BN - 1) / GA_BN * GA_BN;
    const int k_begin = min(crank * per, P);
    const int nkeys = min(P, k_begin + per) - k_begin;
    const int nt = (nkeys + GA_BN - 1) / GA_BN;

    if (threadIdx.x == 0) {
        if (nt > 0) { tma_prefetch_desc(&p.tma_k); tma_prefetch_desc(&p.tma_v); }
        for (int s = 0; s < GA_STAGES; ++s) {
            mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 4); mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 4);
        }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < (GA_M - n) * D; i += GA_THREADS) {   // pad query rows: zero
        const int row = n + i / D, d = i % D;
        *reinterpret_cast<__nv_bfloat16*>(Qs + ga_sw128_off(row, d)) = __float2bfloat16_rn(0.f);
    }
    __syncthreads();
    cluster_sync_all();                  // every CTA of the cluster runs before any DSMEM store
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int pos = *p.pos_ptr, s_new = pos - P;

    if (warp == 4) {
        cluster_arrive_relaxed();        // the prologue barrier: the producer has nothing to publish
        if (lane == 0) {
            const int row0 = (b * H + h) * P + k_begin;
            for (int j = 0; j < nt; ++j) {
                const int st = j % GA_STAGES;
                const uint32_t ph = (j / GA_STAGES) & 1;
                mbar_wait(&k_empty[st], ph ^ 1);
                mbar_expect_tx(&k_full[st], GA_TILE);
#pragma unroll
                for (int blk = 0; blk < 2; ++blk)
                    tma_load_2d(Ks + st * GA_TILE + blk * (GA_BN * 128), &p.tma_k, &k_full[st], blk * 64, row0 + j * GA_BN);
                mbar_wait(&v_empty[st], ph ^ 1);
                mbar_expect_tx(&v_full[st], GA_TILE);
#pragma unroll
                for (int blk = 0; blk < 2; ++blk)
                    tma_load_2d(Vs + st * GA_TILE + blk * (GA_BN * 128), &p.tma_v, &v_full[st], blk * 64, row0 + j * GA_BN);
            }
        }
        __syncwarp();
        cluster_wait();
    } else {
        {   // prologue: rows jr = crank + SPLIT * i, two rows per pass (a thread per rotary pair)
            const int j = threadIdx.x & 63;
            const int N = 3 * H * D;
            const int cols[3] = {h * D, H * D + h * D, 2 * H * D + h * D};
            const float c = p.cos_t[(long long)pos * half + j], sn = p.sin_t[(long long)pos * half + j];
            for (int jr = crank + SPLIT * (threadIdx.x >> 6); jr < n; jr += 2 * SPLIT) {
                const int r = b * n + jr;
                float s1[3], s2[3];
                splitk_pairs<3>(p.ws, p.S, R, N, r, cols, j, half, s1, s2);
                __nv_bfloat16 q1, q2, k1, k2;
                rope_pair(bf16_round(s1[0]), bf16_round(s2[0]), c, sn, q1, q2);
                rope_pair(bf16_round(s1[1]), bf16_round(s2[1]), c, sn, k1, k2);
                const long long row = (((long long)r * H + h) * p.rcap + s_new) * D;
                p.rk[row + j] = k1; p.rk[row + j + half] = k2;
                p.rv[row + j] = __float2bfloat16_rn(s1[2]); p.rv[row + j + half] = __float2bfloat16_rn(s2[2]);
                const uint32_t o1 = ga_sw128_off(jr, j), o2 = ga_sw128_off(jr, j + half);
#pragma unroll
                for (int t = 0; t < SPLIT; ++t) {
                    uint8_t* q = cluster.map_shared_rank(Qs, t);
                    *reinterpret_cast<__nv_bfloat16*>(q + o1) = q1;
                    *reinterpret_cast<__nv_bfloat16*>(q + o2) = q2;
                }
            }
        }
        // publishes the Q rows (DSMEM) and the new K/V rows (global) to the cluster
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
        fence_proxy_async();             // generic-proxy stores of Q -> wgmma operand reads

        // ---------------- prefix keys on the tensor cores: this thread holds rows r0 and r0 + 8 of the 64
        const int cq = (lane & 3) * 2;
        const int r0 = warp * 16 + (lane >> 2);
        float o[D / 2];
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        const uint32_t q_addr = smem_u32(Qs);
        for (int j = 0; j < nt; ++j) {
            const int st = j % GA_STAGES;
            const uint32_t ph = (j / GA_STAGES) & 1;
            const int j0 = j * GA_BN;
            float s[GA_BN / 2];
            mbar_wait(&k_full[st], ph);
            {
                const uint32_t k_addr = smem_u32(Ks + st * GA_TILE);
                wgmma_fence_regs(s);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < D / 16; ++kk) {
                    const uint32_t off = (kk >> 2) * (GA_M * 128) + (kk & 3) * 32;   // Q and K tiles both have 64 rows
                    wgmma_ss<GA_BN>(s, ga_desc_sw128(q_addr + off, 0, 1024), ga_desc_sw128(k_addr + off, 0, 1024), kk > 0 ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(s);
            }
            if (lane == 0) mbar_arrive(&k_empty[st]);
            if (j0 + GA_BN > nkeys) {
#pragma unroll
                for (int i = 0; i < GA_BN / 2; ++i) {
                    const int key = j0 + (i >> 2) * 8 + cq + (i & 1);
                    if (key >= nkeys) s[i] = -INFINITY;
                }
            }
            float corr[2];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                float mx = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < GA_BN / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * rr], s[4 * jj + 2 * rr + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[rr], mx * p.scale_log2);
                const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
                corr[rr] = ga_ex2(m_run[rr] - m_use);
                m_run[rr] = m_new;
                float rs = 0.f;
#pragma unroll
                for (int jj = 0; jj < GA_BN / 8; ++jj) {
                    const float p0 = ga_ex2(fmaf(s[4 * jj + 2 * rr], p.scale_log2, -m_use));
                    const float p1 = ga_ex2(fmaf(s[4 * jj + 2 * rr + 1], p.scale_log2, -m_use));
                    rs += p0 + p1;
                    s[4 * jj + 2 * rr] = p0; s[4 * jj + 2 * rr + 1] = p1;
                }
                l_run[rr] = l_run[rr] * corr[rr] + rs;
            }
#pragma unroll
            for (int i = 0; i < D / 2; ++i) o[i] *= corr[(i >> 1) & 1];
            mbar_wait(&v_full[st], ph);
            {
                const uint32_t v_addr = smem_u32(Vs + st * GA_TILE);
                uint32_t a[GA_BN / 16][4];
#pragma unroll
                for (int kk = 0; kk < GA_BN / 16; ++kk) {
                    a[kk][0] = pack_bf16x2(s[8 * kk], s[8 * kk + 1]); a[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
                    a[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]); a[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
                }
                wgmma_fence_regs(o);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < GA_BN / 16; ++kk)   // V tile MN-major: SBO = 8 key rows, LBO = the next 64-wide d block
                    wgmma_rs_tb<D>(o, a[kk], ga_desc_sw128(v_addr + kk * 2048, GA_BN * 128, 1024), 1u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(o);
            }
            if (lane == 0) mbar_arrive(&v_empty[st]);
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");      // every consumer is past the K ring: part_acc may overwrite it
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            float l = l_run[rr];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const int row = r0 + 8 * rr;
            if (row < n) {
                if ((lane & 3) == 0) { part_m[row] = m_run[rr]; part_l[row] = l; }
#pragma unroll
                for (int jj = 0; jj < D / 8; ++jj) {
                    part_acc[row * D + 8 * jj + cq] = o[4 * jj + 2 * rr];
                    part_acc[row * D + 8 * jj + cq + 1] = o[4 * jj + 2 * rr + 1];
                }
            }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");

        // ---------------- own keys g = crank + SPLIT * i <= s_new on CUDA cores: a warp per row, a lane per 4 dims
        const int ng = s_new + 1 > crank ? (s_new + 1 - crank + SPLIT - 1) / SPLIT : 0;
        for (int jr = warp; jr < n; jr += 4) {
            const int r = b * n + jr;
            float qf[4], acc[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                qf[t] = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(Qs + ga_sw128_off(jr, lane * 4 + t)));
                acc[t] = part_acc[jr * D + lane * 4 + t];
            }
            float m = part_m[jr], lsum = part_l[jr];
            const long long base = ((long long)r * H + h) * p.rcap * D + lane * 4;
            constexpr int U = 4;
            for (int i0 = 0; i0 < ng; i0 += U) {
                float s[U];
                uint2 vv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int i = i0 + u;
                    const long long off = base + (long long)(crank + i * SPLIT) * D;
                    uint2 kk = make_uint2(0u, 0u);
                    vv[u] = make_uint2(0u, 0u);
                    if (i < ng) {   // L2 reads: rows written this step by other CTAs of the cluster
                        kk = __ldcg(reinterpret_cast<const uint2*>(p.rk + off));
                        vv[u] = __ldcg(reinterpret_cast<const uint2*>(p.rv + off));
                    }
                    const __nv_bfloat162* k2 = reinterpret_cast<const __nv_bfloat162*>(&kk);
                    const float2 f0 = __bfloat1622float2(k2[0]), f1 = __bfloat1622float2(k2[1]);
                    float d = f0.x * qf[0] + f0.y * qf[1] + f1.x * qf[2] + f1.y * qf[3];
#pragma unroll
                    for (int x = 16; x > 0; x >>= 1) d += __shfl_xor_sync(0xffffffffu, d, x);
                    s[u] = i < ng ? d * p.scale_log2 : -INFINITY;
                }
                float mn = m;
#pragma unroll
                for (int u = 0; u < U; ++u) mn = fmaxf(mn, s[u]);
                const float mref = (mn == -INFINITY) ? 0.f : mn;
                const float corr = exp2f(m - mref);
                m = mn;
                lsum *= corr;
#pragma unroll
                for (int t = 0; t < 4; ++t) acc[t] *= corr;
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (s[u] == -INFINITY) continue;
                    const float pu = exp2f(s[u] - mref);
                    lsum += pu;
                    const float pb = bf16_round(pu);
                    const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(&vv[u]);
                    const float2 f0 = __bfloat1622float2(v2[0]), f1 = __bfloat1622float2(v2[1]);
                    acc[0] += pb * f0.x; acc[1] += pb * f0.y; acc[2] += pb * f1.x; acc[3] += pb * f1.y;
                }
            }
            if (lane == 0) { part_m[jr] = m; part_l[jr] = lsum; }
#pragma unroll
            for (int t = 0; t < 4; ++t) part_acc[jr * D + lane * 4 + t] = acc[t];
        }
    }
    // ---------------- merge of the SPLIT partial states: rank c writes rows jr = c (mod SPLIT)
    cluster_sync_all();
    {
        const int mine = (n - crank + SPLIT - 1) / SPLIT;
        for (int i = threadIdx.x; i < mine * D; i += GA_THREADS) {
            const int jr = crank + (i / D) * SPLIT, d = i % D;
            float mr[SPLIT];
            float M = -INFINITY;
#pragma unroll
            for (int t = 0; t < SPLIT; ++t) {
                mr[t] = *cluster.map_shared_rank(&part_m[jr], t);
                M = fmaxf(M, mr[t]);
            }
            float num = 0.f, den = 0.f;
#pragma unroll
            for (int t = 0; t < SPLIT; ++t) {
                const float c = (mr[t] == -INFINITY) ? 0.f : exp2f(mr[t] - M);
                num += c * *cluster.map_shared_rank(&part_acc[jr * D + d], t);
                den += c * *cluster.map_shared_rank(&part_l[jr], t);
            }
            p.out[((long long)(b * n + jr) * H + h) * D + d] = __float2bfloat16_rn(den > 0.f ? num / den : 0.f);
        }
    }
    cluster_sync_all();                  // no CTA leaves while a peer still reads its partial state
}

typedef CUresult (*PFN_encodeTiledGa)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int ga_make_map(CUtensorMap* map, const void* ptr, uint64_t rows) {
    static PFN_encodeTiledGa enc = nullptr;
    if (!enc) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return GROMA_ERR_DRIVER;
        enc = reinterpret_cast<PFN_encodeTiledGa>(fp);
    }
    cuuint64_t dims[2] = {GA_D, rows};
    cuuint64_t strides[1] = {GA_D * 2};
    cuuint32_t box[2] = {64, GA_BN};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
               ? GROMA_OK : GROMA_ERR_TMA_ENCODE;
}

template <int SPLIT>
static cudaError_t launch_grouped(cudaLaunchConfig_t cfg, const GroupAttnParams& p, int B) {
    static bool set = false;
    if (!set) {
        const cudaError_t e = cudaFuncSetAttribute(decode_attention_grouped_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, GA_SMEM);
        if (e != cudaSuccess) return e;
        set = true;
    }
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (cfg.numAttrs) attr[na++] = cfg.attrs[0];
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = SPLIT; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
    cfg.attrs = attr; cfg.numAttrs = na;
    cfg.gridDim = dim3(p.H * SPLIT, B, 1);
    cfg.dynamicSmemBytes = GA_SMEM;
    return cudaLaunchKernelEx(&cfg, decode_attention_grouped_kernel<SPLIT>, p);
}

}  // namespace gb

using namespace gb;

GROMA_API int32_t groma_decode_rope_attention_grouped(const float* ws, int32_t splits, const void* prefix_k, const void* prefix_v,
                                                      int32_t prefix_len, void* row_k, void* row_v, int64_t row_cap,
                                                      const int32_t* pos_ptr, const float* cos_t, const float* sin_t, void* out,
                                                      int32_t B, int32_t n, int32_t H, int32_t D, float scale, int32_t pdl,
                                                      void* stream) {
    if (!ws || !row_k || !row_v || !pos_ptr || !cos_t || !sin_t || !out || B <= 0 || H <= 0 || splits < 1 || row_cap < 1 ||
        prefix_len < 0 || (prefix_len > 0 && (!prefix_k || !prefix_v)))
        return GROMA_ERR_ARG;
    if (D != GA_D || n < 1 || n > GROMA_GROUP_MAX_PROMPTS || B * n > GROMA_BEAM_MAX_ROWS) return GROMA_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(prefix_k) & 15) || (reinterpret_cast<uintptr_t>(prefix_v) & 15) ||
        (reinterpret_cast<uintptr_t>(row_k) & 7) || (reinterpret_cast<uintptr_t>(row_v) & 7))
        return GROMA_ERR_ALIGN;
    GroupAttnParams p;
    memset(&p, 0, sizeof(p));
    if (prefix_len > 0) {
        const uint64_t rows = (uint64_t)B * H * prefix_len;
        int rc = ga_make_map(&p.tma_k, prefix_k, rows); if (rc) return rc;
        rc = ga_make_map(&p.tma_v, prefix_v, rows); if (rc) return rc;
    }
    p.ws = ws; p.S = splits;
    p.rk = (__nv_bfloat16*)row_k; p.rv = (__nv_bfloat16*)row_v; p.rcap = row_cap;
    p.pos_ptr = pos_ptr; p.cos_t = cos_t; p.sin_t = sin_t;
    p.out = (__nv_bfloat16*)out;
    p.H = H; p.n = n; p.P = prefix_len;
    p.scale_log2 = scale * 1.4426950408889634f;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(GA_THREADS);
    cfg.stream = reinterpret_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    if (pdl) { cfg.attrs = attr; cfg.numAttrs = 1; }
    // key split: the smallest cluster that puts two CTAs (82 KB of shared memory each) on every SM, so that B = 1 with 32 heads
    // still fills the GPU; no more splits than 64-key tiles of the prefix
    const long long clusters = (long long)H * B, want = 2LL * groma_num_sms();
    int split = clusters >= want ? 1 : clusters * 2 >= want ? 2 : clusters * 4 >= want ? 4 : 8;
    while (split > 1 && (long long)(split / 2) * GA_BN >= prefix_len) split /= 2;
    const cudaError_t e = split == 1 ? launch_grouped<1>(cfg, p, B) : split == 2 ? launch_grouped<2>(cfg, p, B)
                        : split == 4 ? launch_grouped<4>(cfg, p, B) : launch_grouped<8>(cfg, p, B);
    return e == cudaSuccess ? GROMA_OK : GROMA_ERR_CUDA;
}
