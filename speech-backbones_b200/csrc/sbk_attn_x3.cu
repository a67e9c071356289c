// LinearAttention pass 1 fused (Grad-TTS/model/diffusion.py:93-96): k|v projection, softmax-over-pixels statistics and
// the context partials S[d][e] = sum_px P[d,px] V[e,px] in ONE persistent wgmma kernel - k and v never reach HBM.
//
// One ITEM = 64 consecutive pixels of one sample, all four heads.  The pixels are the M operand of the projection:
//     warpgroup 0:  K^T[px][k row 32*head+d] = X Wk^T,     warpgroup 1:  V^T[px][v row 32*head+e] = X Wv^T
// (one m64n128 wgmma per K step each, the same activation tile for both).  The two results go to shared memory as K-major
// images [4-pixel chunk][row][16 B] - the operand layout of the context MMAs - and the softmax runs over those images,
// one thread per (row, half of the item's pixels): P = exp(k - max) replaces K in place.  The context S = P V^T is a
// second pair of wgmmas (warpgroup c: rows / columns 64c..64c+63, i.e. heads 2c and 2c+1; only the two diagonal 32 x 32
// blocks are kept).  Per item and head one partial {max[32], sum[32], S[32][32]} is written, merged by k_attn_ctx.
//
// Precision modes.  tf32: tf32 projection, fp32 softmax, tf32 context (P and V fp32 in shared memory, read as tf32).
// bf16: the activations and weights are bf16 (a stage carries 64 channels), the rest as tf32.  fp32x3: every product is
// fp32-class: each 32-channel K stage runs as an f16 correction sub-stage on the packed fp16 chunks ({x_lo, x*2^-12} x
// {w, w_lo*2^12}, sbk_internal.h: corr_chunk) followed by the tf32 main sub-stage (x_hi * w_hi), and the context adds
//     [ P_lo V^T + P V_lo^T ]  from  Pc = {P_lo*2^8, P*2^-4},  Vc = {V*2^-8, V_lo*2^4}  (fp16 images)
// to P_hi V_hi^T.  The powers of two are exact and keep neither the tiny softmax numerators nor V_lo in fp16's subnormals.
//
// Pipeline (one CTA per SM, persistent over items): loader warp (cp.async.bulk, STAGES-deep ring of 40 KB stages) and two
// consumer warpgroups; the projection of item i+1 streams in while the softmax / context of item i run.
#include "sbk_tc.cuh"

#include <type_traits>

namespace sbk {

using namespace tc;

namespace kx3 {
constexpr int PX = 64;                         // pixels per item: M of the projection, K extent of the context MMAs
constexpr int KCH = 8;                         // 16-byte channel chunks per stage
constexpr int XS = KCH * PX * 16;              // activation stage [chunk][pixel][16 B]
constexpr int WS = 2 * KCH * 128 * 16;         // weight stage     [k|v][chunk][row][16 B]
constexpr int STAGE = XS + WS;
constexpr int STAGES = 2;
constexpr int OPI = (PX / 4) * 128 * 16;       // one context operand image [pixel chunk][row][16 B]
constexpr int THREADS = 256 + 32;              // 2 consumer warpgroups + loader warp
constexpr int NBARS = 2 * STAGES;
constexpr size_t SMEM = (size_t)STAGES * STAGE + 4 * OPI + 4 * 128 * 4 + NBARS * 8 + 16;
static_assert(SMEM <= 227 * 1024, "shared memory budget");
static_assert(XS <= OPI && STAGES == 2, "fp32x3: the converted x fits a context image; a K stage is the whole ring");
}

// MODE: 0 = tf32, 1 = bf16, 2 = fp32x3.  p.in0: x (fp32x3: its correction chunks are derived here: the loader brings x with the main sub-stage only and the consumers convert it into the idle Pc / Vc images, alternating
// between them per K stage so that one warpgroup may still read the last stage's chunks); p.c0 = C; p.wpk: the k|v rows
// of to_qkv as per-stage images [k|v][chunk][row][16 B] (fp32x3: [32-channel stage][hi | correction][k|v]...,
// sbk_conv_tc.cu attn_kv_pack_image);
// p.kv_part: [B][items per sample][4][kKvPartFloats]
template <int MODE>
__global__ void __launch_bounds__(kx3::THREADS, 1) k_attn_kv_wg(const ConvTcParams p) {
    using namespace kx3;
    constexpr bool X3 = MODE == 2;
    constexpr int EPC = MODE == 1 ? 8 : 4;                         // channels per 16-byte chunk
    constexpr int KMAIN = MODE == 1 ? K_BF16 : K_TF32;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sS = smem;                                            // [STAGES][X | Wk | Wv]
    uint8_t* kp = sS + STAGES * STAGE;                             // K, then P (fp32)
    uint8_t* vt = kp + OPI;                                        // V (fp32)
    uint8_t* pc = vt + OPI;                                        // Pc fp16 pairs (fp32x3)
    uint8_t* vc = pc + OPI;                                        // Vc fp16 pairs (fp32x3)
    float* s_mx = reinterpret_cast<float*>(vc + OPI);              // [2 halves][128 rows]
    float* s_z = s_mx + 2 * 128;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_z + 2 * 128);

    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // (warp-uniform, see sbk_conv_tc.cu)
    const int HW = p.H * p.W;
    const int ksteps = p.c0 / (KCH * EPC);
    const int ksteps_t = X3 ? 2 * ksteps : ksteps;                 // fp32x3: correction + main sub-stage per 32 channels
    const int items = (HW + PX - 1) / PX;                          // items per sample
    const int total = p.B * items;
    const uint32_t bar0 = smem_u32(bars);
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (STAGES + s); };

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        const int wg = warp >> 2, wt = tid & 127;
        const int row = tid & 127, half = tid >> 7;                // softmax: one row, half of the item's pixels
        constexpr uint32_t D_HI = desc_hi(128);
        const uint32_t s0 = smem_u32(sS);
        uint32_t it = 0;
        for (int t = blockIdx.x; t < total; t += gridDim.x) {
            const int b = t / items, mt = t - b * items;
            // ---- projection: warpgroup 0 -> K^T, warpgroup 1 -> V^T  (64 pixels x 128 rows)
            float acc[64];
            if constexpr (X3) {
                // K stage kb = ring stages it (correction weights) and it + 1 (x, main weights): correction MMAs, then main
                for (int kb = 0; kb < ksteps; ++kb, it += 2) {
                    const int sc = it % STAGES, sm = (it + 1) % STAGES;
                    mbar_wait(full(sc), (it / STAGES) & 1);
                    mbar_wait(full(sm), ((it + 1) / STAGES) & 1);
                    const uint32_t xc = s0 + sc * STAGE, xm = s0 + sm * STAGE;
                    uint8_t* cx = (kb & 1) ? vc : pc;
                    {
                        const float4* src = reinterpret_cast<const float4*>(sS + sm * STAGE);
#pragma unroll
                        for (int i = tid; i < XS / 16; i += 256) {
                            const float4 v = src[i];
                            reinterpret_cast<float4*>(cx)[i] = corr_chunk(v.x, v.y, v.z, v.w);
                        }
                    }
                    fence_proxy_async();                           // converted chunks -> visible to the tensor core
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    const uint32_t c_lo = desc_lo(smem_u32(cx), PX * 16), x_lo = desc_lo(xm, PX * 16);
                    const uint32_t wc_lo = desc_lo(xc + XS + wg * (KCH * 128 * 16), 128 * 16), wm_lo = desc_lo(xm + XS + wg * (KCH * 128 * 16), 128 * 16);
                    wg_fence();
#pragma unroll
                    for (int kk = 0; kk < KCH / 2; ++kk)
                        wgmma<128, K_F16>(acc, desc_pack(c_lo + (uint32_t)(kk * 2 * PX), D_HI), desc_pack(wc_lo + (uint32_t)(kk * 2 * 128), D_HI),
                                          (kb | kk) != 0 ? 1u : 0u);
#pragma unroll
                    for (int kk = 0; kk < KCH / 2; ++kk)
                        wgmma<128, K_TF32>(acc, desc_pack(x_lo + (uint32_t)(kk * 2 * PX), D_HI), desc_pack(wm_lo + (uint32_t)(kk * 2 * 128), D_HI), 1u);
                    wg_commit();
                    wg_wait<0>();
                    wg_fence_regs(acc);
                    __syncwarp();
                    if (lane == 0) { mbar_arrive(empty(sc)); mbar_arrive(empty(sm)); }
                }
            } else
            for (int ks = 0; ks < ksteps_t; ++ks, ++it) {
                const int s = it % STAGES;
                mbar_wait(full(s), (it / STAGES) & 1);
                const uint32_t xs = s0 + s * STAGE;
                const uint32_t x_lo = desc_lo(xs, PX * 16), w_lo = desc_lo(xs + XS + wg * (KCH * 128 * 16), 128 * 16);
                auto issue = [&](auto kind) {
#pragma unroll
                    for (int kk = 0; kk < KCH / 2; ++kk)
                        wgmma<128, decltype(kind)::value>(acc, desc_pack(x_lo + (uint32_t)(kk * 2 * PX), D_HI),
                                                          desc_pack(w_lo + (uint32_t)(kk * 2 * 128), D_HI), (ks | kk) != 0 ? 1u : 0u);
                };
                wg_fence();
                issue(std::integral_constant<int, KMAIN>{});
                wg_commit();
                wg_wait<0>();
                wg_fence_regs(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty(s));
            }
            // ---- K^T / V^T fragments -> [pixel chunk][row][16 B] images
            {
                uint8_t* img = wg == 0 ? kp : vt;
#pragma unroll
                for (int i = 0; i < 64; ++i) {
                    const int px = frag_row(wt, i), r = frag_col(wt, i);
                    *reinterpret_cast<float*>(img + ((size_t)(px / 4) * 128 + r) * 16 + (px % 4) * 4) = acc[i];
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // ---- softmax over the item's pixels: max, P = exp(k - max) in place, row sums
            const int nvalid = min(PX, HW - mt * PX) - half * (PX / 2);   // valid pixels of this thread's half (may be <= 0)
            float kr[PX / 2];
#pragma unroll
            for (int c = 0; c < PX / 8; ++c) {
                const float4 q = *reinterpret_cast<const float4*>(kp + ((size_t)(half * (PX / 8) + c) * 128 + row) * 16);
                kr[4 * c] = q.x; kr[4 * c + 1] = q.y; kr[4 * c + 2] = q.z; kr[4 * c + 3] = q.w;
            }
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < PX / 2; ++i) mx = fmaxf(mx, i < nvalid ? kr[i] : -INFINITY);
            s_mx[half * 128 + row] = mx;
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const float md = fmaxf(s_mx[row], s_mx[128 + row]);
            float z0 = 0.f, z1 = 0.f;
#pragma unroll
            for (int i = 0; i < PX / 2; i += 2) {                  // (pixels past the image hold k = 0: finite, then selected away)
                const float e0 = i < nvalid ? (X3 ? expf(kr[i] - md) : __expf(kr[i] - md)) : 0.f;
                const float e1 = i + 1 < nvalid ? (X3 ? expf(kr[i + 1] - md) : __expf(kr[i + 1] - md)) : 0.f;
                z0 += e0; z1 += e1;
                kr[i] = e0; kr[i + 1] = e1;
            }
            s_z[half * 128 + row] = z0 + z1;
#pragma unroll
            for (int c = 0; c < PX / 8; ++c) {
                const size_t o = ((size_t)(half * (PX / 8) + c) * 128 + row) * 16;
                const float e0 = kr[4 * c], e1 = kr[4 * c + 1], e2 = kr[4 * c + 2], e3 = kr[4 * c + 3];
                *reinterpret_cast<float4*>(kp + o) = make_float4(e0, e1, e2, e3);
                if constexpr (X3) {
                    // Pc = {P_lo * 2^8, P * 2^-4},  Vc = {V * 2^-8, V_lo * 2^4}: one 16-byte chunk per 4 pixels
                    *reinterpret_cast<uint4*>(pc + o) =
                        make_uint4(f16x2_sat(tf32_lo(e0) * 256.f, tf32_lo(e1) * 256.f), f16x2_sat(tf32_lo(e2) * 256.f, tf32_lo(e3) * 256.f),
                                   f16x2_sat(e0 * 0.0625f, e1 * 0.0625f), f16x2_sat(e2 * 0.0625f, e3 * 0.0625f));
                    const float4 v = *reinterpret_cast<const float4*>(vt + o);
                    *reinterpret_cast<uint4*>(vc + o) =
                        make_uint4(f16x2_sat(v.x * 0.00390625f, v.y * 0.00390625f), f16x2_sat(v.z * 0.00390625f, v.w * 0.00390625f),
                                   f16x2_sat(tf32_lo(v.x) * 16.f, tf32_lo(v.y) * 16.f), f16x2_sat(tf32_lo(v.z) * 16.f, tf32_lo(v.w) * 16.f));
                }
            }
            fence_proxy_async();                                   // operand images in smem -> visible to the tensor core
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // ---- context: warpgroup wg, rows and columns 64 wg .. 64 wg + 63 (heads 2 wg, 2 wg + 1)
            float sacc[32];
            {
                const uint32_t p_lo = desc_lo(smem_u32(kp) + 64 * wg * 16, 128 * 16), v_lo = desc_lo(smem_u32(vt) + 64 * wg * 16, 128 * 16);
                const uint32_t pc_lo = desc_lo(smem_u32(pc) + 64 * wg * 16, 128 * 16), vc_lo = desc_lo(smem_u32(vc) + 64 * wg * 16, 128 * 16);
                wg_fence();
                if constexpr (X3) {
#pragma unroll
                    for (int kk = 0; kk < PX / 8; ++kk)            // correction: K = 16 fp16 = 8 pixels x {P_lo V, P V_lo}
                        wgmma<64, K_F16>(sacc, desc_pack(pc_lo + (uint32_t)(kk * 2 * 128), D_HI), desc_pack(vc_lo + (uint32_t)(kk * 2 * 128), D_HI),
                                         kk != 0 ? 1u : 0u);
                }
#pragma unroll
                for (int kk = 0; kk < PX / 8; ++kk)                // main: K = 8 pixels, P and V read as tf32 (P_hi V_hi)
                    wgmma<64, K_TF32>(sacc, desc_pack(p_lo + (uint32_t)(kk * 2 * 128), D_HI), desc_pack(v_lo + (uint32_t)(kk * 2 * 128), D_HI),
                                      (X3 || kk != 0) ? 1u : 0u);
                wg_commit();
                wg_wait<0>();
                wg_fence_regs(sacc);
            }
            // ---- partials of this item: max, sum (softmax threads of the first half), diagonal S blocks (fragments)
            float* pt0 = p.kv_part + ((long long)b * items + mt) * kHeads * kKvPartFloats;
            if (half == 0) {
                float* pt = pt0 + (row / 32) * kKvPartFloats;
                pt[row % 32] = md;
                pt[32 + row % 32] = s_z[row] + s_z[128 + row];
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int dl = frag_row(wt, i), el = frag_col(wt, i);
                if ((dl >> 5) == (el >> 5)) {
                    float* pt = pt0 + (2 * wg + (dl >> 5)) * kKvPartFloats;
                    pt[64 + (dl & 31) * 32 + (el & 31)] = sacc[i];
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");        // the images are rewritten by the next item
        }
    } else {
        // ---------------------------------------------------------------- loader warp: weights + activation runs (cp.async.bulk)
        // lane 0 owns the ring protocol and the weight copy; lanes 0-7 each issue the activation runs of one channel chunk
        uint32_t it = 0;
        const int chs = p.c0 / EPC;
        for (int t = blockIdx.x; t < total; t += gridDim.x) {
            const int b = t / items, mt = t - b * items;
            const int m0 = mt * PX, m_hi = m0 + PX < HW ? m0 + PX : HW;
            const int hh0 = m0 / p.W, ww0 = m0 - hh0 * p.W;
            for (int ks = 0; ks < ksteps_t; ++ks, ++it) {
                const int s = it % STAGES;
                const int kb = X3 ? ks >> 1 : ks;
                const bool corr = X3 && (ks & 1) == 0;
                const uint32_t xs = smem_u32(sS) + s * STAGE;
                if (lane == 0) {
                    mbar_wait(empty(s), ((it / STAGES) & 1) ^ 1);
                    mbar_arrive_expect_tx(full(s), corr ? WS : STAGE);
                    bulk_g2s(xs + XS, reinterpret_cast<const uint8_t*>(p.wpk) + (size_t)(X3 ? 2 * kb + (corr ? 1 : 0) : ks) * WS, WS, full(s));
                }
                __syncwarp();
                if (lane < KCH && !corr) {
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.in0);
                    const int k = lane, cl = kb * KCH + k;
                    int m = m0, hh = hh0, ww = ww0, qx = 0;
                    while (m < m_hi) {                             // split the flattened run at image-row boundaries
                        const int n = (p.W - ww) < (m_hi - m) ? (p.W - ww) : (m_hi - m);
                        bulk_g2s(xs + (k * PX + qx) * 16, src + (((long long)(b * p.H + hh) * chs + cl) * p.W + ww) * 16,
                                 (uint32_t)n * 16u, full(s));
                        m += n; qx += n; ++hh; ww = 0;
                    }
                    if (qx < PX) bulk_g2s(xs + (k * PX + qx) * 16, p.zero_page, (uint32_t)(PX - qx) * 16u, full(s));
                }
            }
        }
    }
}

template <int MODE>
static int launch_kv(const ConvTcParams& p, cudaStream_t s) {
    static DevCache cache;
    const int num_sms = cache.get(reinterpret_cast<const void*>(k_attn_kv_wg<MODE>));
    if (num_sms <= 0) return -1;
    if (p.c0 % (kx3::KCH * (MODE == 1 ? 8 : 4)) != 0) return -1;
    const long long total = (long long)p.B * ((p.H * p.W + kx3::PX - 1) / kx3::PX);
    const int grid = (int)(total < num_sms ? total : num_sms);
    k_attn_kv_wg<MODE><<<grid, kx3::THREADS, kx3::SMEM, s>>>(p);
    return 1;
}

int attn_kv_tile_pixels() { return kx3::PX; }
int launch_attn_kv(const ConvTcParams& p, cudaStream_t s) {
    return p.form == FORM_X3 ? launch_kv<2>(p, s) : p.form == FORM_BF16 ? launch_kv<1>(p, s) : launch_kv<0>(p, s);
}

}  // namespace sbk
