// Warpgroup-MMA (wgmma) implicit-GEMM convolutions for sm_90a: the 3x3 Block convs (81.5 % of the step's MACs), the
// 1x1 channel mixes (res_conv, attention apply), Downsample / Upsample, the vocoder's dilated Conv1d and the 7x7 convs of
// DiffVC's PostNet (G_C7: one kernel row per ring stage, see Geo<G_C7>).  tf32 (or bf16)
// operands from shared memory, fp32 accumulation in registers.
//
//   D[pixel][cout] (fp32, registers) += A[pixel][tap, cin] (smem) * W[cout][tap, cin] (smem)
//
// Mapping.  One CTA owns one row of TPX = 128 pixels x NT output channels of one sample; each of its two consumer
// warpgroups owns 64 of the pixels (one m64nNT wgmma per tap and K step).  For the 3x3 conv a row is 128 consecutive
// frames of one mel bin; for 1x1 convs the image is flattened and a row is any 128 consecutive pixels.  A 3x3 tile may
// also be two rows x 128 pixels x 64 channels (Geo<G_C3, 2>): each consumer warpgroup owns one row, and every weight stage
// feeds twice the pixels.  The consumers hold up to 128 accumulator registers (fp32x3: accumulators + running sums)
// because the producer warpgroup hands its registers over (setmaxnreg).
//
// A operand.  Conv inputs are stored in HBM already in operand form (masked; Block activations GroupNorm-ed, Mish-ed
// and time-biased by k_gn_act, see sbk_kernels.cu), so producing the A tile is a pure copy straight into the wgmma
// no-swizzle K-major layout [16 B channel chunk][halo row][pixel][16 B].  In that layout eight consecutive pixels x 16 B
// are one core matrix, so EVERY one of the nine taps is only a different descriptor start address into the same halo
// tile (start += (r*130 + s)*16 B): each input element is fetched once per CTA and feeds nine MMAs.
//
// B operand.  Weights are packed on the host into exactly the per-stage shared-memory image
// [tap][chunk][cout][16 B] and streamed with one cp.async.bulk per stage, mbarrier complete_tx.
//
// Pipeline.  STAGES-deep ring with full_a / full_b / empty mbarriers; a loader warp (the first warp of the producer
// warpgroup) fills it with bulk copies (the
// Downsample gathers are cp.async issued by the consumers themselves) while the consumer warpgroups issue one stage's
// MMAs back to back as one wgmma group.  fp32x3 keeps that group in flight while it issues the next stage's and frees a
// stage once the group after it has been issued; tf32 / bf16 (and Downsample) wait for each group and then free its
// stage.  The epilogue stages the accumulators through shared memory ([pixel][column]), so one thread owns one pixel and
// a contiguous run of output channels.
// All waits are bounded spins that trap instead of hanging the GPU.
#include "sbk_tc.cuh"

#include <cuda_fp16.h>
#include <string.h>
#include <type_traits>

namespace sbk {

namespace tc {

constexpr int TPX = 128;              // pixels per row = 2 consumer warpgroups x wgmma M (64)
constexpr int NCONS = 256;            // consumer threads (2 warpgroups): MMAs + epilogue (Downsample: + A gathers)
constexpr int NTHREADS = NCONS + 128; // + producer warpgroup: its first warp is the loader; the other three exit, or derive
                                      // the fp32x3 correction operand in shared memory (NCONV converter threads)
constexpr int NCONV = 96;
// Register split (setmaxnreg): the CTA starts with 65536 / 384 registers per thread; the producer warpgroup gives most of
// its share back so that the consumers can hold a 128-register accumulator tile (+ fp32x3 running sums) without spilling.
constexpr int PROD_REGS = 40, CONS_REGS = 232;
static_assert(128 * PROD_REGS + NCONS * CONS_REGS <= 65536, "register file");

// geometry of the A tile in shared memory, [16-byte K chunk][row][pixel][16 B]; ROWS output rows of TPX pixels per tile,
// NACC accumulators per consumer thread
template <int GEOM, int R = 1> struct Geo;
// 3x3: halo tile of R + 2 input rows.  R = 1: consumer warpgroup w owns pixels 64w..64w+63 of the row.  R = 2: warpgroup w
// owns output row h0 + w, i.e. two m64 pixel blocks (two accumulators) that share every weight descriptor - each weight
// byte brought to shared memory feeds twice the pixels.
template <int R> struct Geo<G_C3, R> {
    static_assert(R == 1 || R == 2, "3x3 tiles are 1 or 2 rows");
    static constexpr int ROWS = R, HR = R + 2, PXP = TPX + 2, TAPS = 9, KCH = 2, NACC = R;
};
template <> struct Geo<G_PW> { static constexpr int ROWS = 1, HR = 1, PXP = TPX, TAPS = 1, KCH = 8, NACC = 1; };           // 1x1: plain tile
// 3x3 stride 2 (Downsample): 3 input rows; input columns de-interleaved into an odd plane (129 px: 2*w0-1+2i) and
// an even plane (2*w0+2i) so that consecutive OUTPUT pixels read consecutive smem pixels for every tap.
template <> struct Geo<G_DOWN> { static constexpr int ROWS = 1, HR = 3, PXP = 2 * (TPX + 1), TAPS = 9, KCH = 2, NACC = 1; };
// ConvTranspose2d(4,2,1) (Upsample): per output parity (ph,pw) a 2x2-tap conv over the same 3x3-style input halo;
// all four phases are computed from one halo tile into 4 accumulators; the stage carries all 16 (kh,kw) taps.
template <> struct Geo<G_UP> { static constexpr int ROWS = 1, HR = 3, PXP = TPX + 2, TAPS = 16, KCH = 2, NACC = 4; };

// Conv1d, K taps, runtime dilation d (HiFi-GAN V1: K in {3,7,11}, d in {1,3,5}; halo (K-1)*d <= 50 samples): ONE strip of
// TPX + HALO samples per channel chunk; tap t is the descriptor start t*d samples into it - each input sample is fetched
// once for all taps.  HALO = 64, or 128 for the wide geometries G_C1K*W (V3's K = 7 at d = 12: 72 samples); the strip
// width only changes the A tile, so both widths read the same weight image.
template <int K, int HALO = 64> struct GeoC1 { static constexpr int ROWS = 1, HR = 1, PXP = TPX + HALO, TAPS = K, KCH = 2, NACC = 1; };
template <> struct Geo<G_C1K3> : GeoC1<3> {};
template <> struct Geo<G_C1K5> : GeoC1<5> {};
template <> struct Geo<G_C1K7> : GeoC1<7> {};
template <> struct Geo<G_C1K11> : GeoC1<11> {};
template <> struct Geo<G_C1K3W> : GeoC1<3, 128> {};
template <> struct Geo<G_C1K5W> : GeoC1<5, 128> {};
template <> struct Geo<G_C1K7W> : GeoC1<7, 128> {};
template <> struct Geo<G_C1K11W> : GeoC1<11, 128> {};
static_assert(Geo<G_C1K3>::PXP == TPX + conv_tc_c1_halo(G_C1K3) && Geo<G_C1K3W>::PXP == TPX + conv_tc_c1_halo(G_C1K3W), "strip widths");
// (a wide strip row is the longest run copied from ConvTcParams::zero_page)
static_assert(Geo<G_C1K3W>::PXP * 16 <= 4096, "zero page");

// 7x7, pad 3 (PostNet): a 3x3-style stage (halo tile + all taps of one 8-channel K step) would carry 49 x 2 x NT x 16 B
// of weights - 200 KB at NT = 128 - and leave no room for a second stage.  A K step is therefore split by kernel row:
// stage (K step, kernel row r) holds ONE input row of TPX + 6 pixels per channel chunk (4.3 KB) and the 7 taps of row r
// (28 KB at NT = 128); tap s is the descriptor start s pixels into the row, as in the 3x3 halo tile.  Every input row is
// fetched by up to 7 stages of a tile (from L2 after the first), ~15 % of the weight bytes.
template <> struct Geo<G_C7> { static constexpr int ROWS = 1, HR = 1, PXP = TPX + 6, TAPS = 7, KCH = 2, NACC = 1; };
// (the weight image's stage shape, sbk_internal.h: conv_tc_wimg)
static_assert(Geo<G_PW>::KCH == conv_tc_kch(G_PW) && Geo<G_C3>::KCH == conv_tc_kch(G_C3) && Geo<G_C7>::KCH == conv_tc_kch(G_C7) &&
              Geo<G_C7>::TAPS * conv_tc_stage_rows(G_C7) == conv_tc_taps(G_C7), "weight-image stage shape");

}  // namespace tc

using namespace tc;


// Persistent CTAs (one per SM: each CTA loops over output tiles round-robin) with as deep a ring as shared memory
// allows next to the epilogue's [TPX][NT + 4] fp32 staging tile (a 2-row tile passes through it one m64 block pair at a time).
template <int GEOM, int NT, int R = 1> struct Depth {
    using G = Geo<GEOM, R>;
    static constexpr int STAGE_BYTES = G::KCH * G::HR * G::PXP * 16 + G::TAPS * G::KCH * NT * 16;
    static constexpr int LDS = NT + 4;                       // staging row pitch (floats): conflict-free float4 reads
    static constexpr int SD_BYTES = TPX * LDS * 4;
    static constexpr int FIT = (220 * 1024 - SD_BYTES) / STAGE_BYTES;
    static constexpr int STAGES = FIT > 6 ? 6 : FIT;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + SD_BYTES + 3 * STAGES * 8 + 128 * 4 * G::ROWS + 3 * NT * 4 + 64;
    static_assert(STAGES >= 2, "need at least 2 stages");
    static_assert(SMEM <= 227 * 1024, "shared memory budget");
};
// fp32x3 derives a correction sub-stage's A tile from the main sub-stage that FOLLOWS it in the ring, so stage g is full
// only once stage g + 1 has landed.  A consumer that waits for stage g has released every
// stage up to g - 2 (one MMA group in flight), and the loader fills stage g + 1 once stage g + 1 - STAGES is released:
// g + 1 - STAGES <= g - 2, i.e. three stages.  (Downsample's consumers gather stage g + 1 themselves before they convert
// it, LAG = STAGES - 2 >= 1 stages ahead of the MMAs: three stages again.)
template <int GEOM, int NT, int R> constexpr bool x3_depth_ok = Depth<GEOM, NT, R>::STAGES >= 3;

// RES: ResnetBlock-tail epilogue (1x1 res_conv + Mish(GN(h2raw)) side input), compile-time so that the plain 1x1 /
// 3x3 instantiations do not pay its registers.
//
// X3 (fp32x3 mode, FORM_X3): two sub-stages per K stage (the f16 correction MMAs over the packed fp16 chunks, then the tf32
// main MMAs - sbk_internal.h: corr_chunk) AND chunked accumulation.  The tensor core truncates its fp32 accumulator on
// every MMA (a bias of ~2^-25 |acc| per instruction towards zero), so a single accumulation run over the hundreds of MMAs
// of a 3x3 conv would lose several 1e-6 relative - more than the fp32 rounding of the reference's own sums.  An
// accumulation run is therefore cut every FLUSH sub-stages and the partial sums are added in round-to-nearest fp32 into a
// second register array.  (Upsample runs unchunked: its runs are short, 4 taps per phase.)
//
// VOC: the vocoder's output forms (ConvTcParams::voc) on a 1x1 GEMM; the Conv1d geometries always use them.  They only
// differ from the sampler's in the bf16 mode (an output is bf16 only when it is an activated operand).
template <int GEOM, bool BF16, int NT, bool RES, bool X3, bool VOC = false, int R = 1>
__device__ __forceinline__ void conv_tc_body(const ConvTcParams& p) {
    static_assert(!(X3 && BF16), "fp32x3 runs on tf32 operands");
    using G = Geo<GEOM, R>;
    using D = Depth<GEOM, NT, R>;
    constexpr int NACC = G::NACC, ROWS = G::ROWS;
    constexpr bool ROW2 = ROWS == 2;                       // 3x3, 2-row tile: accumulator a = pixel block a of the row
    constexpr bool CHUNKED = X3 && GEOM != G_UP;
    // sub-stages per accumulation run: 6 = three K stages of correction + main sub-stage, 54 MMAs per accumulator for a
    // 3x3 conv (7x7: three (K step, kernel row) stages, 42 MMAs)
    const int FLUSH = CHUNKED ? 6 : (1 << 30);
    constexpr int STAGES = D::STAGES, LDS = D::LDS;
    constexpr int LAG = STAGES >= 3 ? STAGES - 2 : 0;      // G_DOWN only: cp.async groups in flight behind the newest
    constexpr int HR = G::HR, PXP = G::PXP, TAPS = G::TAPS, KCH = G::KCH;
    constexpr int EPC = BF16 ? 8 : 4;                      // elements per 16-byte channel chunk
    constexpr int CPS = KCH * EPC;                         // input channels per stage
    constexpr bool C1 = geom_is_c1(GEOM);                  // Conv1d strip geometry
    // bf16 mode: the raw Block-conv outputs (GroupNorm inputs) stay fp32 [C/4]; every other output is an operand tensor
    // of a later tensor-core kernel and is written as bf16 [B][H][C/8][W][8].  The vocoder's forms (VF16) instead pick
    // the dtype per output: bf16 for an activated output (act_out) and the second output act, fp32 for the others.
    constexpr bool VF16 = BF16 && (C1 || VOC);
    constexpr bool OUT16 = BF16 && GEOM != G_C3 && !VF16;
    constexpr int PLANE = HR * PXP * 16;                   // bytes between K chunks of the A tile
    constexpr int A_STAGE_BYTES = KCH * PLANE;
    constexpr int B_STAGE_BYTES = TAPS * KCH * NT * 16;
    constexpr bool BULK = GEOM != G_DOWN;                  // A tile = contiguous runs -> cp.async.bulk (no LSU work)
    constexpr int SPAN = TPX;                              // output pixels per tile along W
    constexpr int FR = NT / 2;                             // accumulator registers per thread and accumulator
    constexpr int KMAIN = BF16 ? K_BF16 : K_TF32;

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sA = smem;                                            // [STAGES][KCH][HR][PXP][16]
    uint8_t* sB = sA + STAGES * A_STAGE_BYTES;                     // [STAGES][TAPS][KCH][NT][16]
    float* sD = reinterpret_cast<float*>(sB + STAGES * B_STAGE_BYTES);            // [TPX][LDS] accumulator staging
    uint64_t* bars = reinterpret_cast<uint64_t*>(sD + TPX * LDS);                 // full_b[S], empty[S], full_a[S]
    // GroupNorm partials of the current tile: one private slot row per consumer warp (plain read-modify-write by lane 0,
    // no atomics), summed in a fixed order at the end of the tile and flushed as fp64 -> the totals can only differ between
    // runs through the order of the fp64 global atomics (1e-16), so the fp32 mean / rstd - and the sampler - are reproducible.
    // A 2-row tile keeps one slot set per output row, and a slot row is the warp that covers the same pixels in a 1-row tile,
    // so every row's fp64 total receives exactly the fp32 partials a 1-row tile would flush.
    float* s_st = reinterpret_cast<float*>(bars + 3 * STAGES);                    // [ROWS][8 warps][8 groups][2]
    float* s_rg = s_st + 128 * ROWS;                                              // EPI_RES: mean|scale|beta [NT] each

    // (the warp index is broadcast from lane 0 so that the compiler can prove the role branches warp-uniform: wgmma code
    // under a branch it considers divergent is serialised)
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    const int Cin = p.c0 + p.c1;
    const int HW = p.H * p.W;
    const int ksteps = Cin / CPS * conv_tc_stage_rows(GEOM);            // ring stages per tile (7x7: one per K step and kernel row)
    // fp32x3 mode: each K stage runs twice - the f16 correction sub-stage (x_lo*w + x*w_lo from the packed fp16 chunks,
    // sbk_internal.h: corr_chunk) first, then the tf32 main sub-stage (x_hi*w_hi): small terms first
    const int ksteps_t = X3 ? 2 * ksteps : ksteps;
    // fp32x3: the correction sub-stage's A tile is corr_chunk of the main sub-stage's tile, computed in shared memory - by
    // the converter warps of the producer warpgroup for the bulk-copy geometries, by the gathering consumers themselves for
    // Downsample.  The tile is converted whole, so the zero padding (border columns, out-of-image rows, the ragged end of a
    // 1x1 tile) becomes zero chunks and needs no pattern logic.
    static_assert(!X3 || x3_depth_ok<GEOM, NT, R>, "in-SM correction operand: stage g needs stage g + 1, three stages");
    // ---- tile space: (sample, pixel tile, N tile), N tile fastest so neighbours in time share the A tile in L2
    const int wt_w = (GEOM == G_DOWN ? p.Wo : p.W), wt_h = (GEOM == G_DOWN ? p.Ho : p.H);
    const int wtiles = (wt_w + SPAN - 1) / SPAN;
    const int mtiles = GEOM == G_PW ? (HW + TPX - 1) / TPX : wtiles * ((wt_h + ROWS - 1) / ROWS);
    const int ntn = p.Cout / NT;
    const int total_tiles = p.B * mtiles * ntn;
    auto decode = [&](int t, int& b, int& h0, int& w0, int& n0) {
        const int nt = t % ntn; const int r = t / ntn;
        const int mt = r % mtiles; b = r / mtiles; n0 = nt * NT;
        if (GEOM == G_PW) { w0 = 0; h0 = mt; }
        else { w0 = (mt % wtiles) * SPAN; h0 = (mt / wtiles) * ROWS; }
    };

    const uint32_t bar0 = smem_u32(bars);
    auto full_b = [&](int s) { return bar0 + 8u * s; };                       // weights (+ bulk A runs): tx-count
    auto empty = [&](int s) { return bar0 + 8u * (STAGES + s); };             // every consumer warp done with the stage
    auto full_a = [&](int s) { return bar0 + 8u * (2 * STAGES + s); };        // G_DOWN cp.async producers

    // ---- one-time setup
    if (tid == 0) {
        // full_a: one arrival per warp that writes A tiles from registers (Downsample's consumers, else the converter warps)
        constexpr int A_WARPS = X3 && BULK ? NCONV / 32 : NCONS / 32;
        for (int s = 0; s < STAGES; ++s) { mbar_init(full_a(s), A_WARPS); mbar_init(full_b(s), 1); mbar_init(empty(s), NCONS / 32); }
        fence_barrier_init();
    }
    if (tid < 128 * ROWS) s_st[tid] = 0.f;
    __syncthreads();

    if (warp < NCONS / 32) {
        // =========================================================================================================
        // consumer warpgroups: (G_DOWN: cp.async A producers,) MMAs, epilogue of every tile
        // =========================================================================================================
        setmaxnreg_inc<CONS_REGS>();
        const int wg = warp >> 2, wt = tid & 127;                  // warpgroup = pixel half of the tile (2-row tile: its row)
        uint32_t it = 0;                                           // ring counter (stages consumed by this CTA)
        // ---- A producers (Downsample only): 16-byte cp.async gathers that de-interleave even/odd columns
        constexpr int SLOTS = HR * PXP * KCH;
        constexpr int PER = BULK ? 1 : (SLOTS + NCONS - 1) / NCONS;
        uint32_t sl_dst[PER]; long long sl_off[PER]; int sl_chunk[PER]; bool sl_ok[PER];
        const uint32_t a0 = smem_u32(sA), b0 = smem_u32(sB);
        constexpr uint32_t D_HI = desc_hi(128);                    // SBO = 128 B for both operands
        float acc[NACC][FR];
        float sum[CHUNKED ? NACC : 1][CHUNKED ? FR : 1];
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            int b, h0, w0, n0;
            decode(t, b, h0, w0, n0);
            if constexpr (!BULK) {
#pragma unroll
                for (int j = 0; j < PER; ++j) {
                    const int e = tid + j * NCONS;
                    const bool in = e < SLOTS;
                    const int k = in ? e / (HR * PXP) : 0, item = in ? e - k * (HR * PXP) : 0;     // pixel fastest
                    const int r = item / PXP, q = item - r * PXP;
                    const int par = q / (TPX + 1), i = q - par * (TPX + 1);      // plane 0: odd columns, plane 1: even
                    const int hi = 2 * h0 - 1 + r, wi = par == 0 ? 2 * w0 - 1 + 2 * i : 2 * w0 + 2 * i;
                    const bool ok = in && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W && !(par == 1 && i == TPX);
                    sl_ok[j] = ok; sl_chunk[j] = k;
                    sl_off[j] = (ok ? (long long)(b * p.H + hi) : 0) * 1048576 + (ok ? wi : 0);   // pack (row, w)
                    sl_dst[j] = in ? (uint32_t)(k * PLANE + (r * PXP + q) * 16) : 0xFFFFFFFFu;
                }
            }
            auto produce = [&](int ks) {
                const uint32_t g = it + ks;
                const int s = g % STAGES;
                mbar_wait(empty(s), ((g / STAGES) & 1) ^ 1);
                if (X3 && (ks & 1) == 0) return;           // correction sub-stage: converted from the main sub-stage's gathers
                const int ck = (X3 ? ks / 2 : ks) * KCH;
                const bool second = ck * EPC >= p.c0;
                const uint8_t* src = reinterpret_cast<const uint8_t*>(second ? p.in1 : p.in0);
                const int chs = (second ? p.c1 : p.c0) / EPC;
                const int c0k = second ? ck - p.c0 / EPC : ck;
#pragma unroll
                for (int j = 0; j < PER; ++j) {
                    if (sl_dst[j] == 0xFFFFFFFFu) continue;
                    const long long row = sl_off[j] / 1048576, wi = sl_off[j] % 1048576;
                    const uint8_t* gp = src + ((row * chs + c0k + sl_chunk[j]) * p.W + wi) * 16;
                    cp_async16(a0 + s * A_STAGE_BYTES + sl_dst[j], gp, sl_ok[j] ? 16u : 0u);
                }
            };
            auto release = [&](uint32_t g) {                        // this warp's MMAs of stage g have completed
                __syncwarp();
                if (lane == 0) mbar_arrive(empty(g % STAGES));
            };
            // conv: a correction sub-stage whose A tile the converter warps write.  Its full_a only completes a phase when the
            // buffer holds a correction sub-stage: every turn of the ring when STAGES is even (even buffers always do), every
            // second turn when it is odd.
            auto wait_full = [&](uint32_t g, bool conv = false) {
                const int s = g % STAGES;
                const uint32_t ph = (g / STAGES) & 1;
                if (!BULK) mbar_wait(full_a(s), ph);
                else if (conv) mbar_wait(full_a(s), (g / (STAGES % 2 ? 2 * STAGES : STAGES)) & 1);
                mbar_wait(full_b(s), ph);                  // weights (+ the A runs when they are bulk copies)
            };
            // MMAs of ring stage g as one wgmma group; first: g starts an accumulation run (the first MMA overwrites)
            // (kind: the MMA kind of the sub-stage as a compile-time constant, so no branch separates the wgmmas of a run)
            auto issue = [&](uint32_t g, bool first, auto kind) {
                constexpr int KD = decltype(kind)::value;
                const int s = g % STAGES;
                // this warpgroup's 64 pixels (2-row tile: its halo row; block a of the row adds 64 a)
                const uint32_t a_lo = desc_lo(a0 + s * A_STAGE_BYTES, PLANE) + (uint32_t)(ROW2 ? wg * PXP : 64 * wg);
                const uint32_t b_lo = desc_lo(b0 + s * B_STAGE_BYTES, NT * 16);
                const uint32_t dil = C1 ? (uint32_t)p.dil : 0u;
                wg_fence();
#pragma unroll
                for (int kk = 0; kk < KCH / 2; ++kk) {
                    const uint32_t a_k = a_lo + (uint32_t)(kk * 2 * (PLANE / 16)), b_k = b_lo + (uint32_t)(kk * 2 * NT);
                    if (GEOM == G_UP) {
                        // ho = 2*hi - 1 + kh: parity ph uses (kh=1,dh=0),(kh=3,dh=-1) if ph=0 and (kh=0,dh=+1),(kh=2,dh=0) if ph=1
#pragma unroll
                        for (int phase = 0; phase < 4; ++phase) {
                            const int pph = phase >> 1, pw = phase & 1;
#pragma unroll
                            for (int t2 = 0; t2 < 4; ++t2) {
                                const int a = t2 >> 1, bb = t2 & 1;
                                const int kh = pph ? (a ? 2 : 0) : (a ? 3 : 1), kw = pw ? (bb ? 2 : 0) : (bb ? 3 : 1);
                                const int dh = pph ? (a ? 0 : 1) : (a ? -1 : 0), dw = pw ? (bb ? 0 : 1) : (bb ? -1 : 0);
                                wgmma<NT, KD>(acc[GEOM == G_UP ? phase : 0], desc_pack(a_k + (uint32_t)((1 + dh) * PXP + 1 + dw), D_HI),
                                              desc_pack(b_k + (uint32_t)((kh * 4 + kw) * KCH * NT), D_HI),
                                              (!first || (kk | t2) != 0) ? 1u : 0u);
                            }
                        }
                    } else {
#pragma unroll
                        for (int tap = 0; tap < TAPS; ++tap) {
                            const int r = TAPS == 9 ? tap / 3 : 0, sx = TAPS == 9 ? tap % 3 : (GEOM == G_C7 ? tap : 0);
                            // DOWN: input row r; column tap s reads the odd plane at x (s=0) / x+1 (s=2), the even plane at x (s=1)
                            const uint32_t aoff = GEOM == G_DOWN ? (uint32_t)(r * PXP + (sx == 1 ? TPX + 1 : (sx == 2 ? 1 : 0)))
                                                : C1 ? (uint32_t)tap * dil
                                                     : (uint32_t)(r * PXP + sx);
#pragma unroll
                            for (int a = 0; a < NACC; ++a)
                                wgmma<NT, KD>(acc[a], desc_pack(a_k + aoff + (uint32_t)(64 * a), D_HI),
                                              desc_pack(b_k + (uint32_t)(tap * KCH * NT), D_HI), (!first || (kk | tap) != 0) ? 1u : 0u);
                        }
                    }
                }
                wg_commit();
            };
            auto fence_acc = [&]() {
#pragma unroll
                for (int a = 0; a < NACC; ++a) wg_fence_regs(acc[a]);
            };
            constexpr auto kind_c = std::integral_constant<int, K_F16>{};     // fp32x3 correction sub-stage (even ks)
            constexpr auto kind_m = std::integral_constant<int, KMAIN>{};
            if constexpr (BULK && X3) {
                // One wgmma group in flight: sub-stage ks is issued while ks - 1 still runs, and stage ks - 1 is released
                // once wait<1> has retired it, so the tensor pipe does not drain between sub-stages.  The accumulators are
                // only read at the end of a run (every FLUSH sub-stages; Upsample: once per tile), after wait<0>; every
                // stage is released exactly once per consumer warp, one sub-stage late, the last one after wait<0>.
                // (tf32 / bf16 keep one wait per stage below: with nothing to fold their drains are short, and the stage
                // a consumer holds while its MMAs are in flight costs the loader more lead than the drains cost.)
                auto step = [&](int ks, bool first, auto kind) {
                    const uint32_t g = it + ks;
                    wait_full(g, decltype(kind)::value == K_F16);
                    issue(g, first, kind);
                    wg_wait<1>();                            // every group but g's has completed
                    __syncwarp();
                    if (lane == 0 && !first) mbar_arrive(empty((g - 1) % STAGES));
                };
                if constexpr (CHUNKED) {
                    // (the first MMA of a run ignores acc; defining it here ends its live range at the last fold of the
                    // previous tile, so the epilogue, which stages sum, can use its registers)
#pragma unroll
                    for (int a = 0; a < NACC; ++a)
#pragma unroll
                        for (int i = 0; i < FR; ++i) acc[a][i] = 0.f;
                }
                bool first_run = true;
                for (int ks = 0; ks < ksteps_t;) {
                    const int run_hi = ksteps_t - ks < FLUSH ? ksteps_t : ks + FLUSH;
                    bool first = true;
                    do {                                     // K stage: correction, then main sub-stage
                        step(ks, first, kind_c);
                        step(ks + 1, false, kind_m);
                        ks += 2;
                        first = false;
                    } while (ks < run_hi);
                    wg_wait<0>();
                    fence_acc();
                    release(it + ks - 1);
                    if constexpr (CHUNKED) {                 // fold the run into the running sums (round-to-nearest fp32)
                        if (first_run) {
#pragma unroll
                            for (int a = 0; a < NACC; ++a)
#pragma unroll
                                for (int i = 0; i < FR; ++i) sum[a][i] = acc[a][i];
                        } else {
#pragma unroll
                            for (int a = 0; a < NACC; ++a)
#pragma unroll
                                for (int i = 0; i < FR; ++i) sum[a][i] += acc[a][i];
                        }
                    }
                    first_run = false;
                }
            } else {
                // Each sub-stage's MMAs are waited for before its stage is released, and a finished run is folded
                // branch-free.  Downsample: the consumers themselves gather the A tile by cp.async, LAG stages ahead.
                auto compute = [&](int ks, auto kind) {
                    wait_full(it + ks);
                    const int run_lo = CHUNKED ? ks - ks % FLUSH : 0;
                    issue(it + ks, ks == run_lo, kind);
                    wg_wait<0>();
                    fence_acc();
                    release(it + ks);
                    if constexpr (CHUNKED) {
                        const bool first = run_lo == 0, last = ks == ksteps_t - 1 || ks - run_lo == FLUSH - 1;
#pragma unroll
                        for (int a = 0; a < NACC; ++a)
#pragma unroll
                            for (int i = 0; i < FR; ++i) sum[a][i] = last ? (first ? acc[a][i] : sum[a][i] + acc[a][i]) : sum[a][i];
                    }
                };
                if constexpr (BULK) {
                    for (int ks = 0; ks < ksteps_t; ++ks) compute(ks, kind_m);
                } else {
                    for (int ks = 0; ks < ksteps_t + LAG; ++ks) {
                        if (ks < ksteps_t) produce(ks);
                        cp_async_commit();                       // (empty groups past the last stage keep the accounting uniform)
                        if (ks >= LAG) {
                            const bool corr = X3 && ((ks - LAG) & 1) == 0;
                            if (X3 && corr) {
                                // Correction operand: this thread's gathers of the main sub-stage ks-LAG+1 (issued at
                                // iteration ks-LAG+1 <= ks) have landed; their corr_chunk goes to the same slots of the
                                // correction stage, whose previous occupant produce(ks-LAG) saw released.  Zero-filled
                                // slots (padding) convert to zero chunks.
                                static_assert(!X3 || LAG >= 1, "the main gather runs ahead of its correction sub-stage");
                                cp_async_wait<(LAG > 0 ? LAG - 1 : 0)>();
                                const uint32_t sc = (it + ks - LAG) % STAGES, sm = (it + ks - LAG + 1) % STAGES;
#pragma unroll
                                for (int j = 0; j < PER; ++j) {
                                    if (sl_dst[j] == 0xFFFFFFFFu) continue;
                                    const float4 v = *reinterpret_cast<const float4*>(sA + sm * A_STAGE_BYTES + sl_dst[j]);
                                    *reinterpret_cast<float4*>(sA + sc * A_STAGE_BYTES + sl_dst[j]) = corr_chunk(v.x, v.y, v.z, v.w);
                                }
                            }
                            cp_async_wait<LAG>();                // this thread's copies of stage ks-LAG have landed
                            fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor core
                            __syncwarp();
                            if (lane == 0) mbar_arrive(full_a((it + ks - LAG) % STAGES));
                            if (corr) compute(ks - LAG, kind_c);
                            else compute(ks - LAG, kind_m);
                        }
                    }
                }
            }
            it += ksteps_t;

            // ---- epilogue of tile t
            if constexpr (RES) {
                asm volatile("bar.sync 1, 256;" ::: "memory");        // previous tile's readers of s_rg are done
                const int cpg = p.Cout / kGroups;
                for (int i = tid; i < NT; i += NCONS) {
                    const int c = n0 + i, g = c / cpg;
                    const double sm_ = p.rgn.stats[(b * kGroups + g) * 2], ss = p.rgn.stats[(b * kGroups + g) * 2 + 1];
                    const double m = sm_ * (double)p.rgn.inv_count;
                    double var = ss * (double)p.rgn.inv_count - m * m;
                    var = var < 0.0 ? 0.0 : var;
                    s_rg[i] = (float)m;
                    s_rg[NT + i] = (float)(1.0 / sqrt(var + 1e-5)) * p.rgn.gamma[c];
                    s_rg[2 * NT + i] = p.rgn.beta[c];
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
            // one thread = one pixel x a contiguous half of the NT columns (NT = 32: the first 128 threads, all columns)
            const int px = tid & 127, chalf = tid >> 7;
            const int cb_lo = NT >= 64 ? chalf * (NT / 2) : 0, cb_hi = NT >= 64 ? cb_lo + NT / 2 : (chalf == 0 ? NT : 0);
            const int Ho = (GEOM == G_DOWN || GEOM == G_UP) ? p.Ho : p.H, Wo = (GEOM == G_DOWN || GEOM == G_UP) ? p.Wo : p.W;
            const int CHo = p.Cout / 4;                            // 16-byte channel chunks of the output tensor
            int ho, wo; bool valid;
            if (GEOM == G_C3 || GEOM == G_C7 || GEOM == G_DOWN) {
                ho = h0; wo = w0 + px;
                valid = ho < Ho && wo < Wo;
            } else if (C1) {
                ho = 0; wo = w0 + px;
                valid = wo < Wo;
            } else if (GEOM == G_UP) {
                valid = h0 < p.H && (w0 + px) < p.W;                 // per-phase coordinates are formed below
                ho = 2 * h0; wo = 2 * (w0 + px);
            } else {
                const long long m = (long long)h0 * TPX + px;
                valid = m < HW;
                ho = valid ? (int)(m / p.W) : 0;
                wo = valid ? (int)(m - (long long)ho * p.W) : 0;
            }
            if (!valid) { ho = 0; wo = 0; }
            const int cpg = p.Cout / kGroups;
            const float* bp = p.bias ? p.bias + (long long)b * p.bias_bstride + n0 : nullptr;
#pragma unroll
            for (int phase = 0; phase < NACC; ++phase) {
            if constexpr (ROW2) {
                // pass `phase` stages pixel block `phase` of both rows: staging pixel px is row px / 64, column 64 phase + px % 64
                ho = h0 + (px >> 6); wo = w0 + 64 * phase + (px & 63);
                valid = ho < Ho && wo < Wo;
                if (!valid) { ho = 0; wo = 0; }
            }
            // GroupNorm slot row of this warp's 32 pixels (2-row tile: the row's slot set, the warp of the 1-row tile)
            const int slot = ROW2 ? ((warp & 3) >> 1) * 64 + ((warp >> 2) * 4 + 2 * phase + (warp & 1)) * 8 : warp * 8;
            // accumulators -> staging tile [pixel][column]
            asm volatile("bar.sync 2, 256;" ::: "memory");            // previous readers of the staging tile are done
            {
                auto stage_out = [&](const float (&res)[FR]) {
#pragma unroll
                    for (int i = 0; i < FR; i += 2)
                        *reinterpret_cast<float2*>(&sD[(64 * wg + frag_row(wt, i)) * LDS + frag_col(wt, i)]) = make_float2(res[i], res[i + 1]);
                };
                if constexpr (CHUNKED) stage_out(sum[phase]);
                else stage_out(acc[phase]);
            }
            asm volatile("bar.sync 2, 256;" ::: "memory");
            const int ho_p = GEOM == G_UP ? ho + (phase >> 1) : ho;
            const int wo_p = GEOM == G_UP ? wo + (phase & 1) : wo;
            const float mo = (p.out_mask || RES) ? __ldg(p.mask + (long long)b * p.T + ((long long)wo_p << p.lvl)) : 1.f;
            // element (b, ho, chunk, wo) of a [B][H][C/4][W][4] tensor; consecutive threads = consecutive pixels = 16 B apart
            const long long obase = (((long long)(b * Ho + ho_p) * CHo + n0 / 4) * Wo + wo_p) * 4;
            const long long cstride = (long long)Wo * 4;           // floats between consecutive channel chunks
            // bf16 outputs: index of the 16-byte chunk (b, ho, n0/8, wo) in a [B][H][C/8][W] grid of chunks; the chunks of one
            // pixel are Wo apart, consecutive threads (pixels) are adjacent: a warp store is again 512 contiguous bytes
            const long long ochunk = (OUT16 || VF16) ? (((long long)(b * Ho + ho_p) * (p.Cout / 8) + n0 / 8) * Wo + wo_p) : 0;
            // ResnetBlock tail: the h2raw side input does not depend on the accumulators, so the first 32-column block is
            // requested before the staging-tile reads and block cb+32 as soon as block cb has been consumed
            constexpr bool SIDE = GEOM == G_PW;                     // the 1x1 convs never carry GN statistics
            const float* pre_src = RES ? p.rraw : nullptr;
            const bool pre_on = RES && valid && mo != 0.f;
            float4 pre[RES ? 8 : 1];
            if constexpr (RES) {
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    pre[i] = pre_on && cb_lo < cb_hi ? __ldg(reinterpret_cast<const float4*>(pre_src + obase + (cb_lo / 4 + i) * cstride))
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll 1
            for (int cb = cb_lo; cb < cb_hi; cb += 32) {
                float v[32];
#pragma unroll
                for (int i = 0; i < 32; i += 4) {
                    const float4 r = *reinterpret_cast<const float4*>(&sD[px * LDS + cb + i]);
                    const float4 bb = bp ? __ldg(reinterpret_cast<const float4*>(bp + cb + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    v[i] = r.x + bb.x; v[i + 1] = r.y + bb.y; v[i + 2] = r.z + bb.z; v[i + 3] = r.w + bb.w;
                }
                if constexpr (RES) {
                    // ResnetBlock tail: + Mish(GN(h2raw)) * mask  (diffusion.py:77-78)
                    if (pre_on) {
#pragma unroll
                        for (int i = 0; i < 32; i += 4) {
                            const float rr[4] = {pre[i / 4].x, pre[i / 4].y, pre[i / 4].z, pre[i / 4].w};
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const int cl = cb + i + e;
                                const float xn = (rr[e] - s_rg[cl]) * s_rg[NT + cl] + s_rg[2 * NT + cl];
                                v[i + e] += X3 ? mish_exact(xn) : mish_fast(xn);
                            }
                        }
                        if (cb + 32 < cb_hi) {
#pragma unroll
                            for (int i = 0; i < 8; ++i)
                                pre[i] = __ldg(reinterpret_cast<const float4*>(pre_src + obase + ((cb + 32) / 4 + i) * cstride));
                        }
                    }
                } else if (p.addin && valid) {
                    // fp32-exact residual (attention: x + g*P x): the tensor core only carries the small g*P x term
                    if constexpr (OUT16) {
                        const uint4* ap = reinterpret_cast<const uint4*>(p.addin) + ochunk + (long long)(cb / 8) * Wo;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const uint4 a = __ldg(ap + (long long)j * Wo);
                            v[8 * j + 0] += bf16_lo(a.x); v[8 * j + 1] += bf16_hi(a.x); v[8 * j + 2] += bf16_lo(a.y); v[8 * j + 3] += bf16_hi(a.y);
                            v[8 * j + 4] += bf16_lo(a.z); v[8 * j + 5] += bf16_hi(a.z); v[8 * j + 6] += bf16_lo(a.w); v[8 * j + 7] += bf16_hi(a.w);
                        }
                    } else {
                        const float* ap = p.addin + obase + (cb / 4) * cstride;
#pragma unroll
                        for (int i = 0; i < 32; i += 4) {
                            const float4 av = __ldg(reinterpret_cast<const float4*>(ap + (i / 4) * cstride));
                            v[i] += av.x; v[i + 1] += av.y; v[i + 2] += av.z; v[i + 3] += av.w;
                        }
                    }
                }
                if (p.out_mask) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] *= mo;
                }
                if (C1 && p.act_out) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] = v[i] > 0.f ? v[i] : v[i] * p.slope;
                }
                if (valid) {
                    if constexpr (OUT16) {
                        uint4* op = reinterpret_cast<uint4*>(p.out) + ochunk + (long long)(cb / 8) * Wo;
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            op[(long long)j * Wo] = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                                                               pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
                    } else if constexpr (VF16) {
                        // bf16 [C/8] chunks of the activated operand (out, or lrelu(out) through act); fp32 x / Z otherwise
                        auto st16 = [&](void* base, float sl) {
                            uint4* op = reinterpret_cast<uint4*>(base) + ochunk + (long long)(cb / 8) * Wo;
                            float a[32];
#pragma unroll
                            for (int i = 0; i < 32; ++i) a[i] = v[i] > 0.f ? v[i] : v[i] * sl;
#pragma unroll
                            for (int j = 0; j < 4; ++j)
                                op[(long long)j * Wo] = make_uint4(pack_bf16x2(a[8 * j], a[8 * j + 1]), pack_bf16x2(a[8 * j + 2], a[8 * j + 3]),
                                                                   pack_bf16x2(a[8 * j + 4], a[8 * j + 5]), pack_bf16x2(a[8 * j + 6], a[8 * j + 7]));
                        };
                        if (p.act_out) {
                            st16(p.out, 1.f);                       // v is already lrelu(acc + bias)
                        } else {
                            float* op = p.out + obase + (cb / 4) * cstride;
#pragma unroll
                            for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(op + (i / 4) * cstride) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
                            if (C1 && p.act) st16(p.act, p.slope);
                        }
                    } else {
                        // (__stwb: one 16-byte store per chunk; the compiler splits a plain float4 store here into four)
                        float* op = p.out + obase + (cb / 4) * cstride;
#pragma unroll
                        for (int i = 0; i < 32; i += 4) __stwb(reinterpret_cast<float4*>(op + (i / 4) * cstride), make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]));
                        if (C1 && p.act) {
                            float* ap = reinterpret_cast<float*>(p.act) + obase + (cb / 4) * cstride;
                            const float sl = p.slope;
#pragma unroll
                            for (int i = 0; i < 32; i += 4)
                                *reinterpret_cast<float4*>(ap + (i / 4) * cstride) =
                                    make_float4(v[i] > 0.f ? v[i] : v[i] * sl, v[i + 1] > 0.f ? v[i + 1] : v[i + 1] * sl,
                                                v[i + 2] > 0.f ? v[i + 2] : v[i + 2] * sl, v[i + 3] > 0.f ? v[i + 3] : v[i + 3] * sl);
                        }
                    }
                }
                if (!SIDE && p.ostats) {
                    // GroupNorm partials of this 32-column chunk: 8-channel sub-sums first (static register indexing),
                    // then merged to the group width cpg (8 -> 4 groups, 16 -> 2 groups, >= 32 -> 1 group)
                    float s8[4], q8[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float s = 0.f, q = 0.f;
#pragma unroll
                        for (int i = 0; i < 8; ++i) { const float x = valid ? v[8 * k + i] : 0.f; s += x; q = fmaf(x, x, q); }
                        s8[k] = s; q8[k] = q;
                    }
                    const int ngrp = cpg == 8 ? 4 : (cpg == 16 ? 2 : 1);
                    if (ngrp == 2) { s8[0] += s8[1]; q8[0] += q8[1]; s8[1] = s8[2] + s8[3]; q8[1] = q8[2] + q8[3]; }
                    if (ngrp == 1) { s8[0] += s8[1] + s8[2] + s8[3]; q8[0] += q8[1] + q8[2] + q8[3]; }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (k < ngrp) {
                            float s = s8[k], q = q8[k];
#pragma unroll
                            for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
                            if (lane == 0) {
                                const int gl = (n0 + cb + k * (32 / ngrp)) / cpg - n0 / cpg;
                                s_st[(slot + gl) * 2] += s;
                                s_st[(slot + gl) * 2 + 1] += q;
                            }
                        }
                    }
                }
            }
            }
            if (GEOM != G_PW && p.ostats) {
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const int gb = n0 / cpg, ng = (NT + cpg - 1) / cpg;
                const int r = tid / (ng * 2), e = tid - r * (ng * 2);       // output row of the tile, (group, sum | squares)
                if (tid < ng * 2 * ROWS) {
                    double tot = 0.0;
                    float* sl = s_st + r * 128 + e;
#pragma unroll
                    for (int w8 = 0; w8 < NCONS / 32; ++w8) { tot += (double)sl[w8 * 16]; sl[w8 * 16] = 0.f; }
                    if (!ROW2 || h0 + r < Ho)                          // (the missing second row of an odd H adds nothing)
                        atomicAdd(&p.ostats[((long long)b * kGroups + gb + (e >> 1)) * 2 + (e & 1)], tot);
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
        }
    } else {
        setmaxnreg_dec<PROD_REGS>();
        if (warp != NCONS / 32) {
            if constexpr (X3 && BULK) {
                // =================================================================================================
                // converter warps (fp32x3): correction stage g = corr_chunk of main stage g + 1
                // =================================================================================================
                // Stage g + 1's full_b says its A tile has landed AND that the loader, which fills the ring in order, has
                // seen stage g's previous occupant released, so stage g's A area is free to write.  Stage g + 1 cannot be
                // overwritten while it is read here: the consumers release it after its MMAs, which they issue after stage
                // g's, which wait for this warp's arrival on full_a(g).
                const int ct = tid - (NCONS + 32);
                uint32_t it = 0;
                for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                    for (int ks = 0; ks < ksteps_t; ks += 2, it += 2) {
                        const uint32_t sc = it % STAGES, sm = (it + 1) % STAGES;
                        mbar_wait(full_b(sm), ((it + 1) / STAGES) & 1);
                        const float4* src = reinterpret_cast<const float4*>(sA + sm * A_STAGE_BYTES);
                        float4* dst = reinterpret_cast<float4*>(sA + sc * A_STAGE_BYTES);
                        // (four loads in flight per thread: the conversion's latency is lead the loader loses)
                        constexpr int NCHK = A_STAGE_BYTES / 16, UN = 4;
                        for (int i0 = ct; i0 < NCHK; i0 += UN * NCONV) {
                            float4 v[UN];
#pragma unroll
                            for (int u = 0; u < UN; ++u)
                                if (i0 + u * NCONV < NCHK) v[u] = src[i0 + u * NCONV];
#pragma unroll
                            for (int u = 0; u < UN; ++u)
                                if (i0 + u * NCONV < NCHK) dst[i0 + u * NCONV] = corr_chunk(v[u].x, v[u].y, v[u].z, v[u].w);
                        }
                        fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor core
                        __syncwarp();
                        if (lane == 0) mbar_arrive(full_a(sc));
                    }
                }
            }
            return;
        }
        // =========================================================================================================
        // loader warp: weights + A runs by cp.async.bulk.  Every byte of the A tile is written every stage:
        // out-of-image rows / columns (the conv's zero padding, the ragged last 1x1 tile) come from a zero page.
        // =========================================================================================================
        // Lane 0 owns the ring protocol, the border bookkeeping and the weight copy; the (chunk, row) activation runs of a
        // stage are issued by KCH*HR lanes in parallel.
        uint32_t it = 0;
        const float* zero = p.zero_page;
        uint32_t stage_pat[STAGES];
#pragma unroll
        for (int i = 0; i < STAGES; ++i) stage_pat[i] = 0xFFFFFFFFu;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            int b, h0, w0, n0;
            decode(t, b, h0, w0, n0);
            // weight image: [ntile][kstage][tap][chunk][NT][16 B]; fp32x3: [ntile][kstage][hi|correction][tap][chunk][NT][16 B]
            const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.wpk) + (size_t)b * p.w_bstride_bytes +
                                  (size_t)(n0 / NT) * ksteps * (X3 ? 2 : 1) * B_STAGE_BYTES;
            // 3x3 / 7x7 halo: input row of halo row r of a stage is h0 - PADK + krow + r
            constexpr int PADK = GEOM == G_C7 ? 3 : 1;
            for (int ks = 0; ks < ksteps_t; ++ks, ++it) {
                const int s = it % STAGES;
                const int st = X3 ? ks / 2 : ks, var = X3 ? (ks & 1) : 1;          // 0: correction (fp16 chunks), 1: main (x, w_hi)
                const int kb = st / conv_tc_stage_rows(GEOM), krow = st - kb * conv_tc_stage_rows(GEOM);     // K step, kernel row (7x7) of weight stage st
                const bool conv = X3 && BULK && var == 0;     // A tile written by the converter warps: weights only
                if (lane == 0) {
                    mbar_wait(empty(s), ((it / STAGES) & 1) ^ 1);
                    uint32_t a_tx = BULK && !conv ? A_STAGE_BYTES : 0;
                    if (BULK && GEOM != G_PW) {
                        // Image-border columns (the conv's zero padding) are never written by the row copies, so they only
                        // need zeroing when this stage buffer last served a tile with a different border pattern.  With
                        // the round-robin tile order a CTA normally keeps one pattern, so this (and its proxy fence,
                        // which would otherwise serialise against the bulk copies in flight) runs a handful of times.
                        const int pad = C1 ? p.pad : PADK;          // Conv1d: (K-1)*dil/2 samples of halo on each side
                        const int wlo = w0 - pad < 0 ? 0 : w0 - pad, whi = w0 + SPAN + pad > p.W ? p.W : w0 + SPAN + pad;
                        const int qlo = wlo - (w0 - pad), qhi = qlo + (whi - wlo);
                        const uint32_t pat = (uint32_t)qlo | ((uint32_t)qhi << 16);
                        if (conv) {
                            stage_pat[s] = pat;              // the converters write the whole tile, its zero borders included
                        } else if (stage_pat[s] != pat) {
                            stage_pat[s] = pat;
                            if (qlo > 0 || qhi < PXP) {
                                uint8_t* st = sA + s * A_STAGE_BYTES;
                                for (int k = 0; k < KCH; ++k)
                                    for (int r = 0; r < HR; ++r) {
                                        uint4* rowp = reinterpret_cast<uint4*>(st + k * PLANE + (r * PXP) * 16);
                                        for (int q = 0; q < qlo; ++q) rowp[q] = make_uint4(0u, 0u, 0u, 0u);
                                        for (int q = qhi; q < PXP; ++q) rowp[q] = make_uint4(0u, 0u, 0u, 0u);
                                    }
                                fence_proxy_async();
                            }
                        }
                        int vrows = 0;
                        for (int r = 0; r < HR; ++r) { const int hi = C1 ? 0 : h0 - PADK + krow + r; vrows += (hi >= 0 && hi < p.H) ? 1 : 0; }
                        if (!conv) a_tx -= (uint32_t)(KCH * vrows * (PXP - (qhi - qlo))) * 16u;
                    }
                    mbar_arrive_expect_tx(full_b(s), B_STAGE_BYTES + a_tx);
                    bulk_g2s(smem_u32(sB + s * B_STAGE_BYTES), wsrc + (size_t)(X3 ? 2 * st + (var == 0) : ks) * B_STAGE_BYTES,
                             B_STAGE_BYTES, full_b(s));
                }
                __syncwarp();
                if (BULK && !conv && lane < KCH * HR) {
                    const uint32_t a_s = smem_u32(sA) + s * A_STAGE_BYTES;
                    const int k = lane / HR, r = lane - k * HR;
                    const int ck = kb * KCH + k;                     // 16-byte channel chunk index over the concat
                    const bool second = ck * EPC >= p.c0;
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(second ? p.in1 : p.in0);
                    const int chs = (second ? p.c1 : p.c0) / EPC;
                    const int cl = second ? ck - p.c0 / EPC : ck;
                    if (GEOM == G_PW) {
                        long long m = (long long)(h0 + r) * TPX;
                        const long long m_hi = m >= HW ? m : (m + TPX < HW ? m + TPX : HW);
                        int q = 0;
                        if (m < m_hi) {
                            int hh = (int)(m / p.W), ww = (int)(m - (long long)hh * p.W);
                            while (m < m_hi) {                     // split the flattened run at image-row boundaries
                                const int n = (int)((p.W - ww) < (m_hi - m) ? (p.W - ww) : (m_hi - m));
                                bulk_g2s(a_s + k * PLANE + (r * PXP + q) * 16,
                                         src + (((long long)(b * p.H + hh) * chs + cl) * p.W + ww) * 16, (uint32_t)n * 16u, full_b(s));
                                m += n; q += n; ++hh; ww = 0;
                            }
                        }
                        if (q < PXP) bulk_g2s(a_s + k * PLANE + (r * PXP + q) * 16, zero, (uint32_t)(PXP - q) * 16u, full_b(s));
                    } else {
                        const int pad = C1 ? p.pad : PADK;
                        const int wlo = w0 - pad < 0 ? 0 : w0 - pad, whi = w0 + SPAN + pad > p.W ? p.W : w0 + SPAN + pad;
                        const int qlo = wlo - (w0 - pad);
                        const int hi = C1 ? 0 : h0 - PADK + krow + r;
                        const uint32_t row_s = a_s + k * PLANE + (r * PXP) * 16;
                        if (hi < 0 || hi >= p.H) bulk_g2s(row_s, zero, PXP * 16u, full_b(s));
                        else bulk_g2s(row_s + qlo * 16, src + (((long long)(b * p.H + hi) * chs + cl) * p.W + wlo) * 16,
                                      (uint32_t)(whi - wlo) * 16u, full_b(s));
                    }
                }
            }
        }
    }
}

template <int GEOM, bool BF16, int NT, bool RES = false, int R = 1>
__global__ void __launch_bounds__(NTHREADS, 1) k_conv_tc(const ConvTcParams p) {
    conv_tc_body<GEOM, BF16, NT, RES, false, false, R>(p);
}
template <int GEOM, int NT, bool RES = false, int R = 1>
__global__ void __launch_bounds__(NTHREADS, 1) k_conv_tc_x3(const ConvTcParams p) {
    conv_tc_body<GEOM, false, NT, RES, true, false, R>(p);
}
// the vocoder's transposed-conv GEMM in bf16 mode: bf16 operands, fp32 output Z (ConvTcParams::voc)
template <int NT>
__global__ void __launch_bounds__(NTHREADS, 1) k_gemm_voc_bf16(const ConvTcParams p) {
    conv_tc_body<G_PW, true, NT, false, false, true>(p);
}

// the kernel of one launch configuration; VOC: the vocoder's bf16 GEMM
template <int GEOM, int FORM, int NT, bool RES, int R, bool VOC>
constexpr auto tc_kernel() {
    if constexpr (VOC) return k_gemm_voc_bf16<NT>;
    else if constexpr (FORM == FORM_X3) return k_conv_tc_x3<GEOM, NT, RES, R>;
    else return k_conv_tc<GEOM, FORM == FORM_BF16, NT, RES, R>;
}

template <int GEOM, int FORM, int NT, bool RES = false, int R = 1, bool VOC = false>
static int launch_tc(const ConvTcParams& p, cudaStream_t s) {
    using D = Depth<GEOM, NT, R>;
    static_assert(!VOC || (GEOM == G_PW && FORM == FORM_BF16 && !RES), "VOC selects the bf16 GEMM with fp32 output");
    constexpr auto kernel = tc_kernel<GEOM, FORM, NT, RES, R, VOC>();
    // the dynamic-shared-memory opt-in is a per-device function attribute and the persistent grid is sized from the
    // current device's SM count: both are cached per device ordinal (a process may drive several GPUs through several handles)
    static DevCache cache;
    const int num_sms = cache.get(reinterpret_cast<const void*>(kernel));
    if (num_sms <= 0) return -1;
    int mt;
    if (geom_is_c1(GEOM)) mt = (p.W + TPX - 1) / TPX;
    else if (GEOM == G_C3 || GEOM == G_C7 || GEOM == G_UP) mt = ((p.W + TPX - 1) / TPX) * ((p.H + R - 1) / R);
    else if (GEOM == G_DOWN) mt = ((p.Wo + TPX - 1) / TPX) * p.Ho;
    else mt = (p.H * p.W + TPX - 1) / TPX;
    const long long total = (long long)mt * (p.Cout / NT) * p.B;
    const int grid = (int)(total < num_sms ? total : num_sms);       // persistent: one wave of resident CTAs
    kernel<<<grid, NTHREADS, D::SMEM, s>>>(p);
    return 1;
}

// N tile per geometry and form: Upsample keeps 4 phase accumulators per thread, so its tiles are 64 channels wide.  In
// fp32x3 the running sums live in registers next to the accumulators: the 128-wide variants of the 7x7 conv and of the
// Conv1d would spill them.
int conv_tc_ntile(int geom, int Cout, int form) {
    if (geom == G_UP || geom == G_DOWN) return 64;
    if (geom_is_c1(geom)) return Cout % 128 == 0 && form != FORM_X3 ? 128 : (Cout % 64 == 0 ? 64 : 32);
    if (geom == G_C7 && form == FORM_X3) return 64;
    return Cout % 128 == 0 ? 128 : 64;
}

// one launch configuration: geometry, operand form, N tile, output rows per tile, ResnetBlock tail, vocoder GEMM
static constexpr int tc_key(int geom, int form, int nt, int rows = 1, bool res = false, bool voc = false) {
    return ((((geom * 4 + form) * 256 + nt) * 2 + rows - 1) * 2 + (res ? 1 : 0)) * 2 + (voc ? 1 : 0);
}

// Conv1d (vocoder): tf32 and bf16 at N tiles 128 / 64 / 32, fp32x3 at 64 / 32 (conv_tc_ntile)
template <int GEOM> static int launch_c1(const ConvTcParams& p, cudaStream_t s) {
    constexpr int T = FORM_TF32, X = FORM_X3, B = FORM_BF16;
    switch (tc_key(GEOM, p.form, p.nt)) {
        case tc_key(GEOM, T, 128): return launch_tc<GEOM, T, 128>(p, s);
        case tc_key(GEOM, T, 64):  return launch_tc<GEOM, T, 64>(p, s);
        case tc_key(GEOM, T, 32):  return launch_tc<GEOM, T, 32>(p, s);
        case tc_key(GEOM, B, 128): return launch_tc<GEOM, B, 128>(p, s);
        case tc_key(GEOM, B, 64):  return launch_tc<GEOM, B, 64>(p, s);
        case tc_key(GEOM, B, 32):  return launch_tc<GEOM, B, 32>(p, s);
        case tc_key(GEOM, X, 64):  return launch_tc<GEOM, X, 64>(p, s);
        case tc_key(GEOM, X, 32):  return launch_tc<GEOM, X, 32>(p, s);
        default:                   return -1;
    }
}

int launch_conv_tc(const ConvTcParams& p, cudaStream_t s) {
    if (p.form < FORM_TF32 || p.form > FORM_BF16 || p.nt <= 0 || p.nt > 128 || p.Cout % p.nt != 0) return -1;
    if (p.geom == G_PW && p.epi == EPI_KV) return launch_attn_kv(p, s);   // fused projection + softmax + context (sbk_attn_x3.cu)
    if (geom_is_c1(p.geom) && (p.dil < 1 || p.pad < 0 || 2 * p.pad > conv_tc_c1_halo(p.geom))) return -1;   // the strip's halo
    switch (p.geom) {                                // Conv1d (vocoder): K = 3, 5, 7, 11, each with the 64- and the 128-sample-halo strip
        case G_C1K3:   return launch_c1<G_C1K3>(p, s);
        case G_C1K5:   return launch_c1<G_C1K5>(p, s);
        case G_C1K7:   return launch_c1<G_C1K7>(p, s);
        case G_C1K11:  return launch_c1<G_C1K11>(p, s);
        case G_C1K3W:  return launch_c1<G_C1K3W>(p, s);
        case G_C1K5W:  return launch_c1<G_C1K5W>(p, s);
        case G_C1K7W:  return launch_c1<G_C1K7W>(p, s);
        case G_C1K11W: return launch_c1<G_C1K11W>(p, s);
        default:       break;
    }
    const int rows = p.geom == G_C3 && p.rows == 2 ? 2 : 1;
    const bool res = p.geom == G_PW && p.epi == EPI_RES;
    const bool voc = p.voc && p.geom == G_PW && p.form == FORM_BF16;     // the vocoder's GEMM: fp32 Z from bf16 operands
    constexpr int T = FORM_TF32, X = FORM_X3, B = FORM_BF16;
    switch (tc_key(p.geom, p.form, p.nt, rows, res, voc)) {
        // 3x3: one-row tiles, and two-row tiles 64 channels wide
        case tc_key(G_C3, T, 128):                  return launch_tc<G_C3, T, 128>(p, s);
        case tc_key(G_C3, T, 64):                   return launch_tc<G_C3, T, 64>(p, s);
        case tc_key(G_C3, T, 64, 2):                return launch_tc<G_C3, T, 64, false, 2>(p, s);
        case tc_key(G_C3, B, 128):                  return launch_tc<G_C3, B, 128>(p, s);
        case tc_key(G_C3, B, 64):                   return launch_tc<G_C3, B, 64>(p, s);
        case tc_key(G_C3, B, 64, 2):                return launch_tc<G_C3, B, 64, false, 2>(p, s);
        case tc_key(G_C3, X, 128):                  return launch_tc<G_C3, X, 128>(p, s);
        case tc_key(G_C3, X, 64):                   return launch_tc<G_C3, X, 64>(p, s);
        case tc_key(G_C3, X, 64, 2):                return launch_tc<G_C3, X, 64, false, 2>(p, s);
        // 1x1: plain, the ResnetBlock tail, and the vocoder's bf16 GEMM
        case tc_key(G_PW, T, 128):                  return launch_tc<G_PW, T, 128>(p, s);
        case tc_key(G_PW, T, 64):                   return launch_tc<G_PW, T, 64>(p, s);
        case tc_key(G_PW, T, 128, 1, true):         return launch_tc<G_PW, T, 128, true>(p, s);
        case tc_key(G_PW, T, 64, 1, true):          return launch_tc<G_PW, T, 64, true>(p, s);
        case tc_key(G_PW, B, 128):                  return launch_tc<G_PW, B, 128>(p, s);
        case tc_key(G_PW, B, 64):                   return launch_tc<G_PW, B, 64>(p, s);
        case tc_key(G_PW, B, 128, 1, true):         return launch_tc<G_PW, B, 128, true>(p, s);
        case tc_key(G_PW, B, 64, 1, true):          return launch_tc<G_PW, B, 64, true>(p, s);
        case tc_key(G_PW, B, 128, 1, false, true):  return launch_tc<G_PW, B, 128, false, 1, true>(p, s);
        case tc_key(G_PW, B, 64, 1, false, true):   return launch_tc<G_PW, B, 64, false, 1, true>(p, s);
        case tc_key(G_PW, X, 128):                  return launch_tc<G_PW, X, 128>(p, s);
        case tc_key(G_PW, X, 64):                   return launch_tc<G_PW, X, 64>(p, s);
        case tc_key(G_PW, X, 128, 1, true):         return launch_tc<G_PW, X, 128, true>(p, s);
        case tc_key(G_PW, X, 64, 1, true):          return launch_tc<G_PW, X, 64, true>(p, s);
        // Downsample, Upsample
        case tc_key(G_DOWN, T, 64):                 return launch_tc<G_DOWN, T, 64>(p, s);
        case tc_key(G_DOWN, B, 64):                 return launch_tc<G_DOWN, B, 64>(p, s);
        case tc_key(G_DOWN, X, 64):                 return launch_tc<G_DOWN, X, 64>(p, s);
        case tc_key(G_UP, T, 64):                   return launch_tc<G_UP, T, 64>(p, s);
        case tc_key(G_UP, B, 64):                   return launch_tc<G_UP, B, 64>(p, s);
        case tc_key(G_UP, X, 64):                   return launch_tc<G_UP, X, 64>(p, s);
        // 7x7 (PostNet): tf32 and fp32x3
        case tc_key(G_C7, T, 128):                  return launch_tc<G_C7, T, 128>(p, s);
        case tc_key(G_C7, T, 64):                   return launch_tc<G_C7, T, 64>(p, s);
        case tc_key(G_C7, X, 64):                   return launch_tc<G_C7, X, 64>(p, s);
        default:                                    return -1;
    }
}

// ---- host: weight images (sbk_internal.h: ConvTcWImg) ----
static uint32_t f32_to_tf32_rna(float x) {
    uint32_t u; memcpy(&u, &x, 4);
    if ((u & 0x7F800000u) != 0x7F800000u) u += 0x1000u;     // round to nearest, ties away (cvt.rna.tf32.f32)
    return u & 0xFFFFE000u;
}
static uint16_t f32_to_f16_rn(float x) {              // saturating, like the device side's cvt.rn.satfinite.f16x2.f32
    if (x > 65504.f) x = 65504.f;
    if (x < -65504.f) x = -65504.f;
    const __half h = __float2half_rn(x);
    uint16_t u; memcpy(&u, &h, 2);
    return u;
}
static uint16_t f32_to_bf16_rn(float x) {
    uint32_t u; memcpy(&u, &x, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((u >> 16) | 0x40);
    u += 0x7FFFu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
// weight w -> its element of image g: tf32 (RNA), bf16 (RNE), or FORM_X3's w_hi = tf32(w) in the main stage and
// {w, (w - w_hi) * 2^12} in the correction stage
static void wimg_put(uint8_t* img, const ConvTcWImg& g, int co, int ks, int tap, int ch, int e, float w) {
    const size_t i = conv_tc_wimg_index(g, co, ks, tap, ch, e);
    if (g.form == FORM_BF16) {
        reinterpret_cast<uint16_t*>(img)[i] = f32_to_bf16_rn(w);
        return;
    }
    const uint32_t uh = f32_to_tf32_rna(w);
    reinterpret_cast<uint32_t*>(img)[i] = uh;
    if (g.form == FORM_X3) {
        float fh; memcpy(&fh, &uh, 4);
        uint16_t* cc = reinterpret_cast<uint16_t*>(img) + 2 * conv_tc_wimg_index(g, co, ks, tap, ch, 0, 1);
        cc[e] = f32_to_f16_rn(w);
        cc[4 + e] = f32_to_f16_rn((w - fh) * 4096.f);
    }
}

// The 7x7 geometry streams one kernel row per stage: weight stage ks = (K step ks / 7, kernel row ks % 7) holds the 7 taps
// of that row.  Every other geometry has one stage per K step, holding all taps.
size_t conv_tc_pack_image(const float* w, int cout, int cin, int geom, int form, int nt, uint8_t* dst) {
    const ConvTcWImg g = conv_tc_wimg(geom, form, nt, cin);
    const int taps = conv_tc_taps(geom), rows = conv_tc_stage_rows(geom), epc = form_epc(form), cps = g.kch * epc;
    if (dst)
        for (int co = 0; co < cout / nt * nt; ++co) for (int ks = 0; ks < g.ksteps; ++ks) for (int tap = 0; tap < g.taps; ++tap)
            for (int ch = 0; ch < g.kch; ++ch) for (int e = 0; e < epc; ++e) {
                const int ci = ks / rows * cps + ch * epc + e;
                wimg_put(dst, g, co, ks, tap, ch, e, w[((size_t)co * cin + ci) * taps + ks % rows * g.taps + tap]);
            }
    return conv_tc_wimg_bytes(g, cout);
}

// k and v rows of to_qkv ('(qkv heads c)': k = rows 128.., v = rows 256..) as k_attn_kv_wg's per-stage image
// [k|v][chunk][row][16 B]: the 1x1 conv's image of one 128-wide N tile with two taps per stage, k and v
size_t attn_kv_pack_image(const float* q, int C, int form, uint8_t* dst) {
    ConvTcWImg g = conv_tc_wimg(G_PW, form, 128, C);
    g.taps = 2;
    const int epc = form_epc(form), cps = g.kch * epc;
    if (dst)
        for (int row = 0; row < 128; ++row) for (int ks = 0; ks < g.ksteps; ++ks) for (int kv = 0; kv < 2; ++kv)
            for (int ch = 0; ch < g.kch; ++ch) for (int e = 0; e < epc; ++e)
                wimg_put(dst, g, row, ks, kv, ch, e, q[(size_t)(128 + kv * 128 + row) * C + ks * cps + ch * epc + e]);
    return conv_tc_wimg_bytes(g, 128);
}

}  // namespace sbk
