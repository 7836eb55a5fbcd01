// br_phases.cuh -- the bootstrap step as CTA-wide phases over shared-memory-resident polynomials.
//
// Why: the first version kept a whole polynomial in one warp's registers (32 elements per lane) and was
// limited by instruction supply.  Here every phase is executed by all
// threads of the CTA at the same time on 16 elements per thread, with 16 warps per SM, so that four warps
// per scheduler share each fetched line and no thread needs more than 128 registers.
//
// A CTA owns CT ciphertexts (BrCfg below).  Shared memory holds, per ciphertext, the accumulator
// (2 x 1024 Torus32) and 4 work polynomials of 1024 field elements; a work polynomial is 16 rows of 64
// columns (padded to 66) -- row r holds inner-transform output k1 = brev4(r), column = position along
// the outer 64-point transform.  The transform is the factorisation of ntt_lane.cuh,
//     X[k1 + 16 k2] = sum_j2 w64^(j2 k2) psi^(j2 (2 k1 + 1)) sum_j1 x[64 j1 + j2] w32^(j1 (2 k1 + 1)),
// computed in three in-place passes:
//     fwd1: 16-point transform over j1 (stride 64) + the psi twiddle       task = (poly, j2)
//     fwd2: first two layers of the 64-point transform (radix 4 over a = j2 / 16) and the 2^(3 b kappa)
//           twiddle, b = j2 % 16                                            task = (poly, row, g = b / 4)
//     fwd3: 16-point transform over b                                       task = (poly, row, u)
// The inverse runs the mirrored passes inv3, inv2, inv1.  Between fwd3 and inv3 the multiply-accumulate
// with the bootstrap-key row works point-wise on pairs of adjacent columns.
//
// Column c = 16 a + b of a row is stored at 16 a + swz(a, b) (an XOR on the pair index) so that the
// 128-bit accesses of fwd2/fwd3/inv3/inv2 are bank-conflict free; see the derivation in DESIGN.md.
//
// All functions are __host__ __device__: csrc/host_emul.cpp runs them phase by phase on the CPU (a
// barrier between phases), which lets the CPU-only test-suite check every index map against the oracle.
#pragma once
#include <cmath>
#include <cstring>
#include "ntt_lane.cuh"
#include "fft_layout.cuh"

namespace nb {

#ifndef NB_BR_CT
#define NB_BR_CT 2
#endif
#ifndef NB_BR_STAGE_KEY
#define NB_BR_STAGE_KEY 0
#endif
#ifndef NB_FWD1_BOTH_DIGITS
#define NB_FWD1_BOTH_DIGITS 1
#endif
// Deferred canonicalisation: the general multiplications of fwd1 / inv1 and the MAC leave their result as "some
// 64-bit value of the right residue" (ff_mul_nc, ff_dot4_sub_nc) instead of paying 6 ALU instructions per element
// for the conditional subtraction of p.  Such a value is above p with probability 2^-32 (a few elements per
// 4096-ciphertext bootstrap), and then its high limb is 2^32 - 1: every thread keeps the maximum of the high limbs
// it produced (one instruction per element) and canonicalises its elements when that maximum reaches
// nb_c_canon_trigger (= 2^32 - 1; the tests lower it to 0 to drive the rare path on every task).
#ifndef NB_LAZY_CANON
#define NB_LAZY_CANON 1
#endif
#if defined(__CUDACC__)
__constant__ u32 nb_c_canon_trigger = 0xffffffffu;
#endif
NB_HD bool canon_needed(u32 hmax)
{
#if defined(__CUDA_ARCH__)
    return hmax >= nb_c_canon_trigger;
#else
    return hmax == 0xffffffffu;
#endif
}
NB_HD u32 umax32(u32 a, u32 b) { return a > b ? a : b; }

// EXPERIMENT, off by default: butterfly networks with deferred canonicalisation of their SUMS
// (ff_add_nc, ntt_lane.cuh).  The network runs with the cheap additions and collects the high limbs of the sums; if one
// of them is 2^32 - 1 (probability 2^-33 per addition) the thread restores its inputs (`reload`) and runs the exact
// network.  165 fewer instructions per thread-step, bit-exact (GPU suite green with it) -- and SLOWER, in the bootstrap
// and in the stand-alone transforms: ptxas turns the carry of the new
// sequence into SEL + LOP3 on the ALU pipe where ff_sub gets IMAD.X + IMAD.MOV on the FMA pipe (+126 ALU-pipe
// instructions), and every network gains a divergence-barrier pair around its rare branch.
#ifndef NB_LAZY_ADD
#define NB_LAZY_ADD 0
#endif
#if defined(__CUDA_ARCH__)
#define NB_UNLIKELY(x) __builtin_expect(!!(x), 0)
#else
#define NB_UNLIKELY(x) (x)
#endif
struct NetDif16 {
    template <bool NC> NB_HD static void run(u64 *v, u32 &h) { if constexpr (NC) dif_inlane_nc<4, 12, 0>(v, h); else dif_inlane<4, 12, 0>(v); }
};
struct NetDit16 {
    template <bool NC> NB_HD static void run(u64 *v, u32 &h) { if constexpr (NC) dit_inlane_nc<4, 12, 0>(v, h); else dit_inlane<4, 12, 0>(v); }
};
struct NetDif4x4 {       // four 4-point transforms over a (stride 4), root 2^48
    template <bool NC> NB_HD static void run(u64 *v, u32 &h)
    {
        static_for<0, 4>([&](auto E) {
            if constexpr (NC) dif_inlane_nc<2, 48, decltype(E)::value, 4>(v, h); else dif_inlane<2, 48, decltype(E)::value, 4>(v);
        });
    }
};
struct NetDit4x4 {
    template <bool NC> NB_HD static void run(u64 *v, u32 &h)
    {
        static_for<0, 4>([&](auto E) {
            if constexpr (NC) dit_inlane_nc<2, 48, decltype(E)::value, 4>(v, h); else dit_inlane<2, 48, decltype(E)::value, 4>(v);
        });
    }
};
template <class Net, class Reload> NB_HD void run_network(u64 *v, Reload reload)
{
    u32 hmax = 0;
#if NB_LAZY_ADD
    Net::template run<true>(v, hmax);
    if (NB_UNLIKELY(canon_needed(hmax))) {
        reload();
        Net::template run<false>(v, hmax);
    }
#else
    (void)reload;
    Net::template run<false>(v, hmax);
#endif
}

constexpr int ROW_STRIDE = 66;                    // u64 per row (64 + 2 padding)
constexpr int POLY_STRIDE = 16 * ROW_STRIDE;      // u64 per work polynomial

// Shape of one CTA of the fused bootstrap: CT ciphertexts on THREADS threads.  Per ciphertext a step has 256
// forward tasks (4 digit polynomials x 64), 128 inverse tasks (2 polynomials x 64) and 512 MAC points pairs.
//   BrCfg<2, 256> (default): 128 threads per ciphertext, every thread busy in every phase, 2 CTAs per SM --
//                            the throughput shape.
//   BrCfg<1, 256> ("wide"):  256 threads per ciphertext: the forward phases take one sweep instead of two and the
//                            inverse phases leave half of the warps idle; 36 % fewer instructions on the critical
//                            path of a step.  Used when the batch fits one wave of such CTAs (latency, not throughput).
//   BrCfg<2, 256, 2, true, true> ("fft"): the throughput shape with the FP64 step (keys with spectra, see below).
template <int CT_, int THREADS_, int CTAS_ = 512 / THREADS_, bool TWD_GLOBAL_ = false, bool FFT_ = false> struct BrCfg {
    static constexpr int CT = CT_, THREADS = THREADS_;
    static constexpr bool FFT = FFT_;                          // the FP64 step (br_fft_step) instead of the NTT step
    static_assert(!FFT_ || (THREADS_ == 128 * CT_ && TWD_GLOBAL_), "the FP64 step runs 128 threads per ciphertext, tables in L1");
    static constexpr int POLYS = 4 * CT;                       // work polynomials per CTA
    // Twice as many threads as forward tasks ("wide2": 1 ciphertext on 512 threads): two threads of different warps per
    // 16-element forward task, 8 outputs each (split forward phases below)
    static constexpr bool SPLIT_FWD = THREADS == 512 * CT;
    static constexpr int FWD_SWEEPS = SPLIT_FWD ? 1 : 256 * CT / THREADS;      // sweeps of the forward phases
    // two forward tasks per thread: the first pass takes both digit polynomials of one accumulator polynomial at once
    // and shares the rotation between them (phase_fwd1_both_digits)
    static constexpr bool FWD1_BOTH_DIGITS = NB_FWD1_BOTH_DIGITS && !SPLIT_FWD && FWD_SWEEPS == 2;
    static constexpr int INV_TASKS = 128 * CT;                 // threads with work in the inverse phases
    // Twice as many threads as inverse tasks (the wide shape): every inverse task is shared by two threads of
    // different warps, 8 elements each ("split inverse phases" below) instead of leaving half of the warps idle
    static constexpr bool SPLIT_INV = 2 * INV_TASKS <= THREADS;
    static constexpr int CTAS_PER_SM = CTAS_;                  // default 512 / THREADS: 16 warps per SM at 128 registers
    static constexpr bool TWD_GLOBAL = TWD_GLOBAL_;            // twiddle tables read from global memory / L1, not staged
    // EXPERIMENT, off by default (NB_BR_STAGE_KEY): warps without inverse work (the
    // upper half of the 512-thread shape) stage the key row of the NEXT step in shared memory while the others run the
    // inverse phases, and the MAC reads shared memory instead of the L2.  What makes the pair shape fast does nothing
    // here: 16 warps per SM already hide the L2 latency of the MAC.
    static constexpr bool STAGE_KEY = NB_BR_STAGE_KEY && SPLIT_INV && THREADS > 2 * INV_TASKS;
    static_assert(FWD_SWEEPS >= 1 && (SPLIT_FWD || FWD_SWEEPS * THREADS == 256 * CT) && INV_TASKS <= THREADS && THREADS % 128 == 0, "shape");
};
#ifndef NB_BR_THREADS
#define NB_BR_THREADS (128 * NB_BR_CT)
#endif
#ifndef NB_BR_CTAS
#define NB_BR_CTAS (512 / NB_BR_THREADS)
#endif
#ifndef NB_BR_TWD_GLOBAL
#define NB_BR_TWD_GLOBAL 0
#endif
constexpr int BR2_CT = NB_BR_CT;                  // ciphertexts per CTA of the default shape (1, 2 or 4)
constexpr int BR2_THREADS = NB_BR_THREADS;
using BrDefault = BrCfg<BR2_CT, BR2_THREADS, NB_BR_CTAS, NB_BR_TWD_GLOBAL != 0>;
using BrWide = BrCfg<1, 256>;
using BrWide2 = BrCfg<1, 512, 1>;                 // lowest latency: one ciphertext per SM, 16 warps in step
using BrFft = BrCfg<2, 256, 2, true, true>;      // throughput shape, FP64 step
struct BrFftMk : BrFft {};                         // the same with one key per ciphertext (multi-key launches)
constexpr int BR2_POLYS = BrDefault::POLYS;
// Engine bootstrap-key row: 8 planes [(mi*2+j)*2+mo][row*64 + stored column] of plain field values plus
// 2 correction planes K[mo] = 512 * NTT(1,...,1) * sum_{mi,j} plane, because the forward transforms run
// on the UNSIGNED digits u = d + 512 in [0, 1023] (cheap twist, no sign handling):
//     sum_d NTT(d) BK = sum_d NTT(u) BK - 512 NTT(1) sum_d BK.
constexpr int BK_PLANES = 10;
constexpr int BK_NTT_U64 = BK_PLANES * NTT_N;
// the row continues with the 16 key spectra of the FP64 step (BK_FFT_U64 below: 16 x 512 complex doubles)
constexpr int BK_ROW_U64 = BK_NTT_U64 + 16 * 512 * 2;

// 16-byte accesses to two adjacent field elements (shared memory rows and key rows are 16-byte aligned)
NB_HD void ld2(const u64 *p, u64 &x, u64 &y)
{
#if defined(__CUDA_ARCH__)
    ulonglong2 t = *reinterpret_cast<const ulonglong2 *>(p);
    x = t.x; y = t.y;
#else
    x = p[0]; y = p[1];
#endif
}
NB_HD void ld2_global(const u64 *p, u64 &x, u64 &y)
{
#if defined(__CUDA_ARCH__)
    ulonglong2 t = __ldg(reinterpret_cast<const ulonglong2 *>(p));
    x = t.x; y = t.y;
#else
    x = p[0]; y = p[1];
#endif
}
#ifndef NB_ST2_SPLIT
#define NB_ST2_SPLIT 0
#endif
NB_HD void st2(u64 *p, u64 x, u64 y)
{
#if defined(__CUDA_ARCH__)
#if NB_ST2_SPLIT
    // Experiment: two 64-bit stores instead of one 128-bit store, whose four registers must
    // form an aligned quad -- ptxas pays 4 register moves per store to line up the two field elements.  151 fewer
    // IMAD.MOV, 56 more STS per step; it was measured slower, so it stays off.
    // (inline asm: the compiler's load / store vectoriser would fuse two plain stores back into one)
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("st.volatile.shared.u64 [%0], %1;\n\tst.volatile.shared.u64 [%0 + 8], %2;" ::"r"(a), "l"(x), "l"(y) : "memory");
#else
    *reinterpret_cast<ulonglong2 *>(p) = make_ulonglong2(x, y);
#endif
#else
    p[0] = x; p[1] = y;
#endif
}

// stored column of logical column (a, b): pair index XOR 2a
NB_HD int swz(int a, int b) { return ((((b >> 1) ^ (2 * a)) & 7) << 1) | (b & 1); }
NB_HD int col_of(int a, int b) { return 16 * a + swz(a, b); }

// natural NTT index of the transformed element stored at (row, stored column)
NB_HD int w_natural_index(int row, int scol)
{
    int u = scol >> 4, sb = scol & 15;
    int i = ((((sb >> 1) ^ (2 * u)) & 7) << 1) | (sb & 1);
    int k1 = brev(row, 4), k2 = brev(u, 2) + 4 * brev(i, 4);
    return k1 + 16 * k2;
}
// twiddle exponent (power of psi) applied by fwd1 to (row, j2)
NB_HD int w_twiddle_exponent(int row, int j2) { return (j2 * (2 * brev(row, 4) + 1)) % 2048; }

// gadget decomposition digit j of one coefficient (tgsw_gpu.py:31-54; blind_rotate.mako:41-43,116-124),
// returned without the "- 512": u = digit + 512 in [0, 1023]
NB_HD u32 decomp_udigit(i32 c, int j)
{
    const u32 offset = 0x80000000u + (1u << 21);
    u32 t = (u32)c + offset;
    return (t >> (22 - 10 * j)) & 1023u;
}

// (X^a - 1) * acc at index idx  (polynomials_gpu.mako:18-77 with minus_one; blind_rotate.mako:100-114)
NB_HD i32 rotate_minus_one(const i32 *acc, int idx, int ar, bool flip)
{
    i32 src = acc[(idx - ar) & (NTT_N - 1)];
    bool neg = (idx < ar) != flip;
    return (i32)((neg ? 0u - (u32)src : (u32)src) - (u32)acc[idx]);
}

// w[r * ROW_STRIDE] = v[r] * twd[r * 64], r = 0..15: the general multiplication that ends the first forward pass
NB_HD void store_twiddled(const u64 *v, u64 *w, const u64 *twd)
{
#if NB_LAZY_CANON
    u32 hmax = 0;
    static_for<0, 16>([&](auto R) {
        constexpr int r = decltype(R)::value;
        const u64 x = ff_mul_nc(v[r], twd[r * 64]);
        hmax = umax32(hmax, hi32(x));
        w[r * ROW_STRIDE] = x;
    });
    if (canon_needed(hmax)) {                              // rare: this thread's own 16 elements, before the barrier
        static_for<0, 16>([&](auto R) {
            constexpr int r = decltype(R)::value;
            w[r * ROW_STRIDE] = ff_canon_almost(w[r * ROW_STRIDE]);
        });
    }
#else
    static_for<0, 16>([&](auto R) {
        constexpr int r = decltype(R)::value;
        w[r * ROW_STRIDE] = ff_mul(v[r], twd[r * 64]);
    });
#endif
}
// v[r] = w[r * ROW_STRIDE] * twd[r * 64]: the general multiplication that opens the last inverse pass
NB_HD void load_twiddled(u64 *v, const u64 *w, const u64 *twd)
{
#if NB_LAZY_CANON
    u32 hmax = 0;
    static_for<0, 16>([&](auto R) {
        constexpr int r = decltype(R)::value;
        v[r] = ff_mul_nc(w[r * ROW_STRIDE], twd[r * 64]);
        hmax = umax32(hmax, hi32(v[r]));
    });
    if (canon_needed(hmax)) {
        static_for<0, 16>([&](auto R) { v[decltype(R)::value] = ff_canon_almost(v[decltype(R)::value]); });
    }
#else
    static_for<0, 16>([&](auto R) {
        constexpr int r = decltype(R)::value;
        v[r] = ff_mul(w[r * ROW_STRIDE], twd[r * 64]);
    });
#endif
}

// ---- fwd1: task = (poly p, j2); reads ACC, writes W[p][row][col(j2)] -------------------------------
// twd: forward table [row][j2] (64 per row).  ROTATE=false: digits of acc itself (plain external product).
template <bool ROTATE>
NB_HD void phase_fwd1(int task, const i32 *acc_all, u64 *w_all, const u64 *twd, const int *rot_a)
{
    const int j2 = task & 63, p = task >> 6;           // p = ct * 4 + mi * 2 + j
    const int ct = p >> 2, mi = (p >> 1) & 1, j = p & 1;
    const i32 *acc = acc_all + (ct * 2 + mi) * NTT_N;
    const int a = ROTATE ? rot_a[ct] : 0;
    const int ar = a & (NTT_N - 1);
    const bool flip = (a >> 10) & 1;
    u64 v[16];
    auto load = [&]() {
        static_for<0, 16>([&](auto J) {
            constexpr int j1 = decltype(J)::value;
            const int idx = 64 * j1 + j2;
            i32 c = ROTATE ? rotate_minus_one(acc, idx, ar, flip) : acc[idx];
            v[j1] = ff_twist_small<j1>(decomp_udigit(c, j));
        });
    };
    load();
    run_network<NetDif16>(v, load);
    u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    store_twiddled(v, w, twd + j2);
}

// The same pass for BOTH digit polynomials of one accumulator polynomial: task = (pm = ct * 2 + mi, j2).  The rotated
// coefficients (two loads, a select and a subtraction each) and the decomposition offset are computed once and serve both
// digits; the digit loop is a real loop (run-time shift amount), so the code is no longer than one digit's.
// Used when a thread would otherwise run two tasks of this pass (BrCfg: FWD1_BOTH_DIGITS).
template <bool ROTATE>
NB_HD void phase_fwd1_both_digits(int task, const i32 *acc_all, u64 *w_all, const u64 *twd, const int *rot_a)
{
    const int j2 = task & 63, pm = task >> 6;
    const i32 *acc = acc_all + pm * NTT_N;
    const int a = ROTATE ? rot_a[pm >> 1] : 0;
    const int ar = a & (NTT_N - 1);
    const bool flip = (a >> 10) & 1;
    u32 t[16];                                         // coefficient + decomposition offset (decomp_udigit)
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        const int idx = 64 * j1 + j2;
        const i32 c = ROTATE ? rotate_minus_one(acc, idx, ar, flip) : acc[idx];
        t[j1] = (u32)c + (0x80000000u + (1u << 21));
    });
    u64 *w = w_all + pm * 2 * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 0; j < 2; j++) {
        const int sh = 22 - 10 * j;
        u64 v[16];
        auto load = [&]() {
            static_for<0, 16>([&](auto J) {
                constexpr int j1 = decltype(J)::value;
                v[j1] = ff_twist_small<j1>((t[j1] >> sh) & 1023u);
            });
        };
        load();
        run_network<NetDif16>(v, load);
        store_twiddled(v, w + j * POLY_STRIDE, twd + j2);
    }
}

// ---- fwd2 / inv2: task = (poly p, row, g); 16 elements (a, e), b = 4 g + e ---------------------------
template <int G> NB_HD void fwd2_twiddle(u64 *v)
{
    static_for<1, 4>([&](auto U) {
        constexpr int u = decltype(U)::value;
        constexpr int kappa = brev(u, 2);
        static_for<0, 4>([&](auto E) {
            constexpr int e = decltype(E)::value;
            v[u * 4 + e] = ff_shl<(3 * kappa * (4 * G + e)) % 192>(v[u * 4 + e]);
        });
    });
}
template <int G> NB_HD void inv2_twiddle(u64 *v)
{
    static_for<1, 4>([&](auto U) {
        constexpr int u = decltype(U)::value;
        constexpr int kappa = brev(u, 2);
        static_for<0, 4>([&](auto E) {
            constexpr int e = decltype(E)::value;
            v[u * 4 + e] = ff_shl<(192 - (3 * kappa * (4 * G + e)) % 192) % 192>(v[u * 4 + e]);
        });
    });
}

// col_of(a, 4 g + e) = 16 a + 4 (g ^ a) + e: the four e of a thread are contiguous (2 x 16 bytes)
NB_HD void load16_ae(u64 *v, const u64 *row, int g)
{
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        const u64 *src = row + 16 * a + 4 * (g ^ a);
        ld2(src, v[a * 4 + 0], v[a * 4 + 1]);
        ld2(src + 2, v[a * 4 + 2], v[a * 4 + 3]);
    });
}
NB_HD void store16_ae(const u64 *v, u64 *row, int g)
{
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        u64 *dst = row + 16 * a + 4 * (g ^ a);
        st2(dst, v[a * 4 + 0], v[a * 4 + 1]);
        st2(dst + 2, v[a * 4 + 2], v[a * 4 + 3]);
    });
}
// the 16 logical columns of block u, pair pi stored at pair position pi ^ 2u
NB_HD void load16_b(u64 *v, const u64 *row, int u)
{
    static_for<0, 8>([&](auto PI) {
        constexpr int pi = decltype(PI)::value;
        ld2(row + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[2 * pi], v[2 * pi + 1]);
    });
}
NB_HD void store16_b(const u64 *v, u64 *row, int u)
{
    static_for<0, 8>([&](auto PI) {
        constexpr int pi = decltype(PI)::value;
        st2(row + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[2 * pi], v[2 * pi + 1]);
    });
}

NB_HD void phase_fwd2(int p, int row, int g, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[16];
    load16_ae(v, w, g);
    run_network<NetDif4x4>(v, [&]() { load16_ae(v, w, g); });
    switch (g) {           // g is warp-uniform by construction of the task map
    case 0: fwd2_twiddle<0>(v); break;
    case 1: fwd2_twiddle<1>(v); break;
    case 2: fwd2_twiddle<2>(v); break;
    default: fwd2_twiddle<3>(v); break;
    }
    store16_ae(v, w, g);
}

NB_HD void phase_inv2(int p, int row, int g, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[16];
    auto load = [&]() {
        load16_ae(v, w, g);
        switch (g) {
        case 0: inv2_twiddle<0>(v); break;
        case 1: inv2_twiddle<1>(v); break;
        case 2: inv2_twiddle<2>(v); break;
        default: inv2_twiddle<3>(v); break;
        }
    };
    load();
    run_network<NetDit4x4>(v, load);
    store16_ae(v, w, g);
}

// ---- fwd3 / inv3: task = (poly p, row, u): the 16 logical columns b of block u ---------------------
NB_HD void phase_fwd3(int p, int row, int u, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[16];
    load16_b(v, w, u);
    run_network<NetDif16>(v, [&]() { load16_b(v, w, u); });
    store16_b(v, w, u);
}
NB_HD void phase_inv3(int p, int row, int u, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[16];
    load16_b(v, w, u);
    run_network<NetDit16>(v, [&]() { load16_b(v, w, u); });
    store16_b(v, w, u);
}

// ---- split forward phases (Cfg::SPLIT_FWD) --------------------------------------------------------------------------
// The mirror image of the split inverse phases below, without an exchange: a 16-point decimation-in-frequency network
// is one layer that pairs element k with element 8 + k, followed by two 8-point networks (dif_inlane<3, 24>) on the sums
// and on the twiddled differences.  Both threads of a task read all 16 inputs; half 0 forms the 8 sums, half 1 the 8
// differences times 2^(12 k), each runs its 8-point network and stores its 8 outputs.
template <int H> NB_HD void dif16_half(const u64 *v16, u64 *u8)
{
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        if constexpr (H == 0) u8[k] = ff_add(v16[k], v16[k + 8]);
        else u8[k] = ff_shl<(12 * k) % 192>(ff_sub(v16[k], v16[k + 8]));
    });
    dif_inlane<3, 24, 0>(u8);
}
template <bool ROTATE, int H>
NB_HD void phase_fwd1_split(int task, const i32 *acc_all, u64 *w_all, const u64 *twd, const int *rot_a)
{
    const int j2 = task & 63, p = task >> 6;           // p = ct * 4 + mi * 2 + j
    const int ct = p >> 2, mi = (p >> 1) & 1, j = p & 1;
    const i32 *acc = acc_all + (ct * 2 + mi) * NTT_N;
    const int a = ROTATE ? rot_a[ct] : 0;
    const int ar = a & (NTT_N - 1);
    const bool flip = (a >> 10) & 1;
    u64 v[16], u[8];
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        const int idx = 64 * j1 + j2;
        i32 c = ROTATE ? rotate_minus_one(acc, idx, ar, flip) : acc[idx];
        v[j1] = ff_twist_small<j1>(decomp_udigit(c, j));
    });
    dif16_half<H>(v, u);
    u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15) + 8 * H * ROW_STRIDE;
    const u64 *tw = twd + 8 * H * 64 + j2;
    u32 hmax = 0;
    static_for<0, 8>([&](auto R) {
        constexpr int r = decltype(R)::value;
#if NB_LAZY_CANON
        const u64 x = ff_mul_nc(u[r], tw[r * 64]);
        hmax = umax32(hmax, hi32(x));
        w[r * ROW_STRIDE] = x;
#else
        w[r * ROW_STRIDE] = ff_mul(u[r], tw[r * 64]);
#endif
    });
#if NB_LAZY_CANON
    if (canon_needed(hmax)) {
        static_for<0, 8>([&](auto R) { w[decltype(R)::value * ROW_STRIDE] = ff_canon_almost(w[decltype(R)::value * ROW_STRIDE]); });
    }
#endif
}
template <int G, int H> NB_HD void fwd2_twiddle_half(u64 *v8)        // v8[a * 2 + e'], e = 2 H + e'
{
    static_for<1, 4>([&](auto U) {
        constexpr int u = decltype(U)::value;
        constexpr int kappa = brev(u, 2);
        static_for<0, 2>([&](auto E) {
            constexpr int e = 2 * H + decltype(E)::value;
            v8[u * 2 + decltype(E)::value] = ff_shl<(3 * kappa * (4 * G + e)) % 192>(v8[u * 2 + decltype(E)::value]);
        });
    });
}
template <int H> NB_HD void phase_fwd2_split(int p, int row, int g, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[8];
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        ld2(w + 16 * a + 4 * (g ^ a) + 2 * H, v[a * 2], v[a * 2 + 1]);
    });
    static_for<0, 2>([&](auto E) { dif_inlane<2, 48, decltype(E)::value, 2>(v); });
    switch (g) {           // warp-uniform
    case 0: fwd2_twiddle_half<0, H>(v); break;
    case 1: fwd2_twiddle_half<1, H>(v); break;
    case 2: fwd2_twiddle_half<2, H>(v); break;
    default: fwd2_twiddle_half<3, H>(v); break;
    }
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        st2(w + 16 * a + 4 * (g ^ a) + 2 * H, v[a * 2], v[a * 2 + 1]);
    });
}
// fwd3 works in place and both halves need all 16 inputs: every thread loads them (phase_fwd3_split_load), the CTA
// synchronises, and only then each half stores its 8 outputs (phase_fwd3_split_finish)
NB_HD void phase_fwd3_split_load(int p, int row, int u, const u64 *w_all, u64 *v)
{
    load16_b(v, w_all + p * POLY_STRIDE + row * ROW_STRIDE, u);
}
template <int H> NB_HD void phase_fwd3_split_finish(int p, int row, int u, u64 *w_all, const u64 *v)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 o[8];
    dif16_half<H>(v, o);
    static_for<0, 4>([&](auto PI) {
        constexpr int pi = 4 * H + decltype(PI)::value;
        st2(w + 16 * u + 2 * ((pi ^ (2 * u)) & 7), o[2 * decltype(PI)::value], o[2 * decltype(PI)::value + 1]);
    });
}

// ---- split inverse phases (Cfg::SPLIT_INV) --------------------------------------------------------------------------
// A 16-point decimation-in-time network is two 8-point networks on elements 0-7 and 8-15 (the first three layers:
// dit_inlane<3, 24>) followed by one layer that pairs element k with element 8 + k.  Thread half h = 0 / 1 (a whole
// warp either way) runs the 8-point network on its elements, half 1 also applies the last layer's twiddles, and both
// park their 8 values in the work polynomial p + 2 -- dead since the MAC, which overwrote polynomials 0 and 1 of the
// ciphertext with its outputs -- at the positions they were read from.  After a CTA barrier each thread reads the 16
// parked values of its task and finishes ITS 8 outputs.  The per-thread instruction stream of the inverse phases
// halves, which is what the latency of a step is made of when few warps are resident (DESIGN.md section 8).
template <int H> NB_HD void dit16_half_a(u64 *v8)
{
    dit_inlane<3, 24, 0>(v8);
    if constexpr (H == 1) {
        // last-layer twiddles 2^(-12 k) = -2^(96 - 12 k), k >= 1: shift by the positive amount, the sign goes into
        // the add / sub choice of dit16_half_b (as in dit_inlane)
        static_for<1, 8>([&](auto K) { constexpr int k = decltype(K)::value; v8[k] = ff_shl<96 - 12 * k>(v8[k]); });
    }
}
// a[k], t[k]: the parked values of elements k and 8 + k; o[k]: output element 8 H + k
template <int H> NB_HD void dit16_half_b(const u64 *a, const u64 *t, u64 *o)
{
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        constexpr bool sub = (H == 1) != (k >= 1);       // element k: a + t for k = 0, a - t otherwise; element 8 + k: the reverse
        o[k] = sub ? ff_sub(a[k], t[k]) : ff_add(a[k], t[k]);
    });
}

// inv3, first half: task (p, row, u), elements 8 H .. 8 H + 7 of block u (logical pairs 4 H .. 4 H + 3)
// ADD_PARKED (pair shape): the polynomial to transform is the sum of W[p] and what the peer CTA left in W[p + 2]; the
// parked values then overwrite the peer's contribution at the very positions this thread has just read
template <int H, bool ADD_PARKED = false> NB_HD void phase_inv3_split_a(int p, int row, int u, u64 *w_all)
{
    const u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 *x = w_all + (p + 2) * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[8];
    static_for<0, 4>([&](auto PI) {
        constexpr int pi = 4 * H + decltype(PI)::value;
        constexpr int k = 2 * decltype(PI)::value;
        ld2(w + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[k], v[k + 1]);
        if constexpr (ADD_PARKED) {
            u64 r0, r1;
            ld2(x + 16 * u + 2 * ((pi ^ (2 * u)) & 7), r0, r1);
            v[k] = ff_add(v[k], r0);
            v[k + 1] = ff_add(v[k + 1], r1);
        }
    });
    dit16_half_a<H>(v);
    static_for<0, 4>([&](auto PI) {
        constexpr int pi = 4 * H + decltype(PI)::value;
        st2(x + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[2 * decltype(PI)::value], v[2 * decltype(PI)::value + 1]);
    });
}
template <int H> NB_HD void phase_inv3_split_b(int p, int row, int u, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    const u64 *x = w_all + (p + 2) * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[16], o[8];
    load16_b(v, x, u);
    dit16_half_b<H>(v, v + 8, o);
    static_for<0, 4>([&](auto PI) {
        constexpr int pi = 4 * H + decltype(PI)::value;
        st2(w + 16 * u + 2 * ((pi ^ (2 * u)) & 7), o[2 * decltype(PI)::value], o[2 * decltype(PI)::value + 1]);
    });
}

// inv2: the four 4-point transforms of a task are independent; half H takes e = 2 H, 2 H + 1 (no exchange)
template <int G, int H> NB_HD void inv2_twiddle_half(u64 *v8)        // v8[a * 2 + e'], e = 2 H + e'
{
    static_for<1, 4>([&](auto U) {
        constexpr int u = decltype(U)::value;
        constexpr int kappa = brev(u, 2);
        static_for<0, 2>([&](auto E) {
            constexpr int e = 2 * H + decltype(E)::value;
            v8[u * 2 + decltype(E)::value] = ff_shl<(192 - (3 * kappa * (4 * G + e)) % 192) % 192>(v8[u * 2 + decltype(E)::value]);
        });
    });
}
template <int H> NB_HD void phase_inv2_split(int p, int row, int g, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[8];
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        ld2(w + 16 * a + 4 * (g ^ a) + 2 * H, v[a * 2], v[a * 2 + 1]);
    });
    switch (g) {           // warp-uniform, like phase_inv2
    case 0: inv2_twiddle_half<0, H>(v); break;
    case 1: inv2_twiddle_half<1, H>(v); break;
    case 2: inv2_twiddle_half<2, H>(v); break;
    default: inv2_twiddle_half<3, H>(v); break;
    }
    static_for<0, 2>([&](auto E) { dit_inlane<2, 48, decltype(E)::value, 2>(v); });
    static_for<0, 4>([&](auto A) {
        constexpr int a = decltype(A)::value;
        st2(w + 16 * a + 4 * (g ^ a) + 2 * H, v[a * 2], v[a * 2 + 1]);
    });
}

// inv1, first half: task = (ct, mo, j2); rows 8 H .. 8 H + 7 of column j2, times the twiddles, 8-point network
template <int H> NB_HD void phase_inv1_split_a(int task, u64 *w_all, const u64 *twd_inv)
{
    const int j2 = task & 63, pp = task >> 6;
    const int p = (pp >> 1) * 4 + (pp & 1);
    const int col = col_of(j2 >> 4, j2 & 15);
    const u64 *w = w_all + p * POLY_STRIDE + col + 8 * H * ROW_STRIDE;
    u64 *x = w_all + (p + 2) * POLY_STRIDE + col + 8 * H * ROW_STRIDE;
    const u64 *twd = twd_inv + 8 * H * 64 + j2;
    u64 v[8];
    u32 hmax = 0;
    static_for<0, 8>([&](auto R) {
        constexpr int r = decltype(R)::value;
#if NB_LAZY_CANON
        v[r] = ff_mul_nc(w[r * ROW_STRIDE], twd[r * 64]);
        hmax = umax32(hmax, hi32(v[r]));
#else
        v[r] = ff_mul(w[r * ROW_STRIDE], twd[r * 64]);
#endif
    });
#if NB_LAZY_CANON
    if (canon_needed(hmax)) {
        static_for<0, 8>([&](auto R) { v[decltype(R)::value] = ff_canon_almost(v[decltype(R)::value]); });
    }
#endif
    dit16_half_a<H>(v);
    static_for<0, 8>([&](auto R) { x[decltype(R)::value * ROW_STRIDE] = v[decltype(R)::value]; });
}
// acc_poly >= 0 (pair shape): the accumulator polynomial to update, instead of polynomial pp of acc_all
template <bool ACCUMULATE, int H> NB_HD void phase_inv1_split_b(int task, i32 *acc_all, const u64 *w_all, int acc_poly = -1)
{
    const int j2 = task & 63, pp = task >> 6;
    const int ct = pp >> 1, mo = pp & 1;
    const u64 *x = w_all + (ct * 4 + mo + 2) * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    u64 a[8], t[8], o[8];
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        a[k] = x[k * ROW_STRIDE];
        t[k] = x[(8 + k) * ROW_STRIDE];
    });
    dit16_half_b<H>(a, t, o);
    i32 *acc = acc_all + (acc_poly >= 0 ? acc_poly : ct * 2 + mo) * NTT_N;
    static_for<0, 8>([&](auto K) {
        constexpr int j1 = 8 * H + decltype(K)::value;
        const int idx = 64 * j1 + j2;
        if constexpr (j1 == 0) {
            i32 r = ff_to_i32(o[0]);
            acc[idx] = ACCUMULATE ? (i32)((u32)acc[idx] + (u32)r) : r;
        } else {
            u32 r = (u32)ff_to_i32(ff_shl<96 - 6 * j1>(o[decltype(K)::value]));
            acc[idx] = ACCUMULATE ? (i32)((u32)acc[idx] - r) : (i32)(0u - r);
        }
    });
}

// ---- MAC: thread = (row, pair q): stored columns 2q, 2q+1 of every work polynomial -----------------
// bk_row: internal layout [mi][j][mo][row * 64 + stored column], plain (non-Montgomery) values.
// out polynomial mo of ciphertext ct overwrites work polynomial ct*4 + mo.
template <int CT, bool KEY_SHARED = false> NB_HD void phase_mac_row(int row, int q, u64 *w_all, const u64 *bk_row)
{
    const int pos = row * 64 + 2 * q;
#ifdef NB_BK_L1_BOUND
    // TIMING EXPERIMENT ONLY (wrong results): every key load hits the same 5 KB, i.e. the L1 -- the time a perfect
    // shared-memory / TMA staging of the key row could at best reach
    const int kpos = pos & 63;
#else
    const int kpos = pos;
#endif
    u64 bk[BK_PLANES][2];
    static_for<0, BK_PLANES>([&](auto M) {
        constexpr int m = decltype(M)::value;            // m = (mi * 2 + j) * 2 + mo; 8 + mo = correction
        if constexpr (KEY_SHARED) ld2(bk_row + m * NTT_N + kpos, bk[m][0], bk[m][1]);
        else ld2_global(bk_row + m * NTT_N + kpos, bk[m][0], bk[m][1]);
    });
    for (int ct = 0; ct < CT; ct++) {
        u64 *w = w_all + ct * 4 * POLY_STRIDE + row * ROW_STRIDE + 2 * q;
        u64 f[4][2];
        static_for<0, 4>([&](auto D) {
            constexpr int d = decltype(D)::value;        // d = mi * 2 + j
            ld2(w + d * POLY_STRIDE, f[d][0], f[d][1]);
        });
#if NB_LAZY_CANON
        u64 o[2][2];
        u32 hmax = 0;
        static_for<0, 2>([&](auto MO) {
            constexpr int mo = decltype(MO)::value;
            static_for<0, 2>([&](auto X) {
                constexpr int x = decltype(X)::value;
                const u64 fa[4] = {f[0][x], f[1][x], f[2][x], f[3][x]};
                const u64 ba[4] = {bk[0 * 2 + mo][x], bk[1 * 2 + mo][x], bk[2 * 2 + mo][x], bk[3 * 2 + mo][x]};
                o[mo][x] = ff_dot4_sub_nc(fa, ba, bk[8 + mo][x]);
                hmax = umax32(hmax, hi32(o[mo][x]));
            });
        });
        if (canon_needed(hmax)) {
            static_for<0, 4>([&](auto I) {
                constexpr int i = decltype(I)::value;
                o[i >> 1][i & 1] = ff_canon_almost(o[i >> 1][i & 1]);
            });
        }
        st2(w, o[0][0], o[0][1]);
        st2(w + POLY_STRIDE, o[1][0], o[1][1]);
#else
        static_for<0, 2>([&](auto MO) {
            constexpr int mo = decltype(MO)::value;
            u64 o[2];
            static_for<0, 2>([&](auto X) {
                constexpr int x = decltype(X)::value;
                const u64 fa[4] = {f[0][x], f[1][x], f[2][x], f[3][x]};
                const u64 ba[4] = {bk[0 * 2 + mo][x], bk[1 * 2 + mo][x], bk[2 * 2 + mo][x], bk[3 * 2 + mo][x]};
                o[x] = ff_sub(ff_dot4(fa, ba), bk[8 + mo][x]);
            });
            st2(w + mo * POLY_STRIDE, o[0], o[1]);
        });
#endif
    }
}

// all 16 rows x 32 pairs, Cfg::THREADS threads
template <class Cfg = BrDefault, bool KEY_SHARED = false> NB_HD void phase_mac(int tid, u64 *w_all, const u64 *bk_row)
{
    for (int row = tid >> 5; row < 16; row += Cfg::THREADS / 32) phase_mac_row<Cfg::CT, KEY_SHARED>(row, tid & 31, w_all, bk_row);
}

// ---- quarter-split inverse phases (pair shape) ----------------------------------------------------------------------
// Four threads (of different warps) per 16-element inverse task.  The 16-point decimation-in-time network is two layers
// inside the blocks {4 B .. 4 B + 3} (a 4-point network, root 2^48) followed by two layers inside the residue classes
// {R, R + 4, R + 8, R + 12} (pairs (R, R + 4) and (R + 8, R + 12) with twiddle 2^(-24 R), then (R, R + 8) with
// 2^(-12 R) and (R + 4, R + 12) with 2^(-12 (R + 4))).  Quarter B runs the first two layers on its block and parks the
// four values in work polynomial p + 2; after a CTA barrier quarter R reads the parked values of its residue class and
// finishes those four outputs.  Same barrier count as the two-way split, about half of its instructions per thread.
template <int E> NB_HD void dit_pair(u64 &a, u64 &b)       // one butterfly of dit_inlane with inverse twiddle 2^-E
{
    if constexpr (E > 0 && E < 96) {
        const u64 x = a, t = ff_shl<96 - E>(b);
        a = ff_sub(x, t);
        b = ff_add(x, t);
    } else {
        const u64 x = a, t = ff_shl<(192 - E) % 192>(b);
        a = ff_add(x, t);
        b = ff_sub(x, t);
    }
}
template <int R> NB_HD void dit16_quarter_b(u64 *x)       // x[m] = parked element R + 4 m, becomes output element R + 4 m
{
    dit_pair<24 * R>(x[0], x[1]);
    dit_pair<24 * R>(x[2], x[3]);
    dit_pair<12 * R>(x[0], x[2]);
    dit_pair<12 * R + 48>(x[1], x[3]);
}
// inv3, first stage: task (p, row, u), logical columns 4 B .. 4 B + 3 of block u (pairs 2 B, 2 B + 1)
template <int B, bool ADD_PARKED> NB_HD void phase_inv3_quarter_a(int p, int row, int u, u64 *w_all)
{
    const u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    u64 *x = w_all + (p + 2) * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[4];
    static_for<0, 2>([&](auto PI) {
        constexpr int pi = 2 * B + decltype(PI)::value;
        constexpr int k = 2 * decltype(PI)::value;
        ld2(w + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[k], v[k + 1]);
        if constexpr (ADD_PARKED) {
            u64 r0, r1;
            ld2(x + 16 * u + 2 * ((pi ^ (2 * u)) & 7), r0, r1);
            v[k] = ff_add(v[k], r0);
            v[k + 1] = ff_add(v[k + 1], r1);
        }
    });
    dit_inlane<2, 48, 0>(v);
    static_for<0, 2>([&](auto PI) {
        constexpr int pi = 2 * B + decltype(PI)::value;
        st2(x + 16 * u + 2 * ((pi ^ (2 * u)) & 7), v[2 * decltype(PI)::value], v[2 * decltype(PI)::value + 1]);
    });
}
// inv3, second stage: logical columns R, R + 4, R + 8, R + 12 of block u
template <int R> NB_HD void phase_inv3_quarter_b(int p, int row, int u, u64 *w_all)
{
    u64 *w = w_all + p * POLY_STRIDE + row * ROW_STRIDE;
    const u64 *x = w_all + (p + 2) * POLY_STRIDE + row * ROW_STRIDE;
    u64 v[4];
    static_for<0, 4>([&](auto M) {
        constexpr int b = R + 4 * decltype(M)::value;
        v[decltype(M)::value] = x[16 * u + 2 * (((b >> 1) ^ (2 * u)) & 7) + (b & 1)];
    });
    dit16_quarter_b<R>(v);
    static_for<0, 4>([&](auto M) {
        constexpr int b = R + 4 * decltype(M)::value;
        w[16 * u + 2 * (((b >> 1) ^ (2 * u)) & 7) + (b & 1)] = v[decltype(M)::value];
    });
}
// inv1, first stage: task = (polynomial pp, column j2); rows 4 B .. 4 B + 3 times the twiddles, 4-point network
template <int B> NB_HD void phase_inv1_quarter_a(int task, u64 *w_all, const u64 *twd_inv)
{
    const int j2 = task & 63, pp = task >> 6;
    const int p = (pp >> 1) * 4 + (pp & 1);
    const int col = col_of(j2 >> 4, j2 & 15);
    const u64 *w = w_all + p * POLY_STRIDE + col + 4 * B * ROW_STRIDE;
    u64 *x = w_all + (p + 2) * POLY_STRIDE + col + 4 * B * ROW_STRIDE;
    const u64 *twd = twd_inv + 4 * B * 64 + j2;
    u64 v[4];
    u32 hmax = 0;
    static_for<0, 4>([&](auto R) {
        constexpr int r = decltype(R)::value;
#if NB_LAZY_CANON
        v[r] = ff_mul_nc(w[r * ROW_STRIDE], twd[r * 64]);
        hmax = umax32(hmax, hi32(v[r]));
#else
        v[r] = ff_mul(w[r * ROW_STRIDE], twd[r * 64]);
#endif
    });
#if NB_LAZY_CANON
    if (canon_needed(hmax)) {
        static_for<0, 4>([&](auto R) { v[decltype(R)::value] = ff_canon_almost(v[decltype(R)::value]); });
    }
#endif
    dit_inlane<2, 48, 0>(v);
    static_for<0, 4>([&](auto R) { x[decltype(R)::value * ROW_STRIDE] = v[decltype(R)::value]; });
}
// inv1, second stage: outputs j1 = R + 4 m of column j2 into accumulator polynomial acc_poly
template <int R> NB_HD void phase_inv1_quarter_b(int task, i32 *acc_all, const u64 *w_all, int acc_poly)
{
    const int j2 = task & 63, pp = task >> 6;
    const u64 *x = w_all + ((pp >> 1) * 4 + (pp & 1) + 2) * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    u64 v[4];
    static_for<0, 4>([&](auto M) { v[decltype(M)::value] = x[(R + 4 * decltype(M)::value) * ROW_STRIDE]; });
    dit16_quarter_b<R>(v);
    i32 *acc = acc_all + acc_poly * NTT_N;
    static_for<0, 4>([&](auto M) {
        constexpr int j1 = R + 4 * decltype(M)::value;
        const int idx = 64 * j1 + j2;
        if constexpr (j1 == 0) {
            acc[idx] = (i32)((u32)acc[idx] + (u32)ff_to_i32(v[0]));
        } else {
            acc[idx] = (i32)((u32)acc[idx] - (u32)ff_to_i32(ff_shl<96 - 6 * j1>(v[decltype(M)::value])));
        }
    });
}

// ---- pair shape: one ciphertext on a cluster of two CTAs (two SMs), 256 threads each ---------------------------------
// CTA `rank` (= mi) owns accumulator polynomial mi: it decomposes it into its two digit polynomials (W[0], W[1]),
// transforms them (split forward phases, 128 tasks x 2 halves), and multiplies them with the four key planes
// (mi, j, mo): two partial sums per point, one for each output polynomial.  The partial sum for its OWN output
// polynomial (mo = rank) stays in W[par]; the other one goes into the peer's W[par + 2] through distributed shared
// memory, par = step parity.  After one cluster barrier each CTA adds what it received to what it kept (fused into the
// first inverse pass), runs the inverse transform of its output polynomial (quarter-split inverse phases, four threads per
// task, W[par + 2] doubling as the exchange area like in the single-CTA shapes) and updates its accumulator polynomial:
// everything but the exchange of 8 KB per step and direction is local to a CTA.  Alternating par is what makes the
// exchange safe without a second synchronisation per step: the peer's next remote stores (into W[(par ^ 1) + 2]) can
// start while this CTA is still in the inverse phases of the current step (W[par], W[par + 2]); the stores after those
// need this CTA's next partial sums first, which it sends after finishing the current step.
// The correction plane of the unsigned digits (BK planes 8, 9) is subtracted by rank 0 alone.
// The per-thread instruction stream is shorter than that of the 512-thread shape and each SM carries 8 warps, not 16.
constexpr int PAIR_THREADS = 256;
constexpr int PAIR_POLYS = 4;
constexpr int PAIR_INV_WORKERS = 128;                 // threads with work in the inverse phases (64 tasks x 2 halves)

NB_HD void pair_fwd1(int tid, const i32 *acc, u64 *w, const u64 *twd, const int *rot)
{
    const int h = tid >> 7, t = tid & 127;             // task = (j, j2)
    if (h) phase_fwd1_split<true, 1>(t, acc, w, twd, rot); else phase_fwd1_split<true, 0>(t, acc, w, twd, rot);
}
NB_HD void pair_fwd2(int tid, u64 *w)
{
    const int h = tid >> 7, t = tid & 127;
    const int g = t >> 5, p = (t >> 4) & 1, row = t & 15;          // g is warp-uniform
    if (h) phase_fwd2_split<1>(p, row, g, w); else phase_fwd2_split<0>(p, row, g, w);
}
NB_HD void pair_fwd3_load(int tid, const u64 *w, u64 *v)
{
    const int t = tid & 127;
    phase_fwd3_split_load(t >> 6, (t >> 2) & 15, t & 3, w, v);
}
NB_HD void pair_fwd3_finish(int tid, u64 *w, const u64 *v)
{
    const int h = tid >> 7, t = tid & 127;
    if (h) phase_fwd3_split_finish<1>(t >> 6, (t >> 2) & 15, t & 3, w, v); else phase_fwd3_split_finish<0>(t >> 6, (t >> 2) & 15, t & 3, w, v);
}
// MAC of one point pair for ONE output polynomial mo: the two partial sums sum_j F_j * key[j][mo] (- correction).
// key4: this CTA's four key planes [j * 2 + mo][row * 64 + stored column]; corr2: the two correction planes or null
// (rank 1).  KEY_SHARED: the planes were staged in shared memory (the device kernel), else they are read in place.
template <bool KEY_SHARED> NB_HD void mac_pair_point(int row, int q, const u64 *w_all, const u64 *key4, const u64 *corr2, int mo, u64 &o0, u64 &o1)
{
    const int pos = row * 64 + 2 * q;
    u64 bk[2][2], cr[2] = {0, 0}, f[2][2];
    static_for<0, 2>([&](auto J) {
        constexpr int j = decltype(J)::value;
        if constexpr (KEY_SHARED) ld2(key4 + (j * 2 + mo) * NTT_N + pos, bk[j][0], bk[j][1]);
        else ld2_global(key4 + (j * 2 + mo) * NTT_N + pos, bk[j][0], bk[j][1]);
    });
    if (corr2) {
        if constexpr (KEY_SHARED) ld2(corr2 + mo * NTT_N + pos, cr[0], cr[1]);
        else ld2_global(corr2 + mo * NTT_N + pos, cr[0], cr[1]);
    }
    const u64 *w = w_all + row * ROW_STRIDE + 2 * q;
    ld2(w, f[0][0], f[0][1]);
    ld2(w + POLY_STRIDE, f[1][0], f[1][1]);
    const u64 fa0[2] = {f[0][0], f[1][0]}, ba0[2] = {bk[0][0], bk[1][0]};
    const u64 fa1[2] = {f[0][1], f[1][1]}, ba1[2] = {bk[0][1], bk[1][1]};
    o0 = ff_dot2_sub_nc(fa0, ba0, cr[0]);
    o1 = ff_dot2_sub_nc(fa1, ba1, cr[1]);
#if NB_LAZY_CANON
    if (canon_needed(umax32(hi32(o0), hi32(o1))))
#endif
    {
        o0 = ff_canon_almost(o0);
        o1 = ff_canon_almost(o1);
    }
}
// The whole MAC of a thread: first the partial sums for the PEER's output polynomial (mo = 1 - rank), handed to
// send(offset, x, y) -- a store at u64 offset `offset` of the peer's work polynomials: distributed shared memory on the
// device, the other CTA's array in the host emulation -- so that they travel while this thread computes the partial sums
// it keeps (mo = rank, into W[par], over the digit transform it has just read).
template <bool KEY_SHARED, class Send>
NB_HD void pair_mac(int tid, u64 *w, Send send, const u64 *key4, const u64 *corr2, int rank, int par)
{
    const int q = tid & 31;
    for (int row = tid >> 5; row < 16; row += PAIR_THREADS / 32) {
        u64 o0, o1;
        mac_pair_point<KEY_SHARED>(row, q, w, key4, corr2, 1 - rank, o0, o1);
        send((par + 2) * POLY_STRIDE + row * ROW_STRIDE + 2 * q, o0, o1);
    }
    for (int row = tid >> 5; row < 16; row += PAIR_THREADS / 32) {
        u64 o0, o1;
        mac_pair_point<KEY_SHARED>(row, q, w, key4, corr2, rank, o0, o1);
        st2(w + par * POLY_STRIDE + row * ROW_STRIDE + 2 * q, o0, o1);
    }
}
// key planes a CTA of the pair needs per step: its four (j, mo) planes, rank 0 also the two correction planes
constexpr int PAIR_KEY_PLANES = 6;
constexpr int PAIR_EXCHANGE_BYTES = NTT_N * (int)sizeof(u64);       // what a CTA receives per step
// inverse phases of output polynomial W[par].  inv3 and inv1: all 256 threads, four per task (quarter = tid / 64, whole
// warps; task t = tid % 64 = (row, u) resp. j2).  inv2: the two-way split on tid < PAIR_INV_WORKERS, task t = (g, row) --
// its four 4-point transforms per task are independent, and the other warps use the time to request the next key row.
template <template <int> class F, class... A> NB_HD void pair_quarter_dispatch(int quarter, A... a)
{
    switch (quarter) {                                 // warp-uniform
    case 0: F<0>::run(a...); break;
    case 1: F<1>::run(a...); break;
    case 2: F<2>::run(a...); break;
    default: F<3>::run(a...); break;
    }
}
template <int Q> struct PairInv3A { NB_HD static void run(int t, u64 *w, int par) { phase_inv3_quarter_a<Q, true>(par, t >> 2, t & 3, w); } };
template <int Q> struct PairInv3B { NB_HD static void run(int t, u64 *w, int par) { phase_inv3_quarter_b<Q>(par, t >> 2, t & 3, w); } };
template <int Q> struct PairInv1A { NB_HD static void run(int t, u64 *w, const u64 *twd_inv, int par) { phase_inv1_quarter_a<Q>(par * 64 + t, w, twd_inv); } };
template <int Q> struct PairInv1B { NB_HD static void run(int t, i32 *acc, const u64 *w, int par) { phase_inv1_quarter_b<Q>(par * 64 + t, acc, w, 0); } };
NB_HD void pair_inv3_a(int tid, u64 *w, int par) { pair_quarter_dispatch<PairInv3A>(tid >> 6, tid & 63, w, par); }
NB_HD void pair_inv3_b(int tid, u64 *w, int par) { pair_quarter_dispatch<PairInv3B>(tid >> 6, tid & 63, w, par); }
NB_HD void pair_inv2(int tid, u64 *w, int par)         // tid < PAIR_INV_WORKERS
{
    // 16 tasks per g: two values of g per warp, the twiddle switch of phase_inv2_split runs twice (the only
    // divergent piece of the shape: 6 shifts per thread)
    const int h = tid >> 6, t = tid & 63;
    if (h) phase_inv2_split<1>(par, t & 15, t >> 4, w); else phase_inv2_split<0>(par, t & 15, t >> 4, w);
}
NB_HD void pair_inv1_a(int tid, u64 *w, const u64 *twd_inv, int par) { pair_quarter_dispatch<PairInv1A>(tid >> 6, tid & 63, w, twd_inv, par); }
NB_HD void pair_inv1_b(int tid, i32 *acc, const u64 *w, int par) { pair_quarter_dispatch<PairInv1B>(tid >> 6, tid & 63, acc, w, par); }

// ---- inv1: task = (ct, mo, j2): reads W[ct*4+mo], writes ACC[ct][mo] --------------------------------
// twd_inv: [row][j2] = psi^-(j2 (2 k1 + 1)) / 1024.  ACCUMULATE: acc += result, else acc = result.
template <bool ACCUMULATE>
NB_HD void phase_inv1(int task, i32 *acc_all, const u64 *w_all, const u64 *twd_inv)
{
    const int j2 = task & 63, pp = task >> 6;          // pp = ct * 2 + mo
    const int ct = pp >> 1, mo = pp & 1;
    const u64 *w = w_all + (ct * 4 + mo) * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    u64 v[16];
    load_twiddled(v, w, twd_inv + j2);
    run_network<NetDit16>(v, [&]() { load_twiddled(v, w, twd_inv + j2); });
    i32 *acc = acc_all + (ct * 2 + mo) * NTT_N;
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        const int idx = 64 * j1 + j2;
        // 2^(-6 j1) = -2^(96 - 6 j1) for j1 >= 1: shift by the positive amount and subtract (the centred lift is odd)
        if constexpr (j1 == 0) {
            i32 r = ff_to_i32(v[0]);
            acc[idx] = ACCUMULATE ? (i32)((u32)acc[idx] + (u32)r) : r;
        } else {
            u32 r = (u32)ff_to_i32(ff_shl<96 - 6 * j1>(v[j1]));
            acc[idx] = ACCUMULATE ? (i32)((u32)acc[idx] - r) : (i32)(0u - r);
        }
    });
}

// ---- stand-alone transforms (nb_ntt_*): same passes, 4 polynomials per sweep of 256 threads ----------
constexpr int NTT_SWEEP_POLYS = 4;
constexpr int NTT_SWEEP_THREADS = 64 * NTT_SWEEP_POLYS;

// stored position (row, stored column) of the transformed element with natural index k
NB_HD int w_position_of_natural(int k)
{
    int k1 = k & 15, k2 = k >> 4;
    int row = brev(k1, 4), u = brev(k2 & 3, 2), i = brev(k2 >> 2, 4);
    return row * ROW_STRIDE + col_of(u, i);
}

// first pass with generic inputs: task = (poly p, j2); x = canonical field elements, natural order
NB_HD void phase_fwd1_generic(int task, const u64 *x /* 16 values, x[j1] = in[64 j1 + j2] */, u64 *w_all, const u64 *twd)
{
    const int j2 = task & 63, p = task >> 6;
    u64 v[16];
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        v[j1] = ff_shl<6 * j1>(x[j1]);
    });
    run_network<NetDif16>(v, [&]() { static_for<0, 16>([&](auto J) { constexpr int j1 = decltype(J)::value; v[j1] = ff_shl<6 * j1>(x[j1]); }); });
    u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    store_twiddled(v, w, twd + j2);
}
// first pass with Torus32 inputs (i32_conversion): the conversion and the twist are one step (ff_twist_i32)
NB_HD void phase_fwd1_i32(int task, const i32 *x /* 16 values, x[j1] = in[64 j1 + j2] */, u64 *w_all, const u64 *twd)
{
    const int j2 = task & 63, p = task >> 6;
    u64 v[16];
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        v[j1] = ff_twist_i32<j1>(x[j1]);
    });
    run_network<NetDif16>(v, [&]() { static_for<0, 16>([&](auto J) { constexpr int j1 = decltype(J)::value; v[j1] = ff_twist_i32<j1>(x[j1]); }); });
    u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    store_twiddled(v, w, twd + j2);
}
// last inverse pass with generic outputs: y[j1] = out[64 j1 + j2], almost-canonical ([0, p])
NB_HD void phase_inv1_generic(int task, u64 *y, const u64 *w_all, const u64 *twd_inv)
{
    const int j2 = task & 63, p = task >> 6;
    const u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    u64 v[16];
    load_twiddled(v, w, twd_inv + j2);
    run_network<NetDit16>(v, [&]() { load_twiddled(v, w, twd_inv + j2); });
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        y[j1] = ff_shl<(192 - 6 * j1) % 192>(v[j1]);
    });
}

// last inverse pass with Torus32 outputs: 2^(-6 j1) = -2^(96 - 6 j1) for j1 >= 1 (the centred lift is odd), like
// the fused kernel's inv1
NB_HD void phase_inv1_i32(int task, i32 *y, const u64 *w_all, const u64 *twd_inv)
{
    const int j2 = task & 63, p = task >> 6;
    const u64 *w = w_all + p * POLY_STRIDE + col_of(j2 >> 4, j2 & 15);
    u64 v[16];
    load_twiddled(v, w, twd_inv + j2);
    run_network<NetDit16>(v, [&]() { load_twiddled(v, w, twd_inv + j2); });
    y[0] = ff_to_i32(v[0]);
    static_for<1, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        y[j1] = (i32)(0u - (u32)ff_to_i32(ff_shl<96 - 6 * j1>(v[j1])));
    });
}

// thread -> task maps (it = sweep).  The inverse maps return false for threads without a task (whole warps).
template <class Cfg = BrDefault> NB_HD void map_fwd2(int tid, int it, int &p, int &row, int &g)
{
    constexpr int Q = Cfg::THREADS / 4;                // threads per value of g (>= 32: g is warp-uniform)
    g = tid / Q;
    int x = it * Q + (tid % Q);
    p = x >> 4; row = x & 15;
}
template <class Cfg = BrDefault> NB_HD void map_fwd3(int tid, int it, int &p, int &row, int &u)
{
    u = tid & 3; row = (tid >> 2) & 15; p = it * (Cfg::THREADS / 64) + (tid >> 6);
}
// inverse passes act on polynomials ct*4 + mo only (half of the work polynomials)
template <class Cfg = BrDefault> NB_HD bool map_inv2(int tid, int &p, int &row, int &g)
{
    constexpr int Q = Cfg::THREADS / 4;
    g = tid / Q;
    int x = tid % Q;                                   // 2 CT polys x 16 rows
    int pp = x >> 4; row = x & 15;
    p = (pp >> 1) * 4 + (pp & 1);
    return x < 32 * Cfg::CT;
}
// split inverse phases: h = thread half (warps 0 .. THREADS/64 - 1: h = 0, the others h = 1), t = task of the unsplit map
// (threads beyond twice the task count -- the upper half of the wide2 shape -- have no inverse work: returns false)
template <class Cfg> NB_HD bool map_split(int tid, int &h, int &t)
{
    h = tid >= Cfg::INV_TASKS;
    t = tid - h * Cfg::INV_TASKS;
    return tid < 2 * Cfg::INV_TASKS;
}
// split forward phases: 256 CT tasks, h = 0 for the lower half of the CTA's threads
template <class Cfg> NB_HD void map_split_fwd(int tid, int &h, int &t) { h = tid >= 256 * Cfg::CT; t = tid - h * 256 * Cfg::CT; }
// inv2 tasks of the split phases: t in [0, INV_TASKS), g warp-uniform (32 consecutive tasks per g and polynomial pair)
template <class Cfg> NB_HD void map_inv2_split(int t, int &p, int &row, int &g)
{
    constexpr int Q = Cfg::INV_TASKS / 4;              // tasks per value of g: 2 CT polynomials x 16 rows
    g = t / Q;
    const int x = t % Q, pp = x >> 4;
    row = x & 15;
    p = (pp >> 1) * 4 + (pp & 1);
}

template <class Cfg = BrDefault> NB_HD bool map_inv3(int tid, int &p, int &row, int &u)
{
    u = tid & 3; row = (tid >> 2) & 15;
    int pp = tid >> 6;
    p = (pp >> 1) * 4 + (pp & 1);
    return pp < 2 * Cfg::CT;
}

// ---- FP64 step (throughput shape, keys with integral coefficients) --------------------------------------------------
// The external product as an exact floating-point computation (DESIGN.md section 3): every coefficient the step
// produces is an integer, so a transform whose rounding error stays below 1/2 gives the same bits as the NTT.  The key
// polynomial k (centred 32-bit integers) is split as k = k_hi 2^16 + k_lo with k_lo in [-2^15, 2^15), k_hi in
// [-2^15, 2^15]; each half's product with the signed 10-bit digits is below 2^37 in magnitude and is rounded to an
// integer on its own; the step then adds lo + (hi << 16) mod 2^32 to the accumulator.
// Negacyclic fold: a polynomial a of degree < 1024 becomes z_j = (a_j + i a_{j+512}) w^j, j < 512, w = e^{i pi / 1024};
// its 512-point DFT (root e^{-2 pi i / 512}) is a evaluated at 512 roots of X^1024 + 1 that carry z^512 = i, so the
// point-wise product of two such spectra is the spectrum of the negacyclic product.
// The DFT is a radix 8 x 16 x 4 plan, decimation in frequency (natural order in, digit-reversed order out); the
// inverse runs the mirrored passes, so the MAC works point-wise and nothing is reordered:
//     pass 1, task n0 < 64:          x[n0 + 64 m]             -> DFT8 over m, times W512^(n0 k1) -> x[n0 + 64 k1]
//     pass 2, task (k1, n2 < 4):     x[64 k1 + n2 + 4 m]      -> DFT16, times W64^(n2 k2)       -> x[64 k1 + n2 + 4 k2]
//     pass 3, task (k1, k2):         x[64 k1 + 4 k2 + m]      -> DFT4                           -> x[64 k1 + 4 k2 + k3]
// leaving X[k1 + 8 k2 + 128 k3] at position 64 k1 + 4 k2 + k3.  Pass 3 is fused with the MAC and the first inverse
// pass: a thread holds the 4 points of group g = 16 k1 + k2 of all 4 digit spectra, transforms them, and for one
// output spectrum at a time multiplies with the key, runs the inverse DFT4 and stores.  A step is five
// barrier-separated phases: fwd1, fwd2, pass 3, inv2, inv1.  Shared-memory positions and thread maps: fft_layout.cuh.
// Every floating-point operation is an explicit, correctly rounded add / mul / fma (__dadd_rn & co. are never
// contracted by the compiler), in the order the error bound of DESIGN.md section 3 assumes; the host emulation
// (csrc/host_emul.cpp, no FMA contraction) computes the same bits.
struct cplx {
    double re, im;
};
// Engine bootstrap-key row, FP64 part: 16 spectra [(m = (mi * 2 + j) * 2 + mo) * 2 + h][512] (h = 0: k_lo, 1: k_hi),
// unpadded, complex doubles, each in the order of fft_key_pos; it follows the NTT planes of the same row.
constexpr int BK_FFT_SPECTRA = 16;
constexpr int BK_FFT_U64 = BK_FFT_SPECTRA * FFT_M * 2;
static_assert(BK_ROW_U64 == BK_NTT_U64 + BK_FFT_U64, "key row layout");
// table (tables.h: FftTables), complex: the pass-1 twiddles merged with the n0 part of the twist,
// T[k1][n0] = w^n0 W512^(n0 k1), stored [k1][n0] so that the consecutive n0 of a warp read consecutive 16-byte
// elements.  The rest of the twist, w^(64 m), and the pass-2 twiddles are compile-time constants (fft_w64).
// The device copy continues at FFT_TAB_ROOTS with the multi-bit step's 2048th roots of unity R[e] = e^{2 pi i e / 2048}
// (FftTables::roots; fft_phase_mac_mb).
constexpr int FFT_TAB_T1 = 0, FFT_TAB_CPLX = 512, FFT_TAB_ROOTS = FFT_TAB_CPLX, FFT_ROOTS = 2048;
NB_HD constexpr int fft_tab_t1(int k1, int n0) { return FFT_TAB_T1 + k1 * 64 + n0; }

#if defined(__CUDA_ARCH__)
NB_HD double d_add(double a, double b) { return __dadd_rn(a, b); }
NB_HD double d_sub(double a, double b) { return __dsub_rn(a, b); }
NB_HD double d_mul(double a, double b) { return __dmul_rn(a, b); }
NB_HD double d_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
// a table load (through the L1) that the compiler can neither merge with the same load of another phase nor move across
// a barrier: fwd1 and inv1 read the same table entries, and ptxas merges two read-only (.nc) loads of one address even
// across barriers -- it then keeps fwd1's 8 values (32 registers) live through the whole step, and the step spills
NB_HD cplx ld_cplx_tab(const cplx *p)
{
    cplx t;
    asm volatile("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(t.re), "=d"(t.im) : "l"(p));
    return t;
}
NB_HD cplx ld_cplx(const cplx *p)
{
    const double2 t = *reinterpret_cast<const double2 *>(p);
    return {t.x, t.y};
}
NB_HD void st_cplx(cplx *p, cplx v) { *reinterpret_cast<double2 *>(p) = make_double2(v.re, v.im); }
NB_HD cplx ld_cplx_stream(const cplx *p)           // key spectra: read once per CTA, keep them out of the L1
{
    const double2 t = __ldcg(reinterpret_cast<const double2 *>(p));
    return {t.x, t.y};
}
NB_HD double d_from_words(u32 hi, u32 lo) { return __hiloint2double((int)hi, (int)lo); }
NB_HD u32 d_lo_word(double x) { return (u32)__double2loint(x); }
#else
NB_HD double d_add(double a, double b) { return a + b; }
NB_HD double d_sub(double a, double b) { return a - b; }
NB_HD double d_mul(double a, double b) { return a * b; }
NB_HD double d_fma(double a, double b, double c) { return std::fma(a, b, c); }
NB_HD cplx ld_cplx_tab(const cplx *p) { return *p; }
NB_HD cplx ld_cplx(const cplx *p) { return *p; }
NB_HD void st_cplx(cplx *p, cplx v) { *p = v; }
NB_HD cplx ld_cplx_stream(const cplx *p) { return *p; }
NB_HD double d_from_words(u32 hi, u32 lo)
{
    const uint64_t b = (uint64_t)hi << 32 | lo;
    double x;
    memcpy(&x, &b, sizeof x);
    return x;
}
NB_HD u32 d_lo_word(double x)
{
    uint64_t b;
    memcpy(&b, &x, sizeof b);
    return (u32)b;
}
#endif
// Conversions between doubles and integers without the conversion unit (I2F.F64 / F2I.F64, a quarter of the FP64
// rate on sm_90), so the step stays on the FP64 pipe:
// the digit u - 512 of u in [0, 1023]: the words 0x43300000 : u are the double 2^52 + u, and one exact subtraction
// removes 2^52 + 512
NB_HD double d_digit(u32 u) { return d_add(d_from_words(0x43300000u, u), -(0x1p52 + 512)); }
// round(x) mod 2^32 for |x| < 2^51: x + 1.5 2^52 lies in [2^52, 2^53), where the spacing of doubles is 1, so the
// correctly rounded sum is 1.5 2^52 + round(x) (to nearest, ties to even, as __double2ll_rn), and its low word is
// round(x) mod 2^32 (the low word of 1.5 2^52 is 0)
NB_HD i32 d_rint_lo32(double x) { return (i32)d_lo_word(d_add(x, 0x1.8p52)); }

NB_HD cplx c_add(cplx a, cplx b) { return {d_add(a.re, b.re), d_add(a.im, b.im)}; }
NB_HD cplx c_sub(cplx a, cplx b) { return {d_sub(a.re, b.re), d_sub(a.im, b.im)}; }
// a * w and a * conj(w): one product and one fma per component
NB_HD cplx c_mul(cplx a, cplx w) { return {d_fma(a.re, w.re, -d_mul(a.im, w.im)), d_fma(a.re, w.im, d_mul(a.im, w.re))}; }
NB_HD cplx c_mul_conj(cplx a, cplx w) { return {d_fma(a.re, w.re, d_mul(a.im, w.im)), d_fma(a.im, w.re, -d_mul(a.re, w.im))}; }
// acc + a * b (complex), four fmas
NB_HD cplx c_mac(cplx acc, cplx a, cplx b)
{
    return {d_fma(-a.im, b.im, d_fma(a.re, b.re, acc.re)), d_fma(a.im, b.re, d_fma(a.re, b.im, acc.im))};
}
// times -i (forward) / +i (inverse): exact
template <bool INV> NB_HD cplx c_mul_mi(cplx a) { return INV ? cplx{-a.im, a.re} : cplx{a.im, -a.re}; }
// times e^{-+ i pi / 4} = (1 -+ i) sqrt(1/2): one addition and one product per component with the rounded constant
template <bool INV> NB_HD cplx c_mul_w8(cplx a)
{
    constexpr double S = 0.70710678118654752440;
    return INV ? cplx{d_mul(d_sub(a.re, a.im), S), d_mul(d_add(a.re, a.im), S)} : cplx{d_mul(d_add(a.re, a.im), S), d_mul(d_sub(a.im, a.re), S)};
}

// W64^e = e^{-2 pi i e / 64}: cos (2 pi r / 64), r <= 16, evaluated in long double and rounded once (as the tables),
// the quadrant e / 16 applied exactly (swap and sign).  Evaluated at compile time: the twiddles of pass 2 are operands
// from the constant bank, not loads into registers.
NB_HD constexpr cplx fft_w64(int e)
{
    constexpr double c[17] = {1, 0.99518472667219693, 0.98078528040323043, 0.95694033573220882, 0.92387953251128674,
                              0.88192126434835505, 0.83146961230254524, 0.77301045336273699, 0.70710678118654757,
                              0.63439328416364549, 0.55557023301960218, 0.47139673682599764, 0.38268343236508978,
                              0.29028467725446239, 0.19509032201612828, 0.098017140329560604, 0};
    const int q = (e >> 4) & 3, r = e & 15;
    const double re = c[r], im = -c[16 - r];
    return q == 0 ? cplx{re, im} : q == 1 ? cplx{im, -re} : q == 2 ? cplx{-re, -im} : cplx{-im, re};
}
// y[k] *= W64^(N2 k) (forward) / its conjugate (inverse), k = 1 .. 15
template <int N2, bool INV> NB_HD void fft_w64_twiddle(cplx *y)
{
    static_for<1, 16>([&](auto K) {
        constexpr int k = decltype(K)::value;
        constexpr cplx w = fft_w64(N2 * k);
        y[k] = INV ? c_mul_conj(y[k], w) : c_mul(y[k], w);
    });
}
// the same for a run-time n2 (warp-uniform in the step: fft_pass2_task); n2 = 0 multiplies by 1
template <bool INV> NB_HD void fft_w64_twiddle(int n2, cplx *y)
{
    switch (n2) {
    case 0: break;
    case 1: fft_w64_twiddle<1, INV>(y); break;
    case 2: fft_w64_twiddle<2, INV>(y); break;
    default: fft_w64_twiddle<3, INV>(y); break;
    }
}

// 8-point DFT in place, natural order in and out: y[k] = sum_m y[m] e^{-+ 2 pi i m k / 8} (INV: the + sign), as three
// radix-2 decimation-in-frequency layers.  Multiplications by -+i are exact (swap and sign); by e^{-+ i pi / 4} one
// addition and one product per component with the rounded constant sqrt(1/2).
template <bool INV> NB_HD void dft8(cplx *y)
{
    cplx t[8];
    static_for<0, 4>([&](auto M) {
        constexpr int m = decltype(M)::value;
        t[m] = c_add(y[m], y[m + 4]);
        t[m + 4] = c_sub(y[m], y[m + 4]);
    });
    // t[4 + m] *= W8^m, W8 = e^{-+ i pi / 4}; W8^3 = -+ i W8
    t[5] = c_mul_w8<INV>(t[5]);
    t[6] = c_mul_mi<INV>(t[6]);
    t[7] = c_mul_mi<INV>(c_mul_w8<INV>(t[7]));
    cplx u[8];
    static_for<0, 2>([&](auto H) {
        constexpr int h = 4 * decltype(H)::value;
        u[h + 0] = c_add(t[h + 0], t[h + 2]);
        u[h + 1] = c_add(t[h + 1], t[h + 3]);
        u[h + 2] = c_sub(t[h + 0], t[h + 2]);
        u[h + 3] = c_mul_mi<INV>(c_sub(t[h + 1], t[h + 3]));
    });
    // last layer; outputs of the DIF network are bit-reversed: position p holds y[brev3(p)]
    y[0] = c_add(u[0], u[1]); y[4] = c_sub(u[0], u[1]);
    y[2] = c_add(u[2], u[3]); y[6] = c_sub(u[2], u[3]);
    y[1] = c_add(u[4], u[5]); y[5] = c_sub(u[4], u[5]);
    y[3] = c_add(u[6], u[7]); y[7] = c_sub(u[6], u[7]);
}

// 16-point DFT in place, natural order in and out: one radix-2 decimation-in-frequency layer (pairs m, m + 8), the
// twiddles W16^(-+m) on the differences, and a DFT8 on the sums (even outputs) and one on the differences (odd
// outputs).  W16^4 = -+i is exact, W16^2 and W16^6 = -+i W16^2 take c_mul_w8, W16^1, W16^3 and W16^5 = -+i W16^1,
// W16^7 = -+i W16^3 one product and one fma per component with the rounded constants cos(pi / 8), sin(pi / 8).
template <bool INV> NB_HD void dft16(cplx *y)
{
    constexpr double C = 0.92387953251128675613, S = 0.38268343236508977173;
    constexpr cplx W1 = {C, INV ? S : -S}, W3 = {S, INV ? C : -C};
    cplx a[8], b[8];
    static_for<0, 8>([&](auto M) {
        constexpr int m = decltype(M)::value;
        a[m] = c_add(y[m], y[m + 8]);
        b[m] = c_sub(y[m], y[m + 8]);
    });
    b[1] = c_mul(b[1], W1);
    b[2] = c_mul_w8<INV>(b[2]);
    b[3] = c_mul(b[3], W3);
    b[4] = c_mul_mi<INV>(b[4]);
    b[5] = c_mul_mi<INV>(c_mul(b[5], W1));
    b[6] = c_mul_mi<INV>(c_mul_w8<INV>(b[6]));
    b[7] = c_mul_mi<INV>(c_mul(b[7], W3));
    dft8<INV>(a);
    dft8<INV>(b);
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        y[2 * k] = a[k];
        y[2 * k + 1] = b[k];
    });
}

// 4-point DFT in place, natural order in and out: two radix-2 layers, the multiplication by -+i exact
template <bool INV> NB_HD void dft4(cplx *y)
{
    const cplx a = c_add(y[0], y[2]), b = c_sub(y[0], y[2]), c = c_add(y[1], y[3]);
    const cplx d = c_mul_mi<INV>(c_sub(y[1], y[3]));
    y[0] = c_add(a, c); y[2] = c_sub(a, c);
    y[1] = c_add(b, d); y[3] = c_sub(b, d);
}

// the 8 pass-1 table values of task n0: t1[k1] = T[k1][n0]; loaded once per phase and shared by both digits (fwd1)
// or both key halves (inv1)
NB_HD void fft_load_t1(int n0, const cplx *tab, cplx *t1)
{
    static_for<0, 8>([&](auto K) { t1[decltype(K)::value] = ld_cplx_tab(tab + fft_tab_t1(decltype(K)::value, n0)); });
}
// pass 1 (forward): x[m'] = real coefficient n0 + 64 m', m' < 16 (exact small integers as doubles); fold, twist,
// DFT8 over m, twiddle, store at position n0 + 64 k1 of spectrum sp.  The twist w^(n0 + 64 m) is split: w^(64 m) =
// e^{i pi m / 16} = conj(W64^(2 m)) is a constant per m (exact for m = 0, the (1 + i) sqrt(1/2) form for m = 4), and
// w^n0, which commutes with the DFT8 over m, is part of the table T[k1][n0] = w^n0 W512^(n0 k1) applied after it.
NB_HD void fft_fwd1_t(int n0, const double *x, cplx *sp, const cplx *t1)
{
    cplx y[8];
    y[0] = {x[0], x[8]};
    y[4] = c_mul_w8<true>({x[4], x[12]});
    static_for<1, 8>([&](auto M) {
        constexpr int m = decltype(M)::value;
        if constexpr (m != 4) y[m] = c_mul_conj({x[m], x[m + 8]}, fft_w64(2 * m));
    });
    dft8<false>(y);
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        st_cplx(sp + fft_pass1_x(n0, k), c_mul(y[k], t1[k]));
    });
}
NB_HD void fft_fwd1(int n0, const double *x, cplx *sp, const cplx *tab)
{
    cplx t1[8];
    fft_load_t1(n0, tab, t1);
    fft_fwd1_t(n0, x, sp, t1);
}
// pass 2 (forward): the 16 points 64 k1 + n2 + 4 m of spectrum sp -> DFT16, times W64^(n2 k2)
NB_HD void fft_fwd2(int k1, int n2, cplx *sp)
{
    cplx y[16];
    static_for<0, 16>([&](auto M) { y[decltype(M)::value] = ld_cplx(sp + fft_pass2_x(k1, n2, decltype(M)::value)); });
    dft16<false>(y);
    fft_w64_twiddle<false>(n2, y);
    static_for<0, 16>([&](auto K) { st_cplx(sp + fft_pass2_x(k1, n2, decltype(K)::value), y[decltype(K)::value]); });
}
// pass 3 (forward only, the key spectra): group g of spectrum sp, in place
NB_HD void fft_fwd3(int g, cplx *sp)
{
    cplx y[4];
    static_for<0, 4>([&](auto I) { y[decltype(I)::value] = ld_cplx(sp + fft_pass3_x(g, decltype(I)::value)); });
    dft4<false>(y);
    static_for<0, 4>([&](auto I) { st_cplx(sp + fft_pass3_x(g, decltype(I)::value), y[decltype(I)::value]); });
}
// pass 2 (inverse), mirrored
NB_HD void fft_inv2(int k1, int n2, cplx *sp)
{
    cplx y[16];
    static_for<0, 16>([&](auto M) { y[decltype(M)::value] = ld_cplx(sp + fft_pass2_x(k1, n2, decltype(M)::value)); });
    fft_w64_twiddle<true>(n2, y);
    dft16<true>(y);
    static_for<0, 16>([&](auto M) { st_cplx(sp + fft_pass2_x(k1, n2, decltype(M)::value), y[decltype(M)::value]); });
}
// pass 1 (inverse): x[m'] = the (unrounded) real coefficient n0 + 64 m', m' < 16, of spectrum sp.  Mirrored: conj(T)
// before the inverse DFT8, the constants conj(w^(64 m)) / 512 = W64^(2 m) / 512 after it (the division is exact)
NB_HD void fft_inv1_t(int n0, const cplx *sp, const cplx *t1, double *x)
{
    constexpr double R = 1.0 / 512, S = 0.70710678118654752440 / 512;
    cplx y[8];
    static_for<0, 8>([&](auto K) {
        constexpr int k = decltype(K)::value;
        y[k] = c_mul_conj(ld_cplx(sp + fft_pass1_x(n0, k)), t1[k]);
    });
    dft8<true>(y);
    static_for<0, 8>([&](auto M) {
        constexpr int m = decltype(M)::value;
        cplx v;
        if constexpr (m == 0) v = {d_mul(y[0].re, R), d_mul(y[0].im, R)};
        else if constexpr (m == 4) v = {d_mul(d_add(y[4].re, y[4].im), S), d_mul(d_sub(y[4].im, y[4].re), S)};
        else {
            constexpr cplx w = fft_w64(2 * m);
            v = c_mul(y[m], cplx{w.re * R, w.im * R});
        }
        x[m] = v.re;
        x[m + 8] = v.im;
    });
}
NB_HD void fft_inv1(int n0, const cplx *sp, const cplx *tab, double *x)
{
    cplx t1[8];
    fft_load_t1(n0, tab, t1);
    fft_inv1_t(n0, sp, t1, x);
}

// ---- the FP64 step of a CTA of 2 ciphertexts on 256 threads: spectra fft_spec(ct, s), s = mi * 2 + j before the MAC
// and s = mo * 2 + h after it.
// fwd1: task (pm = ct * 2 + mi, n0): the rotated coefficients serve both digit polynomials (as phase_fwd1_both_digits)
// ROUND: added to every coefficient before the digits are cut.  0 (the bootstrap, as nufhe's decomposition): the
// digits truncate, Dec(x) g = x - (x mod 2^12).  DIGIT_ROUND (index_lookup.cuh): they round to the nearest multiple of
// 2^12, so the approximation error is centred instead of averaging -2^11.
constexpr u32 DIGIT_ROUND = 1u << 11;      // half the precision 2^(32 - l log2 Bg) of the decomposition
template <bool ROTATE, u32 ROUND = 0>
NB_HD void fft_phase_fwd1(int task, const i32 *acc_all, cplx *spec_all, const cplx *tab, const int *rot_a)
{
    const int n0 = task & 63, pm = task >> 6;
    const i32 *acc = acc_all + pm * NTT_N;
    const int a = ROTATE ? rot_a[pm >> 1] : 0;
    const int ar = a & (NTT_N - 1);
    const bool flip = (a >> 10) & 1;
    u32 t[16];
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        const int idx = 64 * j1 + n0;
        const i32 c = ROTATE ? rotate_minus_one(acc, idx, ar, flip) : acc[idx];
        t[j1] = (u32)c + (0x80000000u + (1u << 21) + ROUND);
    });
    cplx t1[8];
    fft_load_t1(n0, tab, t1);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int j = 0; j < 2; j++) {
        const int sh = 22 - 10 * j;
        double x[16];
        static_for<0, 16>([&](auto J) { x[decltype(J)::value] = d_digit((t[decltype(J)::value] >> sh) & 1023u); });
        fft_fwd1_t(n0, x, spec_all + fft_pass1_spec(task, j), t1);
    }
}
// fwd2 / inv2: one 16-point task per thread (fft_pass2_task)
NB_HD void fft_phase_fwd2(int tid, cplx *spec_all)
{
    const FftPass2 t = fft_pass2_task(tid);
    fft_fwd2(t.k1, t.n2, spec_all + fft_spec(t.ct, t.s));
}
NB_HD void fft_phase_inv2(int tid, cplx *spec_all)
{
    const FftPass2 t = fft_pass2_task(tid);
    fft_inv2(t.k1, t.n2, spec_all + fft_spec(t.ct, t.s));
}

// pass 3, fused: group fft_pass3_group(tid / 2) of ciphertext tid & 1 (fft_pass3_pos): the forward DFT4 of the 4 digit spectra, then for each output
// spectrum s = mo * 2 + h the MAC out = sum_d D_d K[d][mo][h] at the 4 points and the inverse DFT4; the outputs
// overwrite the digit spectra at the same positions (the thread holds all of them).
// The key values of two outputs k3 are in flight at any time, one loop iteration ahead of their use: those of outputs
// 0 and 1 of spectrum s are loaded while outputs 2 and 3 of spectrum s - 1 are computed, transformed and stored (the
// first ones before the digit spectra are read), so the L2 latency of the key stream overlaps work instead of
// stalling every output spectrum.  The arithmetic is the same in the same order.
NB_HD void fft_phase_mac(int tid, cplx *spec_all, const cplx *key)
{
#ifdef NB_FFT_KEY_L1_BOUND
    // TIMING EXPERIMENT ONLY (wrong results): every key load hits the same 2 KB of the row -- what the step would take
    // if the key stream cost nothing (DESIGN.md section 4, FP64 step breakdown)
    const int kj = (tid >> 1) & 15;
#else
    const int kj = tid >> 1;
#endif
    // the 4 key values (digits d) of output k3 of spectrum s
    auto load_key = [&](cplx *k, int s, int k3) {
        static_for<0, 4>([&](auto D) { k[decltype(D)::value] = ld_cplx_stream(key + fft_key_pos(4 * decltype(D)::value + s, kj, k3)); });
    };
    cplx ka[4], kb[4];          // even / odd outputs k3
    load_key(ka, 0, 0);
    load_key(kb, 0, 1);
    cplx dg[4][4];
    static_for<0, 4>([&](auto D) {
        static_for<0, 4>([&](auto I) { dg[decltype(D)::value][decltype(I)::value] = ld_cplx(spec_all + fft_pass3_pos(tid, decltype(D)::value, decltype(I)::value)); });
        dft4<false>(dg[decltype(D)::value]);
    });
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int s = 0; s < 4; s++) {
        cplx o[4];
        static_for<0, 4>([&](auto K3) {
            constexpr int k3 = decltype(K3)::value;
            cplx *k = (k3 & 1) ? kb : ka;
            cplx v = {d_mul(dg[0][k3].re, k[0].re), d_mul(dg[0][k3].re, k[0].im)};
            v = {d_fma(-dg[0][k3].im, k[0].im, v.re), d_fma(dg[0][k3].im, k[0].re, v.im)};
            static_for<1, 4>([&](auto D) { v = c_mac(v, dg[decltype(D)::value][k3], k[decltype(D)::value]); });
            o[k3] = v;
            // refill: outputs 2, 3 of this spectrum, then outputs 0, 1 of the next one
            if constexpr (k3 < 2) load_key(k, s, k3 + 2);
            else if (s < 3) load_key(k, s + 1, k3 - 2);
        });
        dft4<true>(o);
        static_for<0, 4>([&](auto I) { st_cplx(spec_all + fft_pass3_pos(tid, s, decltype(I)::value), o[decltype(I)::value]); });
    }
}
// Multi-bit key (DESIGN.md section 14): one step handles the key bits s_2g, s_2g+1 of group g,
//     ACC += sum_{p = 1..3} (X^{k_p} - 1) (Dec(ACC) [x] BK_{g,p}),   k_1 = abar_2g, k_2 = abar_2g+1, k_3 = k_1 + k_2,
// so pass 3 runs the MAC against the 3 key rows of the group and multiplies each row's product by zeta_f^{k_p} - 1 at
// its spectral point.  Bin f = k1 + 8 k2 + 128 k3 of the folded transform evaluates the polynomial at
// zeta_f = e^{2 pi i (1 - 4 f) / 2048}, so zeta_f^k = R[k (1 - 4 k1 - 32 k2) mod 2048] (-i)^(k k3): one table value per
// row and thread, and an exact quarter turn per output k3.
// z (-i)^r, exact (swap and sign)
NB_HD cplx c_quarter_turns(cplx z, int r)
{
    const bool sw = r & 1, neg_re = (r >> 1) & 1, neg_im = ((r >> 1) ^ r) & 1;
    const double x = sw ? z.im : z.re, y = sw ? z.re : z.im;
    return {neg_re ? -x : x, neg_im ? -y : y};
}
// key: the group's 3 key rows (BK_FFT_U64 each, patterns p = 1, 2, 3 in order); rot: the group's two rotation amounts
// of both ciphertexts, [ct][2]
NB_HD void fft_phase_mac_mb(int tid, cplx *spec_all, const cplx *key, const cplx *tab, const int *rot)
{
    const int j = tid >> 1, ct = tid & 1, g = fft_pass3_group(j);
    const int a0 = rot[2 * ct], a1 = rot[2 * ct + 1];
    const int kp[3] = {a0, a1, (a0 + a1) & (2 * NTT_N - 1)};
    const int e0 = 1 - 4 * (g >> 4) - 32 * (g & 15);
    cplx zb[3];
    static_for<0, 3>([&](auto P) {
        constexpr int p = decltype(P)::value;
        zb[p] = ld_cplx_tab(tab + FFT_TAB_ROOTS + ((kp[p] * e0) & (2 * NTT_N - 1)));
    });
    cplx dg[4][4];
    static_for<0, 4>([&](auto D) {
        static_for<0, 4>([&](auto I) { dg[decltype(D)::value][decltype(I)::value] = ld_cplx(spec_all + fft_pass3_pos(tid, decltype(D)::value, decltype(I)::value)); });
        dft4<false>(dg[decltype(D)::value]);
    });
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int s = 0; s < 4; s++) {
        cplx o[4];
        static_for<0, 4>([&](auto K3) {
            constexpr int k3 = decltype(K3)::value;
            static_for<0, 3>([&](auto P) {
                constexpr int p = decltype(P)::value;
                const cplx *kr = key + p * (BK_FFT_U64 / 2);
                cplx k[4];
                static_for<0, 4>([&](auto D) { k[decltype(D)::value] = ld_cplx_stream(kr + fft_key_pos(4 * decltype(D)::value + s, j, k3)); });
                cplx v = {d_mul(dg[0][k3].re, k[0].re), d_mul(dg[0][k3].re, k[0].im)};
                v = {d_fma(-dg[0][k3].im, k[0].im, v.re), d_fma(dg[0][k3].im, k[0].re, v.im)};
                static_for<1, 4>([&](auto D) { v = c_mac(v, dg[decltype(D)::value][k3], k[decltype(D)::value]); });
                // zeta_f^{k_p} - 1: the rounded table value turned exactly, then one rounded subtraction
                cplx f = c_quarter_turns(zb[p], (kp[p] * k3) & 3);
                f.re = d_sub(f.re, 1.0);
                if constexpr (p == 0) o[k3] = c_mul(v, f);
                else o[k3] = c_mac(o[k3], v, f);
            });
        });
        dft4<true>(o);
        static_for<0, 4>([&](auto I) { st_cplx(spec_all + fft_pass3_pos(tid, s, decltype(I)::value), o[decltype(I)::value]); });
    }
}

// inv1: task (pp = ct * 2 + mo, n0): both key halves of output polynomial mo, rounded and recombined mod 2^32.
// ACCUMULATE: acc += result, else acc = result.
template <bool ACCUMULATE> NB_HD void fft_phase_inv1(int task, i32 *acc_all, const cplx *spec_all, const cplx *tab)
{
    const int n0 = task & 63, pp = task >> 6;
    u32 r[16];
    cplx t1[8];
    fft_load_t1(n0, tab, t1);
    {
        double x[16];
        fft_inv1_t(n0, spec_all + fft_pass1_spec(task, 0), t1, x);
        static_for<0, 16>([&](auto J) { r[decltype(J)::value] = (u32)d_rint_lo32(x[decltype(J)::value]); });
    }
    {
        double x[16];
        fft_inv1_t(n0, spec_all + fft_pass1_spec(task, 1), t1, x);
        static_for<0, 16>([&](auto J) { r[decltype(J)::value] += (u32)d_rint_lo32(x[decltype(J)::value]) << 16; });
    }
    i32 *acc = acc_all + pp * NTT_N;
    static_for<0, 16>([&](auto J) {
        constexpr int j1 = decltype(J)::value;
        const int idx = 64 * j1 + n0;
        acc[idx] = ACCUMULATE ? (i32)((u32)acc[idx] + r[j1]) : (i32)r[j1];
    });
}

// key preparation: the 16 real coefficients n0 + 64 m' of one key polynomial (centred integers, |k| <= 2^31) split into
// k_lo in [-2^15, 2^15) and k_hi = (k - k_lo) / 2^16 in [-2^15, 2^15]
NB_HD void fft_split_key(const long long *k, double *lo, double *hi)
{
    for (int m = 0; m < 16; m++) {
        const long long l = ((k[m] + 32768) & 65535) - 32768;
        lo[m] = (double)l;
        hi[m] = (double)((k[m] - l) / 65536);
    }
}

}  // namespace nb
