// host_emul.cpp -- runs the __host__ __device__ pass code of br_phases.cuh / ntt_lane.cuh on the CPU, one
// "thread" after the other, a phase at a time (a phase boundary = a CTA barrier).  Built with g++ into
// libnb_host_emul.so for tests/test_host_logic.py: it lets the CPU-only test suite check the index maps,
// swizzles, twiddle tables and shift constants of the GPU kernels against the oracle.
// This is a test aid for the CUDA source, not a CPU fallback: nothing in nufhe_b200/ loads it.
#include <cstring>
#include <vector>
#include "tables.h"
#include "lut_index.cuh"
#include "chacha.cuh"
#include "plane_gemm.cuh"
#include "pk_layout.cuh"
#include "pack_layout.cuh"
#include "tree_layout.cuh"
#include "compact_layout.cuh"
#include "reencrypt_layout.cuh"
#include "mk_layout.cuh"
#include "mk_expand_layout.cuh"

using namespace nb;

extern "C" {

// The stand-alone transform kernels' passes, one polynomial at a time; in/out natural order, canonical.
void emul_ntt_forward(const u64 *in, u64 *out, size_t batch)
{
    static PhaseTables T;
    std::vector<u64> w(NTT_SWEEP_POLYS * POLY_STRIDE);
    for (size_t b = 0; b < batch; b++) {
        for (int task = 0; task < 64; task++) {
            u64 x[16];
            for (int j1 = 0; j1 < 16; j1++) x[j1] = ff_canon(in[b * NTT_N + 64 * j1 + task]);
            phase_fwd1_generic(task, x, w.data(), T.fwd.data());
        }
        for (int row = 0; row < 16; row++) for (int g = 0; g < 4; g++) phase_fwd2(0, row, g, w.data());
        for (int row = 0; row < 16; row++) for (int u = 0; u < 4; u++) phase_fwd3(0, row, u, w.data());
        for (int k = 0; k < NTT_N; k++) out[b * NTT_N + k] = ff_canon(w[w_position_of_natural(k)]);
    }
}

void emul_ntt_inverse(const u64 *in, u64 *out, size_t batch)
{
    static PhaseTables T;
    std::vector<u64> w(NTT_SWEEP_POLYS * POLY_STRIDE);
    for (size_t b = 0; b < batch; b++) {
        for (int k = 0; k < NTT_N; k++) w[w_position_of_natural(k)] = ff_canon(in[b * NTT_N + k]);
        for (int row = 0; row < 16; row++) for (int u = 0; u < 4; u++) phase_inv3(0, row, u, w.data());
        for (int row = 0; row < 16; row++) for (int g = 0; g < 4; g++) phase_inv2(0, row, g, w.data());
        for (int task = 0; task < 64; task++) {
            u64 y[16];
            phase_inv1_generic(task, y, w.data(), T.inv.data());
            for (int j1 = 0; j1 < 16; j1++) out[b * NTT_N + 64 * j1 + task] = ff_canon(y[j1]);
        }
    }
}

// the same with Torus32 on the natural-order side (i32_conversion): forward reads int32, inverse writes int32
void emul_ntt_forward_i32(const i32 *in, u64 *out, size_t batch)
{
    static PhaseTables T;
    std::vector<u64> w(NTT_SWEEP_POLYS * POLY_STRIDE);
    for (size_t b = 0; b < batch; b++) {
        for (int task = 0; task < 64; task++) {
            i32 x[16];
            for (int j1 = 0; j1 < 16; j1++) x[j1] = in[b * NTT_N + 64 * j1 + task];
            phase_fwd1_i32(task, x, w.data(), T.fwd.data());
        }
        for (int row = 0; row < 16; row++) for (int g = 0; g < 4; g++) phase_fwd2(0, row, g, w.data());
        for (int row = 0; row < 16; row++) for (int u = 0; u < 4; u++) phase_fwd3(0, row, u, w.data());
        for (int k = 0; k < NTT_N; k++) out[b * NTT_N + k] = ff_canon(w[w_position_of_natural(k)]);
    }
}

void emul_ntt_inverse_i32(const u64 *in, i32 *out, size_t batch)
{
    static PhaseTables T;
    std::vector<u64> w(NTT_SWEEP_POLYS * POLY_STRIDE);
    for (size_t b = 0; b < batch; b++) {
        for (int k = 0; k < NTT_N; k++) w[w_position_of_natural(k)] = ff_canon(in[b * NTT_N + k]);
        for (int row = 0; row < 16; row++) for (int u = 0; u < 4; u++) phase_inv3(0, row, u, w.data());
        for (int row = 0; row < 16; row++) for (int g = 0; g < 4; g++) phase_inv2(0, row, g, w.data());
        for (int task = 0; task < 64; task++) {
            i32 y[16];
            phase_inv1_i32(task, y, w.data(), T.inv.data());
            for (int j1 = 0; j1 < 16; j1++) out[b * NTT_N + 64 * j1 + task] = y[j1];
        }
    }
}

// One external-product step of the phase-structured kernel (br_phases.cuh) for up to BR2_CT
// ciphertexts, phases executed in order with all "threads" of a phase run back to back.
// acc: (nct, 2, 1024) in/out; bk_ref_row: reference layout (2,2,2,1024) Montgomery; rot: rotation
// amounts per ciphertext or NULL (plain external product, overwrite).
int emul_phase_ct(void) { return BR2_CT; }

}  // extern "C"

static void prepare_bk_row(const u64 *bk_ref_row, const PhaseTables &T, std::vector<u64> &bk);

template <class Cfg> static void phase_step(i32 *acc_io, const u64 *bk_ref_row, const int *rot, int nct)
{
    static PhaseTables T;
    std::vector<i32> acc(Cfg::CT * 2 * NTT_N, 0);
    std::vector<u64> w(Cfg::POLYS * POLY_STRIDE, 0);
    std::vector<u64> bk(BK_ROW_U64);
    for (int c = 0; c < nct; c++) memcpy(&acc[c * 2 * NTT_N], acc_io + c * 2 * NTT_N, sizeof(i32) * 2 * NTT_N);
    int rots[4] = {0, 0, 0, 0};
    if (rot) for (int c = 0; c < nct; c++) rots[c] = rot[c];
    prepare_bk_row(bk_ref_row, T, bk);
    constexpr int TH = Cfg::THREADS;
    if constexpr (Cfg::SPLIT_FWD) {
        using Tasks = BrCfg<Cfg::CT, 256 * Cfg::CT>;
        auto each = [&](auto fn) { for (int tid = 0; tid < TH; tid++) { int h, t; map_split_fwd<Cfg>(tid, h, t); fn(h, t); } };
        each([&](int h, int t) {
            if (rot) { if (h) phase_fwd1_split<true, 1>(t, acc.data(), w.data(), T.fwd.data(), rots); else phase_fwd1_split<true, 0>(t, acc.data(), w.data(), T.fwd.data(), rots); }
            else { if (h) phase_fwd1_split<false, 1>(t, acc.data(), w.data(), T.fwd.data(), rots); else phase_fwd1_split<false, 0>(t, acc.data(), w.data(), T.fwd.data(), rots); }
        });
        each([&](int h, int t) { int p, r, g; map_fwd2<Tasks>(t, 0, p, r, g); if (h) phase_fwd2_split<1>(p, r, g, w.data()); else phase_fwd2_split<0>(p, r, g, w.data()); });
        {   // in place: every thread holds its 16 inputs in registers across a barrier
            std::vector<u64> held((size_t)TH * 16);
            each([&](int h, int t) { int p, r, u; map_fwd3<Tasks>(t, 0, p, r, u); phase_fwd3_split_load(p, r, u, w.data(), &held[(size_t)(h * 256 * Cfg::CT + t) * 16]); });
            each([&](int h, int t) {
                int p, r, u; map_fwd3<Tasks>(t, 0, p, r, u);
                const u64 *v = &held[(size_t)(h * 256 * Cfg::CT + t) * 16];
                if (h) phase_fwd3_split_finish<1>(p, r, u, w.data(), v); else phase_fwd3_split_finish<0>(p, r, u, w.data(), v);
            });
        }
    } else {
        if constexpr (Cfg::FWD1_BOTH_DIGITS) {
            for (int tid = 0; tid < TH; tid++) {
                if (rot) phase_fwd1_both_digits<true>(tid, acc.data(), w.data(), T.fwd.data(), rots);
                else phase_fwd1_both_digits<false>(tid, acc.data(), w.data(), T.fwd.data(), rots);
            }
        } else {
            for (int it = 0; it < Cfg::FWD_SWEEPS; it++)
                for (int tid = 0; tid < TH; tid++) {
                    if (rot) phase_fwd1<true>(it * TH + tid, acc.data(), w.data(), T.fwd.data(), rots);
                    else phase_fwd1<false>(it * TH + tid, acc.data(), w.data(), T.fwd.data(), rots);
                }
        }
        for (int it = 0; it < Cfg::FWD_SWEEPS; it++)
            for (int tid = 0; tid < TH; tid++) { int p, r, g; map_fwd2<Cfg>(tid, it, p, r, g); phase_fwd2(p, r, g, w.data()); }
        for (int it = 0; it < Cfg::FWD_SWEEPS; it++)
            for (int tid = 0; tid < TH; tid++) { int p, r, u; map_fwd3<Cfg>(tid, it, p, r, u); phase_fwd3(p, r, u, w.data()); }
    }
    for (int tid = 0; tid < TH; tid++) phase_mac<Cfg>(tid, w.data(), bk.data());
    if constexpr (Cfg::SPLIT_INV) {
        // the split inverse phases of the wide shape, one loop per barrier-separated sub-pass (kernels.cuh: br2_step)
        auto each = [&](auto fn) { for (int tid = 0; tid < TH; tid++) { int h, t; if (map_split<Cfg>(tid, h, t)) fn(h, t); } };
        each([&](int h, int t) { int p, r, u; map_inv3<Cfg>(t, p, r, u); if (h) phase_inv3_split_a<1>(p, r, u, w.data()); else phase_inv3_split_a<0>(p, r, u, w.data()); });
        each([&](int h, int t) { int p, r, u; map_inv3<Cfg>(t, p, r, u); if (h) phase_inv3_split_b<1>(p, r, u, w.data()); else phase_inv3_split_b<0>(p, r, u, w.data()); });
        each([&](int h, int t) { int p, r, g; map_inv2_split<Cfg>(t, p, r, g); if (h) phase_inv2_split<1>(p, r, g, w.data()); else phase_inv2_split<0>(p, r, g, w.data()); });
        each([&](int h, int t) { if (h) phase_inv1_split_a<1>(t, w.data(), T.inv.data()); else phase_inv1_split_a<0>(t, w.data(), T.inv.data()); });
        each([&](int h, int t) {
            if (rot) { if (h) phase_inv1_split_b<true, 1>(t, acc.data(), w.data()); else phase_inv1_split_b<true, 0>(t, acc.data(), w.data()); }
            else { if (h) phase_inv1_split_b<false, 1>(t, acc.data(), w.data()); else phase_inv1_split_b<false, 0>(t, acc.data(), w.data()); }
        });
    } else {
        for (int tid = 0; tid < TH; tid++) { int p, r, u; if (map_inv3<Cfg>(tid, p, r, u)) phase_inv3(p, r, u, w.data()); }
        for (int tid = 0; tid < TH; tid++) { int p, r, g; if (map_inv2<Cfg>(tid, p, r, g)) phase_inv2(p, r, g, w.data()); }
        for (int tid = 0; tid < Cfg::INV_TASKS; tid++) {
            if (rot) phase_inv1<true>(tid, acc.data(), w.data(), T.inv.data());
            else phase_inv1<false>(tid, acc.data(), w.data(), T.inv.data());
        }
    }
    for (int c = 0; c < nct; c++) memcpy(acc_io + c * 2 * NTT_N, &acc[c * 2 * NTT_N], sizeof(i32) * 2 * NTT_N);
}

// the engine layout of one reference key row (kernels.cuh: bk_prepare_kernel)
static void prepare_bk_row(const u64 *bk_ref_row, const PhaseTables &T, std::vector<u64> &bk)
{
    bk.assign(BK_ROW_U64, 0);
    for (int pos = 0; pos < NTT_N; pos++) {
        const int k = w_natural_index(pos >> 6, pos & 63);
        u64 sum[2] = {0, 0};
        for (int m = 0; m < 8; m++) {
            u64 x = ff_mul(ff_canon(bk_ref_row[m * NTT_N + k]), FF_RINV);
            bk[m * NTT_N + pos] = x;
            sum[m & 1] = ff_add(sum[m & 1], x);
        }
        for (int mo = 0; mo < 2; mo++) bk[(8 + mo) * NTT_N + pos] = ff_mul(sum[mo], T.ones512[k]);
    }
}

// `steps` consecutive CMux steps of the pair shape (kernels.cuh: blind_rotate_pair_kernel) with the same key row: two
// "CTAs", each with its own work polynomials and accumulator polynomial, every barrier-separated sub-phase run for both
// before the next one starts; the remote stores of the MAC go straight into the other CTA's array.  Several steps in a
// row exercise both parities of the exchange area and what one step leaves behind for the next.
static void pair_steps(i32 *acc_io, const u64 *bk_ref_row, const int *rots, int steps)
{
    static PhaseTables T;
    std::vector<u64> bk;
    prepare_bk_row(bk_ref_row, T, bk);
    std::vector<u64> w[2] = {std::vector<u64>(PAIR_POLYS * POLY_STRIDE, 0x1234567887654321ull), std::vector<u64>(PAIR_POLYS * POLY_STRIDE, 0x0fedcba987654321ull)};
    i32 *acc[2] = {acc_io, acc_io + NTT_N};
    auto both = [&](int threads, auto fn) { for (int rank = 0; rank < 2; rank++) for (int tid = 0; tid < threads; tid++) fn(rank, tid); };
    for (int i = 0; i < steps; i++) {
        const int par = i & 1;
        const int *rot = rots + i;
        both(PAIR_THREADS, [&](int r, int tid) { pair_fwd1(tid, acc[r], w[r].data(), T.fwd.data(), rot); });
        both(PAIR_THREADS, [&](int r, int tid) { pair_fwd2(tid, w[r].data()); });
        std::vector<u64> held((size_t)2 * PAIR_THREADS * 16);
        both(PAIR_THREADS, [&](int r, int tid) { pair_fwd3_load(tid, w[r].data(), &held[((size_t)r * PAIR_THREADS + tid) * 16]); });
        both(PAIR_THREADS, [&](int r, int tid) { pair_fwd3_finish(tid, w[r].data(), &held[((size_t)r * PAIR_THREADS + tid) * 16]); });
        both(PAIR_THREADS, [&](int r, int tid) {
            u64 *peer = w[r ^ 1].data();
            pair_mac<false>(tid, w[r].data(), [peer](int off, u64 x, u64 y) { peer[off] = x; peer[off + 1] = y; },
                            bk.data() + r * 4 * NTT_N, r == 0 ? bk.data() + 8 * NTT_N : nullptr, r, par);
        });
        both(PAIR_THREADS, [&](int r, int tid) { pair_inv3_a(tid, w[r].data(), par); });
        both(PAIR_THREADS, [&](int r, int tid) { pair_inv3_b(tid, w[r].data(), par); });
        both(PAIR_INV_WORKERS, [&](int r, int tid) { pair_inv2(tid, w[r].data(), par); });
        both(PAIR_THREADS, [&](int r, int tid) { pair_inv1_a(tid, w[r].data(), T.inv.data(), par); });
        both(PAIR_THREADS, [&](int r, int tid) { pair_inv1_b(tid, acc[r], w[r].data(), par); });
    }
}

extern "C" {

// the pair shape: `steps` CMux steps with rotation amounts rots[0 .. steps), all with the same key row
void emul_phase_steps_pair(i32 *acc_io, const u64 *bk_ref_row, const int *rots, int steps)
{
    pair_steps(acc_io, bk_ref_row, rots, steps);
}

void emul_phase_step(i32 *acc_io, const u64 *bk_ref_row, const int *rot, int nct)
{
    phase_step<BrDefault>(acc_io, bk_ref_row, rot, nct);
}
// the wide shape (one ciphertext on 256 threads)
void emul_phase_step_wide(i32 *acc_io, const u64 *bk_ref_row, const int *rot)
{
    phase_step<BrWide>(acc_io, bk_ref_row, rot, 1);
}
// the wide2 shape (one ciphertext on 512 threads: split forward and inverse phases)
void emul_phase_step_wide2(i32 *acc_io, const u64 *bk_ref_row, const int *rot)
{
    phase_step<BrWide2>(acc_io, bk_ref_row, rot, 1);
}

// ---- the FP64 step (br_phases.cuh: FP64 step) ----
// key spectra of one polynomial from its centred integer coefficients k[1024], as bk_spectra_kernel computes them:
// spec[h][512] unpadded in the order of fft_key_pos (h = 0: k_lo, 1: k_hi)
static void fft_key_spectra(const long long *k, cplx *spec, const FftTables &F)
{
    std::vector<cplx> w(2 * FFT_SPEC_CPLX);
    for (int n0 = 0; n0 < 64; n0++) {
        long long kk[16];
        double lo[16], hi[16];
        for (int j = 0; j < 16; j++) kk[j] = k[64 * j + n0];
        fft_split_key(kk, lo, hi);
        fft_fwd1(n0, lo, w.data(), F.tab.data());
        fft_fwd1(n0, hi, w.data() + FFT_SPEC_CPLX, F.tab.data());
    }
    for (int h = 0; h < 2; h++) for (int t = 0; t < 32; t++) fft_fwd2(t & 7, t >> 3, w.data() + h * FFT_SPEC_CPLX);
    for (int h = 0; h < 2; h++) for (int g = 0; g < FFT_M / 4; g++) fft_fwd3(g, w.data() + h * FFT_SPEC_CPLX);
    for (int h = 0; h < 2; h++)
        for (int j = 0; j < FFT_M / 4; j++)
            for (int k3 = 0; k3 < 4; k3++) spec[fft_key_pos(h, j, k3)] = w[h * FFT_SPEC_CPLX + fft_pass3_x(fft_pass3_group(j), k3)];
}

// the FP64 part of one engine key row from the reference row (Montgomery, natural order): -1 if a coefficient is not a
// centred 32-bit integer
static int fft_key_row(const u64 *bk_ref_row, std::vector<cplx> &key)
{
    static FftTables F;
    key.assign(BK_FFT_SPECTRA * FFT_M, cplx{0, 0});
    std::vector<u64> plain(NTT_N), coef(NTT_N);
    std::vector<long long> k(NTT_N);
    for (int m = 0; m < 8; m++) {
        for (int i = 0; i < NTT_N; i++) plain[i] = ff_mul(ff_canon(bk_ref_row[m * NTT_N + i]), FF_RINV);
        emul_ntt_inverse(plain.data(), coef.data(), 1);
        for (int i = 0; i < NTT_N; i++) {
            const u64 v = coef[i], half = 1ull << 31;
            if (v < half) k[i] = (long long)v;
            else if (v >= FF_P - half) k[i] = -(long long)(FF_P - v);
            else return -1;
        }
        fft_key_spectra(k.data(), key.data() + m * 2 * FFT_M, F);
    }
    return 0;
}

// The FP64 part of one engine key row (BK_FFT_U64 doubles: 16 spectra of 512 complex values, the layout
// bk_spectra_kernel writes after the NTT planes) from the reference row; -1 if a coefficient is not a centred 32-bit
// integer
int emul_fft_key_row(const u64 *bk_ref_row, double *out)
{
    std::vector<cplx> key;
    if (fft_key_row(bk_ref_row, key)) return -1;
    memcpy(out, key.data(), key.size() * sizeof(cplx));
    return 0;
}

// One CMux step (rot != NULL) or plain external product of the FP64 step for nct <= 2 ciphertexts, phase by phase as
// br_fft_step runs them (BrFft: 256 threads); returns -1 for a key without integral coefficients
int emul_fft_step(i32 *acc_io, const u64 *bk_ref_row, const int *rot, int nct)
{
    static FftTables F;
    using Cfg = BrFft;
    std::vector<cplx> key;
    if (fft_key_row(bk_ref_row, key)) return -1;
    std::vector<i32> acc(Cfg::CT * 2 * NTT_N, 0);
    std::vector<cplx> w(Cfg::POLYS * FFT_SPEC_CPLX, cplx{1e300, -1e300});
    for (int c = 0; c < nct; c++) memcpy(&acc[c * 2 * NTT_N], acc_io + c * 2 * NTT_N, sizeof(i32) * 2 * NTT_N);
    int rots[2] = {0, 0};
    if (rot) for (int c = 0; c < nct; c++) rots[c] = rot[c];
    const cplx *tab = F.tab.data();
    constexpr int TH = Cfg::THREADS;
    for (int tid = 0; tid < TH; tid++) {
        if (rot) fft_phase_fwd1<true>(tid, acc.data(), w.data(), tab, rots); else fft_phase_fwd1<false>(tid, acc.data(), w.data(), tab, rots);
    }
    for (int tid = 0; tid < TH; tid++) fft_phase_fwd2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) fft_phase_mac(tid, w.data(), key.data());
    for (int tid = 0; tid < TH; tid++) fft_phase_inv2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) {
        if (rot) fft_phase_inv1<true>(tid, acc.data(), w.data(), tab); else fft_phase_inv1<false>(tid, acc.data(), w.data(), tab);
    }
    for (int c = 0; c < nct; c++) memcpy(acc_io + c * 2 * NTT_N, &acc[c * 2 * NTT_N], sizeof(i32) * 2 * NTT_N);
    return 0;
}

// The FP64 step of the encrypted-index kernels (index_lookup.cuh: index_fft_step) on 2 ciphertext slots, each with its
// own key row: bk_ref_rows (2, 8, 1024) u64 in the reference's form, slot c reads row c.  rot != NULL: the CMux step
// ACC += row [x] ((X^rot[c] - 1) ACC); else the plain product ACC = row [x] ACC, both with the rounded decomposition of
// the index kernels (DIGIT_ROUND).  acc_io (2, 2, 1024) is updated.
// Returns -1 for a row without integral coefficients.
int emul_fft_step_slots(i32 *acc_io, const u64 *bk_ref_rows, const int *rot)
{
    static FftTables F;
    using Cfg = BrFft;
    std::vector<cplx> key[2];
    for (int c = 0; c < 2; c++)
        if (fft_key_row(bk_ref_rows + (size_t)c * 8 * NTT_N, key[c])) return -1;
    std::vector<cplx> w(Cfg::POLYS * FFT_SPEC_CPLX, cplx{1e300, -1e300});
    int rots[2] = {0, 0};
    if (rot) for (int c = 0; c < 2; c++) rots[c] = rot[c];
    const cplx *tab = F.tab.data();
    constexpr int TH = Cfg::THREADS;
    for (int tid = 0; tid < TH; tid++) {
        if (rot) fft_phase_fwd1<true, DIGIT_ROUND>(tid, acc_io, w.data(), tab, rots);
        else fft_phase_fwd1<false, DIGIT_ROUND>(tid, acc_io, w.data(), tab, rots);
    }
    for (int tid = 0; tid < TH; tid++) fft_phase_fwd2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) fft_phase_mac(tid, w.data(), key[tid & 1].data());     // the slot's own row
    for (int tid = 0; tid < TH; tid++) fft_phase_inv2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) {
        if (rot) fft_phase_inv1<true>(tid, acc_io, w.data(), tab); else fft_phase_inv1<false>(tid, acc_io, w.data(), tab);
    }
    return 0;
}

// One group of the multi-bit step (br_fft_step<true, BrFft, true>) for nct <= 2 ciphertexts, phase by phase: the 3
// reference rows of the group (bk_ref_rows, each 8 x 1024 u64) and rot[c * 2 + b] = abar_{2g + b} of ciphertext c;
// acc_io (nct, 2, 1024) is updated.  Returns -1 for a key without integral coefficients.
int emul_fft_group_mb(i32 *acc_io, const u64 *bk_ref_rows, const int *rot, int nct)
{
    static FftTables F;
    using Cfg = BrFft;
    std::vector<cplx> key(3 * BK_FFT_SPECTRA * FFT_M), row;
    for (int p = 0; p < 3; p++) {
        if (fft_key_row(bk_ref_rows + (size_t)p * 8 * NTT_N, row)) return -1;
        memcpy(key.data() + (size_t)p * BK_FFT_SPECTRA * FFT_M, row.data(), row.size() * sizeof(cplx));
    }
    // the device table: pass-1 table, then the roots at FFT_TAB_ROOTS
    std::vector<cplx> tab(F.tab);
    tab.insert(tab.end(), F.roots.begin(), F.roots.end());
    std::vector<i32> acc(Cfg::CT * 2 * NTT_N, 0);
    std::vector<cplx> w(Cfg::POLYS * FFT_SPEC_CPLX, cplx{1e300, -1e300});
    for (int c = 0; c < nct; c++) memcpy(&acc[c * 2 * NTT_N], acc_io + c * 2 * NTT_N, sizeof(i32) * 2 * NTT_N);
    int rots[4] = {0, 0, 0, 0};
    for (int i = 0; i < 2 * nct; i++) rots[i] = rot[i];
    constexpr int TH = Cfg::THREADS;
    for (int tid = 0; tid < TH; tid++) fft_phase_fwd1<false>(tid, acc.data(), w.data(), tab.data(), rots);
    for (int tid = 0; tid < TH; tid++) fft_phase_fwd2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) fft_phase_mac_mb(tid, w.data(), key.data(), tab.data(), rots);
    for (int tid = 0; tid < TH; tid++) fft_phase_inv2(tid, w.data());
    for (int tid = 0; tid < TH; tid++) fft_phase_inv1<true>(tid, acc.data(), w.data(), tab.data());
    for (int c = 0; c < nct; c++) memcpy(acc_io + c * 2 * NTT_N, &acc[c * 2 * NTT_N], sizeof(i32) * 2 * NTT_N);
    return 0;
}

// The transform chain of the FP64 step on given inputs, for the exactness tests: digit polynomials dig[4][1024] (signed,
// |d| <= 512) and key polynomials key[4][1024] (centred 32-bit); out[h][1024] = the UNROUNDED coefficients of
// sum_d dig_d * key_d,h mod X^1024 + 1 for the key halves h = 0 (lo), 1 (hi), through the same passes and MAC as the
// kernel (one ciphertext, one output polynomial).
void emul_fft_product(const double *dig, const long long *key, double *out)
{
    static FftTables F;
    const cplx *tab = F.tab.data();
    std::vector<cplx> ks(BK_FFT_SPECTRA * FFT_M, cplx{0, 0});
    for (int d = 0; d < 4; d++) fft_key_spectra(key + d * NTT_N, ks.data() + (d * 2 + 0) * 2 * FFT_M, F);   // mo = 0
    std::vector<cplx> w(BrFft::POLYS * FFT_SPEC_CPLX, cplx{0, 0});
    // ciphertext 0 of the CTA: the tasks that belong to it, in the kernel's thread maps
    for (int tid = 0; tid < 128; tid++) {               // fwd1: digit polynomials mi * 2 + 0 / 1, mi = tid / 64
        const int n0 = tid & 63, mi = tid >> 6;
        double xa[16], xb[16];
        for (int j = 0; j < 16; j++) {
            xa[j] = dig[(mi * 2 + 0) * NTT_N + 64 * j + n0];
            xb[j] = dig[(mi * 2 + 1) * NTT_N + 64 * j + n0];
        }
        fft_fwd1(n0, xa, w.data() + fft_pass1_spec(tid, 0), tab);
        fft_fwd1(n0, xb, w.data() + fft_pass1_spec(tid, 1), tab);
    }
    for (int tid = 0; tid < 128; tid++) fft_phase_fwd2(tid, w.data());
    for (int tid = 0; tid < 256; tid += 2) fft_phase_mac(tid, w.data(), ks.data());
    for (int tid = 0; tid < 128; tid++) fft_phase_inv2(tid, w.data());
    for (int n0 = 0; n0 < 64; n0++) {                   // inv1 of output polynomial mo = 0: both key halves
        double xl[16], xh[16];
        fft_inv1(n0, w.data() + fft_pass1_spec(n0, 0), tab, xl);
        fft_inv1(n0, w.data() + fft_pass1_spec(n0, 1), tab, xh);
        for (int j = 0; j < 16; j++) {
            out[0 * NTT_N + 64 * j + n0] = xl[j];
            out[1 * NTT_N + 64 * j + n0] = xh[j];
        }
    }
}

// The multi-bit chain on given inputs, for the exactness tests: digit polynomials dig[4][1024] (signed, |d| <= 512),
// key polynomials key[3][4][1024] (row p = 0, 1, 2 of a group, digit d; centred 32-bit) and the group's rotation
// amounts rot[2] = (abar_2g, abar_2g+1); out[h][1024] = the UNROUNDED coefficients of
// sum_p (X^{k_p} - 1) sum_d dig_d * key_{p,d},h mod X^1024 + 1 for the key halves h = 0 (lo), 1 (hi), through the same
// passes and pass-3 MAC (fft_phase_mac_mb) as the kernel (one ciphertext, one output polynomial).
void emul_fft_product_mb(const double *dig, const long long *key, const int *rot, double *out)
{
    static FftTables F;
    std::vector<cplx> tab(F.tab);
    tab.insert(tab.end(), F.roots.begin(), F.roots.end());
    std::vector<cplx> ks(3 * BK_FFT_SPECTRA * FFT_M, cplx{0, 0});
    for (int p = 0; p < 3; p++)
        for (int d = 0; d < 4; d++)
            fft_key_spectra(key + (p * 4 + d) * NTT_N, ks.data() + (size_t)p * BK_FFT_SPECTRA * FFT_M + (d * 2 + 0) * 2 * FFT_M, F);
    std::vector<cplx> w(BrFft::POLYS * FFT_SPEC_CPLX, cplx{0, 0});
    const int rots[4] = {rot[0], rot[1], 0, 0};
    for (int tid = 0; tid < 128; tid++) {               // fwd1 of ciphertext 0: digit polynomials mi * 2 + 0 / 1
        const int n0 = tid & 63, mi = tid >> 6;
        double xa[16], xb[16];
        for (int j = 0; j < 16; j++) {
            xa[j] = dig[(mi * 2 + 0) * NTT_N + 64 * j + n0];
            xb[j] = dig[(mi * 2 + 1) * NTT_N + 64 * j + n0];
        }
        fft_fwd1(n0, xa, w.data() + fft_pass1_spec(tid, 0), tab.data());
        fft_fwd1(n0, xb, w.data() + fft_pass1_spec(tid, 1), tab.data());
    }
    for (int tid = 0; tid < 128; tid++) fft_phase_fwd2(tid, w.data());
    for (int tid = 0; tid < 256; tid += 2) fft_phase_mac_mb(tid, w.data(), ks.data(), tab.data(), rots);
    for (int tid = 0; tid < 128; tid++) fft_phase_inv2(tid, w.data());
    for (int n0 = 0; n0 < 64; n0++) {
        double xl[16], xh[16];
        fft_inv1(n0, w.data() + fft_pass1_spec(n0, 0), tab.data(), xl);
        fft_inv1(n0, w.data() + fft_pass1_spec(n0, 1), tab.data(), xh);
        for (int j = 0; j < 16; j++) {
            out[0 * NTT_N + 64 * j + n0] = xl[j];
            out[1 * NTT_N + 64 * j + n0] = xh[j];
        }
    }
}

// The shared-memory accesses of the FP64 step (fft_layout.cuh), for the bank-conflict test: the offsets, in 16-byte
// units from the start of the spectra, that thread tid of a BrFft CTA reads or writes in phase `phase` (0: fwd1 / inv1,
// 1: fwd2 / inv2, 2: pass 3), one per warp-instruction, in program order.  Returns the count.
int emul_fft_smem_offsets(int phase, int tid, int *out)
{
    int n = 0;
    if (phase == 0) {
        for (int k = 0; k < 8; k++)
            for (int h = 0; h < 2; h++) out[n++] = fft_pass1_pos(tid, h, k);
    } else if (phase == 1) {
        const FftPass2 t = fft_pass2_task(tid);
        for (int m = 0; m < 16; m++) out[n++] = fft_pass2_pos(t, m);
    } else if (phase == 2) {
        for (int s = 0; s < 4; s++)
            for (int i = 0; i < 4; i++) out[n++] = fft_pass3_pos(tid, s, i);
    }
    return n;
}
// pass 3's key loads: the offset, in complex values from the FP64 part of the row, of key spectrum ks at output k3 of
// the group of thread tid
int emul_fft_key_offset(int tid, int ks, int k3) { return fft_key_pos(ks, tid >> 1, k3); }

// The FP64 step's table as the library uploads it (tables.h: FftTables), FFT_TAB_CPLX complex values, and the index of
// T[k1][n0] in it; returns FFT_TAB_CPLX
int emul_fft_table(double *out)
{
    static FftTables F;
    memcpy(out, F.tab.data(), F.tab.size() * sizeof(cplx));
    return FFT_TAB_CPLX;
}
int emul_fft_tab_t1(int k1, int n0) { return fft_tab_t1(k1, n0); }
// The conversion-free integer <-> double steps of the FP64 step (br_phases.cuh): the digit u - 512 built from the bits
// of 2^52 + u, and round(x) mod 2^32 through the addition of 1.5 2^52
double emul_fft_digit(unsigned u) { return d_digit(u); }
int emul_fft_rint_lo32(double x) { return d_rint_lo32(x); }

// The programmable bootstrap's index functions (lut_index.cuh): the rounded mod-switch, the initial accumulator
// polynomial X^(2N - barb) * tv, and the sample extracted at index j from an accumulator (2, 1024).
int emul_modswitch_lut(i32 x, int log2_outputs) { return modswitch_lut(x, log2_outputs); }

void emul_lut_head(const i32 *tv, int barb, i32 *out)
{
    for (int x = 0; x < NTT_N; x++) out[x] = lut_head_coef(tv, barb, x);
}

void emul_lut_tail(const i32 *acc, int j, i32 *out_a, i32 *out_b)
{
    for (int x = 0; x < NTT_N; x++) out_a[x] = lut_tail_a(acc, j, x);
    *out_b = acc[NTT_N + j];
}

// The ChaCha20 block function of the seeded masks (chacha.cuh): out[16] = block `counter` of the stream (seed[8], nonce)
void emul_chacha_block(const u32 *seed, u64 counter, u64 nonce, u32 *out) { chacha20_block(seed, counter, nonce, out); }

// The byte-plane GEMM (plane_gemm.cuh): plane_prepare_kernel's planes, then plane_gemm_kernel's tile loop for the
// same operand policy, with a scalar model of mma.sync.m16n8k32.row.col.s32.{u8,s8}.u8.s32.  The model places each
// register byte by the fragment layout of the PTX ISA (not by plane_gemm.cuh), so a lane that feeds the wrong bits,
// digits or plane bytes gives a wrong result here.
static void mma_m16n8k32(bool signed_a, const u32 a[32][4], const u32 b[32][2], i32 c[32][4])
{
    i32 A[16][32], B[32][8];
    for (int l = 0; l < 32; l++) {
        const int g = l >> 2, t = l & 3;
        for (int j = 0; j < 16; j++) {          // a_j: register j / 4, byte j % 4
            const int row = g + ((j < 4 || (j >= 8 && j < 12)) ? 0 : 8), k = 4 * t + (j & 3) + (j >= 8 ? 16 : 0);
            const u32 byte = (a[l][j >> 2] >> (8 * (j & 3))) & 0xFF;
            A[row][k] = signed_a ? (i32)(int8_t)byte : (i32)byte;
        }
        for (int j = 0; j < 8; j++) {           // b_j: register j / 4, byte j % 4
            const int k = 4 * t + (j & 3) + (j >= 4 ? 16 : 0);
            B[k][g] = (b[l][j >> 2] >> (8 * (j & 3))) & 0xFF;
        }
    }
    i32 D[16][8] = {};
    for (int r = 0; r < 16; r++) {
        bool any = false;
        for (int k = 0; k < 32; k++) any |= A[r][k] != 0;
        if (!any) continue;                     // (a zero row adds nothing)
        for (int c2 = 0; c2 < 8; c2++) {
            i32 s = 0;
            for (int k = 0; k < 32; k++) s += A[r][k] * B[k][c2];
            D[r][c2] = s;
        }
    }
    for (int l = 0; l < 32; l++) {
        const int g = l >> 2, t = l & 3;
        for (int i = 0; i < 4; i++) c[l][i] += D[g + (i >= 2 ? 8 : 0)][2 * t + (i & 1)];
    }
}

extern "C++" template <class P, class Src>
void emul_plane_gemm(const P &op, const Src &src, u64 rows)
{
    const u32 K = src.K(), cols = src.cols();
    std::vector<uint8_t> planes((size_t)4 * K * cols);
    for (u32 col = 0; col < cols; col++)
        for (u32 k = 0; k < K; k++) {
            const u32 w = src(k, col);
            for (int p = 0; p < 4; p++) planes[plane_offset(p, col, k, K, cols)] = (uint8_t)(w >> (8 * p));
        }
    auto load32 = [&](u64 off) { u32 v; memcpy(&v, planes.data() + off, 4); return v; };
    const u64 plane_stride = plane_offset(1, 0, 0, K, cols);
    constexpr int NT = P::NTILES;
    std::vector<i32> acc((size_t)4 * GEMM_MTILES * NT * 32 * 4);
    auto A = [&](int p, int mt, int nt) {
        return reinterpret_cast<i32 (*)[4]>(&acc[(((size_t)p * GEMM_MTILES + mt) * NT + nt) * 128]);
    };
    for (u64 row0 = 0; row0 < rows; row0 += 16 * GEMM_MTILES)        // one warp
        for (u32 col0 = 0; col0 < cols; col0 += 8 * NT) {               // its CTA's column tiles
            std::fill(acc.begin(), acc.end(), 0);
            for (u32 ks = 0; ks < K >> 5; ks++) {
                u32 bf[NT][4][32][2], af[GEMM_MTILES][32][4];
                for (int l = 0; l < 32; l++) {
                    const int g = l >> 2, t = l & 3;
                    for (int nt = 0; nt < NT; nt++) {
                        const u64 bcol = plane_offset(0, col0 + 8 * nt + g, 0, K, cols);
                        for (int p = 0; p < 4; p++)
                            for (int h = 0; h < 2; h++)
                                bf[nt][p][l][h] = load32(bcol + p * plane_stride + 32 * ks + frag_k(t, h));
                    }
                    for (int mt = 0; mt < GEMM_MTILES; mt++) {
                        const typename P::Word *row[2];
                        bool ok[2];
                        for (int hr = 0; hr < 2; hr++) {
                            const u64 r = row0 + 16 * mt + acc_row(g, 2 * hr);
                            ok[hr] = r < rows;
                            row[hr] = op.row(ok[hr] ? r : 0);
                        }
                        op.a_frag(row, ok, ks, t, af[mt][l]);
                    }
                }
                for (int mt = 0; mt < GEMM_MTILES; mt++)
                    for (int nt = 0; nt < NT; nt++)
                        for (int p = 0; p < 4; p++) mma_m16n8k32(P::SIGNED_A, af[mt], bf[nt][p], A(p, mt, nt));
            }
            for (int l = 0; l < 32; l++) {
                const int g = l >> 2, t = l & 3;
                for (int mt = 0; mt < GEMM_MTILES; mt++)
                    for (int nt = 0; nt < NT; nt++)
                        for (int i = 0; i < 4; i++) {
                            const u64 row = row0 + 16 * mt + acc_row(g, i);
                            if (row >= rows) continue;
                            const u32 col = col0 + 8 * nt + acc_col(t, i);
                            op.store(row, col, combine(A(0, mt, nt)[l][i], A(1, mt, nt)[l][i], A(2, mt, nt)[l][i],
                                                       A(3, mt, nt)[l][i]), A(0, mt, nt)[l][i]);
                        }
            }
        }
}

// Public-key encryption (pk_layout.cuh): nb_pk_prepare, then nb_pk_encrypt.
void emul_pk_encrypt(const u32 *r_bits, const i32 *a, const i32 *b, size_t m, size_t n, const i32 *mus,
                     float row_variance, i32 *out_a, i32 *out_b, float *out_cv, size_t batch)
{
    emul_plane_gemm(PkGemm{r_bits, (u32)m, (u32)n, mus, row_variance, out_a, out_b, out_cv}, PkSource{a, b, (u32)m, (u32)n},
                    batch);
}

// Result packing (pack_layout.cuh): the digits of `count` mask words (out[2 c + j] = digit j of a[c]), the 16-bit mod
// switch and its inverse, and the slot mapping of input c.
void emul_pack_digits(const i32 *a, size_t count, i32 *out)
{
    for (size_t c = 0; c < count; c++)
        for (int j = 0; j < PACK_LEVELS; j++) out[c * PACK_LEVELS + j] = pack_digit(a[c], j);
}
void emul_pack_round16(const u32 *x, size_t count, uint16_t *out) { for (size_t i = 0; i < count; i++) out[i] = pack_round16(x[i]); }
void emul_pack_unround16(const uint16_t *x, size_t count, u32 *out) { for (size_t i = 0; i < count; i++) out[i] = pack_unround16(x[i]); }
void emul_pack_slot(u64 c, u64 *group, u32 *slot) { *group = pack_group(c); *slot = pack_slot(c); }

// Compact public-key encryption (compact_layout.cuh): `count` output coefficients (body / occupied flags as bytes), and
// the extraction of slot p from one group's data (k + 1, N) uint16 -> a (k N,), *b.
void emul_compact_coeff(const u32 *product, const u32 *noise, const uint8_t *body, const uint8_t *occupied,
                        const u32 *mu, size_t count, uint16_t *out)
{
    for (size_t i = 0; i < count; i++) out[i] = compact_coeff(product[i], noise[i], body[i] != 0, occupied[i] != 0, mu[i]);
}
void emul_compact_extract(const uint16_t *data, int k, u32 p, i32 *a, i32 *b)
{
    std::vector<u32> poly(PACK_N);
    for (int u = 0; u < k; u++) {
        for (int i = 0; i < PACK_N; i++) poly[i] = pack_unround16(data[u * PACK_N + i]);
        for (u32 j = 0; j < (u32)PACK_N; j++) a[u * PACK_N + j] = compact_extract(poly.data(), p, j);
    }
    *b = (i32)pack_unround16(data[k * PACK_N + p]);
}

// Re-encryption (reencrypt_layout.cuh): the key's slot of (i, j), the coefficient of -D that holds d_p and its sign,
// the whole polynomial -D (N words) of one mask a (n words), and the output mask (N words) from a product P (N words).
u32 emul_reenc_slot(u32 i, int j) { return reenc_slot(i, j); }
u32 emul_reenc_coeff(u32 p) { return reenc_coeff(p); }
int emul_reenc_negated(u32 p) { return reenc_negated(p) ? 1 : 0; }
void emul_reenc_digits(const i32 *a, u32 n, i32 *out) { for (u32 c = 0; c < (u32)PACK_N; c++) out[c] = reenc_digit_coeff(a, n, c); }
void emul_reenc_mask(const u32 *prod, i32 *out) { for (u32 j = 0; j < (u32)PACK_N; j++) out[j] = reenc_mask_word(prod, j); }

// Tree-based programmable bootstrapping (tree_layout.cuh).  emul_tree_keyswitch: nb_tree_prepare, then
// nb_tree_keyswitch.
void emul_tree_keyswitch(const i32 *a, const i32 *masks, const i32 *body, size_t n, int k, i32 *out, size_t rows)
{
    emul_plane_gemm(TreeGemm{a, (u32)n, (u32)(k + 1) * PACK_N, out}, TreeSource{masks, body, (u32)n, (u32)k}, rows);
}

// Multi-key tables (mk_layout.cuh).  emul_mk_tree_tiles: the tiles of nb_mk_tree_keyswitch (first row, rows, tenant),
// written when the arrays are not null; returns their number.  emul_mk_tree_keyswitch: nb_mk_tree_keyswitch, every tile
// run as tree_gemm_mk_kernel runs it, with its tenant's masks[t] / body[t].  emul_mk_group_tenants: the tenant of every
// group of nb_mk_ntt_mac.
u64 emul_mk_tree_tiles(const size_t *counts, size_t tenants, u64 *row0, u32 *rows, u32 *tenant)
{
    std::vector<TreeTile> tiles(mk_tree_tiles(counts, tenants, nullptr, nullptr));
    mk_tree_tiles(counts, tenants, nullptr, tiles.data());
    for (size_t i = 0; i < tiles.size() && row0; i++) { row0[i] = tiles[i].row0; rows[i] = tiles[i].rows; tenant[i] = tiles[i].tenant; }
    return tiles.size();
}
void emul_mk_tree_keyswitch(const i32 *a, const i32 *const *masks, const i32 *const *body, const size_t *counts,
                            size_t tenants, size_t n, int k, i32 *out)
{
    const u32 cols = (u32)(k + 1) * PACK_N;
    std::vector<TreeTile> tiles(mk_tree_tiles(counts, tenants, nullptr, nullptr));
    mk_tree_tiles(counts, tenants, nullptr, tiles.data());
    for (const TreeTile &t : tiles)
        emul_plane_gemm(TreeGemm{a + t.row0 * n, (u32)n, cols, out + t.row0 * cols},
                        TreeSource{masks[t.tenant], body[t.tenant], (u32)n, (u32)k}, t.rows);
}
u64 emul_mk_group_tenants(const size_t *group_counts, size_t tenants, u32 *out)
{
    std::vector<u32> ids(tenants);
    for (size_t t = 0; t < tenants; t++) ids[t] = (u32)t;
    return mk_group_keys(group_counts, tenants, ids.data(), out);
}

// Expansion of compressed cloud keys (mk_expand_layout.cuh).  emul_mk_bk_mask_word / emul_mk_bk_body_offset: the index
// functions themselves.  emul_mk_bk_mask_regroup: what mk_bk_expand_kernel's 64 threads hold after the regrouping for
// mask polynomial (i, mi, j, mo) (N = 1024): out[n0 * 16 + jj] = the value thread n0 gives bk_spectra_transform as k[jj].
// emul_mk_ks_expand: ks_a (in, t, base, n) as mk_ks_expand_kernel writes it, every stream word and zero row in turn.
u64 emul_mk_bk_mask_word(u64 i, u32 mi, u32 j, u32 mo, u32 k, u32 l, u32 N) { return mk_bk_mask_word(i, mi, j, mo, k, l, N); }
u64 emul_mk_bk_body_offset(u64 i, u32 mi, u32 j, u32 k, u32 l, u32 N) { return mk_bk_body_offset(i, mi, j, k, l, N); }
void emul_mk_bk_mask_regroup(const u32 *seed, u64 i, u32 mi, u32 j, u32 mo, u32 k, u32 l, i32 *out)
{
    std::vector<u32> buf(MK_REGROUP_WORDS);
    for (int n0 = 0; n0 < 64; n0++) {
        u32 x[16];
        chacha20_block(seed, (mk_bk_mask_word(i, mi, j, mo, k, l, NTT_N) >> 4) + n0, MK_NONCE_BK, x);
        for (int w = 0; w < 16; w++) buf[mk_regroup_slot(16 * n0 + w)] = x[w];
    }
    for (int n0 = 0; n0 < 64; n0++)
        for (int jj = 0; jj < 16; jj++) out[n0 * 16 + jj] = (i32)buf[mk_regroup_slot(mk_spectra_coef(n0, jj))];
}
void emul_mk_ks_expand(const u32 *seed, size_t in_size, int t, int log2_base, size_t n, i32 *ks_a)
{
    const u32 base = 1u << log2_base;
    const u64 rows = (u64)in_size * t, words = rows * (base - 1) * n;
    for (u64 b = 0; b < (words + 15) / 16; b++) {
        u32 x[16];
        chacha20_block(seed, b, MK_NONCE_KS, x);
        for (int w = 0; w < 16 && b * 16 + w < words; w++) ks_a[mk_ks_a_word(b * 16 + w, n, base)] = (i32)x[w];
    }
    for (u64 r = 0; r < rows; r++)
        for (u64 c = 0; c < n; c++) ks_a[mk_ks_zero_word(r, c, n, base)] = 0;
}

// emul_tree_assemble: tree_assemble_kernel's arithmetic, one (test vector, polynomial) after the other, with a serial
// prefix sum
void emul_tree_assemble(const i32 *v, const i32 *b, int bits, int k, i32 *tv, size_t count)
{
    const int M = 1 << bits;
    std::vector<u32> z(PACK_N), ps(PACK_N + 1);
    for (size_t t = 0; t < count; t++)
        for (int u = 0; u <= k; u++) {
            for (int x = 0; x < PACK_N; x++) {
                u32 s = 0;
                for (int m = 0; m < M; m++) {
                    bool neg;
                    const int d = tree_shift_index(tree_offset(m, bits), x, &neg);
                    const u32 gv = tree_glwe_coef(v + ((t * M + m) * (k + 1) + u) * PACK_N, b[t * M + m], u == k, d);
                    s += neg ? 0u - gv : gv;
                }
                z[x] = s;
            }
            ps[0] = 0;
            for (int x = 0; x < PACK_N; x++) ps[x + 1] = ps[x] + z[x];
            for (int x = 0; x < PACK_N; x++) tv[(t * (k + 1) + u) * PACK_N + x] = (i32)tree_window_coef(ps.data(), PACK_N >> bits, x);
        }
}

void emul_ff_shl_var(const u64 *in, const int *s, u64 *out, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_shl_var(in[i], s[i]); }
void emul_ff_mul(const u64 *a, const u64 *b, u64 *out, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_mul(a[i], b[i]); }
void emul_ff_add(const u64 *a, const u64 *b, u64 *out, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_add(a[i], b[i]); }
void emul_ff_sub(const u64 *a, const u64 *b, u64 *out, size_t n)
{ for (size_t i = 0; i < n; i++) out[i] = ff_sub(a[i], b[i]); }

}  // extern "C"
