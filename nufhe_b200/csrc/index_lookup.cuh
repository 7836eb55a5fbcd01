// index_lookup.cuh -- encrypted-index table lookups on the FP64 CMux step (DESIGN.md section 15).
//
// A query is m TGSW selectors C_j (client-encrypted index bits) whose FP64 spectra (BK_FFT_U64 words per bit, the
// layout bk_spectra_kernel writes) are prepared per query.  Two kernels share the FP64 step of the fused bootstrap
// (br_phases.cuh: fwd1, fwd2, pass-3 MAC, inv2, inv1) in its throughput shape, a CTA of two ciphertext slots on 256
// threads.  Unlike the bootstrap, each slot reads the key row of its own query: fft_phase_mac serves slot tid & 1 from
// the pointer its thread passes, so both slots share a row only when they belong to the same query.
//   * CMux level: out[q][i] = in[q][2i] + C_j(q) [x] (in[q][2i+1] - in[q][2i]), one node per slot.
//   * rotation + extraction: ACC <- ACC + C_j(q) [x] ((X^(-2^j) - 1) ACC) for j < min(m, 10), then sample extraction
//     at coefficients w 2^m (m < 10) or 0 (m >= 10).
// With INDIRECT, the level that first reads a table takes one table per query (the multi-key machine's per-tenant
// encrypted tables, DESIGN.md section 20): query q reads its input at table_id[q] in_stride words from `in` instead of
// q in_stride.  Every other level and the existing instantiations read as before.
// Both round the gadget decomposition (fwd1 with ROUND = DIGIT_ROUND = 2^11) where the bootstrap truncates.  With
// truncated digits every CMux whose selector bit is 1 shifts the phase by about -2^11 (1 + HW(S)) in 32-bit units,
// -2.4e-4 of the torus, and those shifts add up coherently along a lookup's m CMuxes (DESIGN.md section 15).
#pragma once

namespace nb {

// int32 selector coefficients -> field elements (the input of bk_spectra_kernel, which recentres them)
__global__ void index_i32_to_field_kernel(const i32 *__restrict__ in, u64 *__restrict__ out, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const i32 x = in[i];
        out[i] = x < 0 ? FF_P - (u64)(-(long long)x) : (u64)x;
    }
}

struct IndexArgs {
    const i32 *in;          // CMux: input nodes (2 per output node), rotation: accumulators; (2, N) int32 each
    size_t in_stride;       // int32 words between queries (0: every query reads the same inputs, a plaintext level)
    const u64 *sel;         // spectra of the selector used (CMux) or of bit 0 (rotation) of query 0
    size_t sel_stride;      // u64 words between queries
    const cplx *fft_tab;
    i32 *out;               // CMux: (queries, nodes, 2, N)
    i32 *out_a, *out_b;     // rotation: (columns, queries, N) and (columns, queries)
    size_t nodes;           // CMux: output nodes per query; rotation: accumulators per query
    size_t queries;
    size_t items;           // queries * nodes
    int steps;              // rotation: min(m, 10)
    int log2_stride;        // rotation: m, the distance between extracted coefficients
    int samples;            // rotation: samples extracted per accumulator
    const u32 *table_id;    // INDIRECT: the table of each query, in_stride words apart from `in`
};

// the int32 words from p.in to the inputs of query q
template <bool INDIRECT>
NB_D size_t index_query_offset(const IndexArgs &p, size_t q)
{
    if constexpr (INDIRECT) return (size_t)p.table_id[q] * p.in_stride;
    else return q * p.in_stride;
}

// the FP64 step (as br_fft_step) with a per-thread key row: the spectra of the selector of the slot this thread's
// pass-3 task belongs to
template <bool ROTATE>
NB_D void index_fft_step(const Br2Smem &s, const cplx *__restrict__ key, const int *rot, const cplx *__restrict__ tab)
{
    cplx *spec = reinterpret_cast<cplx *>(s.w);
    int tid = fft_step_tid();
    fft_phase_fwd1<ROTATE, DIGIT_ROUND>(tid, s.acc, spec, tab, rot);
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_fwd2(tid, spec);
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_mac(tid, spec, key);
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_inv2(tid, spec);
    __syncthreads();
    tid = fft_step_tid();
    fft_phase_inv1<ROTATE>(tid, s.acc, spec, tab);
}

// One CTA per two items (item = q * nodes + i); a slot beyond the batch replays the last item and stores nothing.
template <bool ROTATE, bool INDIRECT = false>
__global__ void __launch_bounds__(BrFft::THREADS, BrFft::CTAS_PER_SM) index_lookup_kernel(IndexArgs p)
{
    using Cfg = BrFft;
    constexpr int ACC_WORDS = Cfg::CT * 2 * NTT_N;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Br2Smem s = br2_carve<Cfg>(smem_raw);
    const int tid = threadIdx.x;
    const size_t item0 = (size_t)blockIdx.x * Cfg::CT;
    auto item_of = [&](int slot) { const size_t i = item0 + slot; return i < p.items ? i : p.items - 1; };
    const size_t my_item = item_of(tid & 1);            // the slot of this thread's pass-3 task
    const cplx *key = reinterpret_cast<const cplx *>(p.sel + (my_item / p.nodes) * p.sel_stride);

    if constexpr (!ROTATE) {
        // the difference of the node pair
        for (int e = tid; e < ACC_WORDS; e += Cfg::THREADS) {
            const size_t it = item_of(e >> 11), q = it / p.nodes, i = it - q * p.nodes;
            const i32 *d0 = p.in + index_query_offset<INDIRECT>(p, q) + 2 * i * 2 * NTT_N;
            const int x = e & (2 * NTT_N - 1);
            s.acc[e] = (i32)((u32)d0[2 * NTT_N + x] - (u32)d0[x]);
        }
        __syncthreads();
        index_fft_step<false>(s, key, s.rot, p.fft_tab);
        __syncthreads();
        for (int e = tid; e < ACC_WORDS; e += Cfg::THREADS) {
            const size_t it = item0 + (e >> 11);
            if (it >= p.items) continue;
            const size_t q = it / p.nodes, i = it - q * p.nodes;
            const i32 *d0 = p.in + index_query_offset<INDIRECT>(p, q) + 2 * i * 2 * NTT_N;
            const int x = e & (2 * NTT_N - 1);
            p.out[it * 2 * NTT_N + x] = (i32)((u32)s.acc[e] + (u32)d0[x]);
        }
    } else {
        for (int e = tid; e < ACC_WORDS; e += Cfg::THREADS) {
            const size_t it = item_of(e >> 11), q = it / p.nodes, c = it - q * p.nodes;
            s.acc[e] = p.in[index_query_offset<INDIRECT>(p, q) + c * 2 * NTT_N + (e & (2 * NTT_N - 1))];
        }
        for (int j = 0; j < p.steps; j++) {
            if (tid < Cfg::CT) s.rot[tid] = 2 * NTT_N - (1 << j);
            __syncthreads();
            index_fft_step<true>(s, key + (size_t)j * (BK_FFT_U64 / 2), s.rot, p.fft_tab);
            __syncthreads();
        }
        // sample extraction at coefficient pos: a_x = A[pos - x] for x <= pos, -A[N + pos - x] otherwise; b = B[pos]
        const int E = p.samples;
        for (int e = tid; e < Cfg::CT * E * NTT_N; e += Cfg::THREADS) {
            const int slot = e / (E * NTT_N), r = e - slot * E * NTT_N, w_in = r >> 10, x = r & (NTT_N - 1);
            const size_t it = item0 + slot;
            if (it >= p.items) continue;
            const size_t q = it / p.nodes, c = it - q * p.nodes;
            const size_t row = (c * E + w_in) * p.queries + q;
            const int pos = w_in << p.log2_stride;
            const i32 *a0 = s.acc + slot * 2 * NTT_N;
            p.out_a[row * NTT_N + x] = x <= pos ? a0[pos - x] : (i32)(0u - (u32)a0[NTT_N + pos - x]);
            if (x == 0) p.out_b[row] = a0[NTT_N + pos];
        }
    }
}

}  // namespace nb
