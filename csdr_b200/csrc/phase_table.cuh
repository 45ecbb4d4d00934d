// phase_table.cuh -- the reference's phase wrap as a table lookup, for chains that advance a float phase by the SAME increment every step.
//
// Every NCO block of the reference carries a float phase from call to call:   ph += rate*PI*n;  while (ph > PI) ph -= 2*PI;  ...
// (libcsdr_gpl.c:48-50, :154-157; libcsdr.c:300-304).  The subtractions round, so the chain ph[k+1] = wrap(fl(ph[k] + inc)) has to be
// replayed step by step; wrap_phase_pm_pi (common.cuh) does one step bit-exactly in about a thousand dependent cycles (nine binade levels),
// and with a few thousand steps per block that serial chain -- not the data path -- sets the pace of the shift bank, of the fused DDC
// bank's pre-pass and of the fastddc inverse bank.
//
// Observation.  With inc fixed, x = fl(ph + inc) only ever lies in [|inc| - pi, |inc| + pi].  Over such a window the loop is a piecewise
// translation:  wrap16(a) = a - K(a)  with K a step function of a few dozen pieces, where wrap16 runs the loop until the value drops below
// 16.  Why: in units of 2^-21 the float 2*pi is the odd integer C = 0xC90FDB; a subtraction whose exact result lands in binade j
// (values [2^j, 2^(j+1)), grid 2^(j-23)) returns  v - R_j,  R_j = C rounded to that grid (never a tie for j >= 4; for j = 3 the minuend
// comes from binade 4, is 0 mod 4, and the tie always resolves to C + 1).  So K(a) is a sum of R_j's whose multiplicities change only where
// some intermediate value crosses a binade boundary or the in-binade step count changes: about two breakpoints per binade level.  Below
// 16 the remaining <= 3 subtractions are done in plain float arithmetic, exactly like the reference.
//
// wrap_table_build() finds the pieces by pushing the window through the levels as integer intervals (exact, no floating point);
// wrap_after_add() is then: count thresholds <= a (independent compares), one double subtraction (exact: all values are multiples of 2^-21
// below 2^32), the float tail loop.  ~150-200 cycles per step instead of ~1 200.  A window that needs more pieces than the table holds, or
// a value outside the window (the caller's first phase may be anything), takes wrap_phase_pm_pi -- the table is an accelerator, never a
// different answer.  Checked against the plain loop for every float in the window, for thousands of increments, on the CPU tier
// (tests/test_phase_table_host.py), and on the GPU (tests/test_gpu_round2.py::test_long_phase_chains_are_bit_exact).
#pragma once
#include "common.cuh"

namespace csdrb {

constexpr int kWrapPieces = 48;

struct WrapTable {
    float lo, hi;                       // |x| window covered (inclusive); n == 0: no table, every step goes through wrap_phase_pm_pi
    int n, pad;
    float thr[kWrapPieces];             // thr[0] == lo, ascending; piece i = [thr[i], thr[i+1])
    double K[kWrapPieces];              // what the loop subtracts in total before the value falls below 16
};

// A chain of more than this many steps runs on its increment's wrap table (building one costs about as much as thirty direct steps).
// The scratch-size functions reserve table space on the same condition.
constexpr int kWrapTableMinSteps = 96;

constexpr long long kWrapC = 0xC90FDBLL;                    // the float 2*pi in units of 2^-21
constexpr long long kWrapV16 = 16LL << 21;

// 2*pi rounded to the float grid of binade j (j >= 3), in units of 2^-21
__host__ __device__ inline long long wrap_rounded_two_pi(int j)
{
    if (j == 3) return kWrapC + 1;                          // tie -> even; holds for minuends on the binade-4 grid (multiples of 2^-19)
    const int sh = j - 2;
    return ((kWrapC + (1LL << (sh - 1))) >> sh) << sh;
}

__host__ __device__ inline int wrap_ilog2(long long v)     // floor(log2(v)), v > 0
{
#if defined(__CUDA_ARCH__)
    return 63 - __clzll(v);
#else
    return 63 - __builtin_clzll((unsigned long long)v);
#endif
}

// smallest float >= v * 2^-21 (v > 0)
__host__ __device__ inline float wrap_float_ceil(long long v)
{
    const double d = (double)v * (1.0 / 2097152.0);         // exact: v < 2^53
    float f = (float)d;                                     // round to nearest
    if ((double)f < d) {                                    // next float up (positive, finite)
        unsigned u; memcpy(&u, &f, 4); u += 1u; memcpy(&f, &u, 4);
    }
    return f;
}

// Table for the chain  ph <- wrap(fl(ph + inc)),  ph in [-pi, pi].
__host__ __device__ inline void wrap_table_build(float inc, WrapTable* t)
{
    t->n = 0; t->pad = 0; t->lo = 0.f; t->hi = 0.f;
    const float ainc = inc < 0.f ? -inc : inc;
    if (!(ainc < 1048576.f)) return;                        // 2^20 and beyond (or nan): rare, no table
    const float hi_f = ainc + 4.5f;                         // pi, the rounding of the sum, and slack
    float lo_f = ainc - 4.5f;
    if (hi_f < 16.f) return;                                // the whole window is below 16: the tail loop is all there is
    if (lo_f < 16.f) lo_f = 16.f;
    const long long LO = (long long)((double)lo_f * 2097152.0), HI = (long long)((double)hi_f * 2097152.0);
    struct Iv { long long lo, hi, K; };
    constexpr int CAP = 96;
    Iv stack[CAP]; int sp = 0;
    Iv fin[CAP]; int nf = 0;
    stack[sp++] = Iv{LO, HI, 0};
    while (sp > 0) {
        Iv it = stack[--sp];
        long long vlo = it.lo - it.K;
        const long long vhi = it.hi - it.K;
        if (vhi < kWrapV16) { if (nf == CAP) return; fin[nf++] = it; continue; }
        if (vlo < kWrapV16) {                               // the part that is already below 16 is final
            if (nf == CAP) return;
            fin[nf++] = Iv{it.lo, it.K + kWrapV16 - 1, it.K};
            it.lo = it.K + kWrapV16; vlo = kWrapV16;
        }
        const int j = wrap_ilog2(vhi) - 21;                 // binade of the top of the interval (>= 4)
        const long long Bj = 1LL << (j + 21);
        if (vlo < Bj) {                                     // spans two binades: the lower part waits its turn
            if (sp == CAP) return;
            stack[sp++] = Iv{it.lo, it.K + Bj - 1, it.K};
            it.lo = it.K + Bj; vlo = Bj;
        }
        // whole interval in binade j: m in-binade subtractions of R_j while the exact difference stays >= 2^j, then the crossing one
        const long long Rj = wrap_rounded_two_pi(j), Rm = wrap_rounded_two_pi(j - 1), base = kWrapC + Bj;
        const long long m_lo = vlo >= base ? (vlo - base) / Rj + 1 : 0, m_hi = vhi >= base ? (vhi - base) / Rj + 1 : 0;
        for (long long m = m_lo; m <= m_hi; m++) {
            long long s_lo = m == 0 ? vlo : base + (m - 1) * Rj, s_hi = (m == 0 ? base : base + m * Rj) - 1;
            if (s_lo < vlo) s_lo = vlo;
            if (s_hi > vhi) s_hi = vhi;
            if (s_lo > s_hi) continue;
            if (sp == CAP) return;
            stack[sp++] = Iv{s_lo + it.K, s_hi + it.K, it.K + m * Rj + Rm};
        }
    }
    // sort by lo (insertion sort: a few dozen entries), merge equal neighbours
    for (int i = 1; i < nf; i++) {
        const Iv v = fin[i]; int k = i - 1;
        while (k >= 0 && fin[k].lo > v.lo) { fin[k + 1] = fin[k]; k--; }
        fin[k + 1] = v;
    }
    int np = 0;
    for (int i = 0; i < nf; i++) {
        if (np > 0 && fin[np - 1].K == fin[i].K) { fin[np - 1].hi = fin[i].hi; continue; }
        fin[np++] = fin[i];
    }
    if (np > kWrapPieces) return;
    for (int i = 0; i < np; i++) {
        t->thr[i] = i == 0 ? lo_f : wrap_float_ceil(fin[i].lo);
        t->K[i] = (double)fin[i].K * (1.0 / 2097152.0);
    }
    for (int i = np; i < kWrapPieces; i++) { const unsigned inf = 0x7f800000u; memcpy(&t->thr[i], &inf, 4); t->K[i] = 0.0; }
    t->lo = lo_f; t->hi = hi_f; t->n = np;
}

// wrap_phase_pm_pi(x) for x = fl(ph + inc) of the chain the table was built for (any other x still gets the right answer, slowly)
__device__ __forceinline__ float wrap_after_add(float x, const WrapTable* __restrict__ t)
{
    float a = fabsf(x);
    if (a >= 16.f) {
        const int n = t->n;
        if (n == 0 || !(a >= t->lo && a <= t->hi)) return wrap_phase_pm_pi(x);
        int cnt = 0;
#pragma unroll 4
        for (int i = 0; i < n; i++) cnt += a >= t->thr[i] ? 1 : 0;
        a = (float)((double)a - t->K[cnt - 1]);             // exact; the result is the float the loop would hold at this point
    }
    while (a > kPiF) a = __fsub_rn(a, kTwoPiF);
    return (__float_as_uint(x) >> 31) ? -a : a;
}


#if defined(__CUDACC__) || defined(CSDRB_HOST_EMULATION)
// ---- one warp per chain: the table lives in registers, a step is two votes and a shuffle ------------------------------------------------
// Thread-per-channel lookups read 32 different tables per load instruction (32 L1 wavefronts each).  With a
// whole warp on ONE chain every lane keeps two thresholds and their K's, the piece index is popc(ballot(a >= thr)), K comes by shuffle:
// no memory traffic at all inside the chain.  All 32 lanes pass the same x and get the same result.
struct WrapLanes { float thr0, thr1, lo, hi; double K0, K1; int n; };

__device__ __forceinline__ WrapLanes wrap_lanes_load(const WrapTable* __restrict__ t, int lane)
{
    static_assert(kWrapPieces <= 64, "two pieces per lane");
    WrapLanes w;
    w.n = t->n; w.lo = t->lo; w.hi = t->hi;
    const unsigned inf = 0x7f800000u;
    w.thr0 = lane < w.n ? t->thr[lane] : __uint_as_float(inf);
    w.K0 = lane < w.n ? t->K[lane] : 0.0;
    w.thr1 = lane + 32 < w.n ? t->thr[lane + 32] : __uint_as_float(inf);
    w.K1 = lane + 32 < w.n ? t->K[lane + 32] : 0.0;
    return w;
}

// Generic form: any table size, values outside the table's window (falls back to the exact loop fast-forward).
static __device__ __noinline__ float wrap_after_add_warp_generic(float x, const WrapLanes& w)
{
    float a = fabsf(x);
    if (a >= 16.f) {                                                    // every branch here is warp-uniform (same x, same table in all lanes)
        if (w.n == 0 || !(a >= w.lo && a <= w.hi)) return wrap_phase_pm_pi(x);
        int idx = __popc(__ballot_sync(0xffffffffu, a >= w.thr0)) - 1;
        double K = __shfl_sync(0xffffffffu, w.K0, idx & 31);
        if (w.n > 32) {
            const int more = __popc(__ballot_sync(0xffffffffu, a >= w.thr1));
            const double K1 = __shfl_sync(0xffffffffu, w.K1, (more - 1) & 31);
            if (more > 0) K = K1;
        }
        a = (float)((double)a - K);                                     // exact; the float the loop would hold when it first drops below 16
    }
    while (a > kPiF) a = __fsub_rn(a, kTwoPiF);
    return (__float_as_uint(x) >> 31) ? -a : a;
}

// The chain kernels' step.  A chain is pure latency, and a looped step has seven branches (>= 16? in the window? more than 32 pieces?
// the wrap loop's three iterations ...); here the common case -- the value inside the table's window or already below 16 -- is
// straight-line code: two votes, popc, shuffles, one double subtraction, three predicated subtractions (below 16 at most three are left:
// 16 - 3*2pi < pi).  Same operations in the same order as the generic form, which takes everything else.
__device__ __forceinline__ float wrap_after_add_warp(float x, const WrapLanes& w)
{
    const float a = fabsf(x);
    const bool below = a < 16.f;
    const bool in = !below && w.n > 0 && a >= w.lo && a <= w.hi;
    if (!(below || in)) return wrap_after_add_warp_generic(x, w);       // outside the table's window: warp-uniform (same x, same table in all lanes), rare
    // pieces 0..31 sit in thr0/K0, pieces 32.. in thr1/K1 (+inf beyond the table, so `more` is 0 for a table of at most 32 pieces): both look-ups, one select
    const int idx = __popc(__ballot_sync(0xffffffffu, a >= w.thr0)) - 1;
    const int more = __popc(__ballot_sync(0xffffffffu, a >= w.thr1));
    const double K0 = __shfl_sync(0xffffffffu, w.K0, idx & 31), K1 = __shfl_sync(0xffffffffu, w.K1, (more - 1) & 31);
    const double K = more > 0 ? K1 : K0;
    float r = in ? (float)((double)a - K) : a;                          // exact; the float the loop would hold when it first drops below 16
    r = r > kPiF ? __fsub_rn(r, kTwoPiF) : r;
    r = r > kPiF ? __fsub_rn(r, kTwoPiF) : r;
    r = r > kPiF ? __fsub_rn(r, kTwoPiF) : r;
    return (__float_as_uint(x) >> 31) ? -r : r;
}

struct NoChainSink { __device__ void operator()(int, float) const {} };

// One warp walks `steps` steps of the chain ph <- wrap(fl(ph + inc)) from `ph` and returns the phase after them.  All 32 lanes pass the same
// arguments and get the same phases.  A step goes through the wrap table `w`, or through wrap_phase_pm_pi without one (the same answer).
// Before step k, `sink(k, ph)` runs in every lane and, given a `row`, ph goes to row[k]: lane i holds the phase of step i mod 32 and the warp
// stores 32 of them at a time.  The walk starts with a __syncwarp: every lane has read the carried state it passed in before the caller's
// lane 0 overwrites it.  (Several chains per warp do not interleave -- the wrap's branches and votes keep them in program order -- so a
// warp walks one chain.)  Pass `w` as the address of a local or as nullptr, not as a pointer chosen at run time: the compiler then drops
// the other step from the loop and keeps the table in registers (chosen at run time, the table goes to local memory and every step waits on it).
template <class Sink = NoChainSink>
__device__ __forceinline__ float chain_walk_warp(float ph, float inc, const WrapLanes* w, int steps, float* __restrict__ row, Sink sink = {})
{
    const int lane = threadIdx.x & 31;
    float mine = 0.f;
    __syncwarp();
    for (int k = 0; k < steps; k++) {
        sink(k, ph);
        if (row) {
            if ((k & 31) == lane) mine = ph;
            if (((k & 31) == 31 || k == steps - 1) && (k & ~31) + lane <= k) row[(k & ~31) + lane] = mine;
        }
        ph = w ? wrap_after_add_warp(__fadd_rn(ph, inc), *w) : phase_step(ph, inc);
    }
    return ph;
}

#endif  // device (or emulated device) code

// CTAs of a chain kernel with `warps` chains (one warp each) per CTA; every caller states its own `warps` at the launch
inline unsigned chain_ctas(int channels, int warps) { return (unsigned)((channels + warps - 1) / warps); }

}  // namespace csdrb
