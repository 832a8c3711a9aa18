// EXPERIMENT (not part of libnmsm.so; measured by tools/gpu/micro/tail_ops.cu): none of these beat mont_mul for a
// lone warp.
// Latency-oriented Montgomery multiplication variants (experiments for the single-warp tails: Horner, reduce2/3, folds).
// mont_mul (field.cuh) is tuned for THROUGHPUT: two interleaved carry chains saturate the multiply pipe once >= 2 warps share
// an SM sub-partition, but a lone warp pays the ~13-cycle carry-to-carry latency of IMAD.WIDE.X on every link
// The variants here expose more independent work.
#pragma once
#include "field.cuh"

namespace nmsm {

// V3: plain 64-bit C arithmetic, no PTX condition codes: every partial product is  t = a[j]*b[i] + T[j] + carry  (never
// overflows 64 bits), so the only ordering the compiler must respect is true data dependence and it is free to overlap rows.
template <class C>
NMSM_HD void mont_mul_c64(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = C::N;
  uint32_t T[N + 2];
#pragma unroll
  for (int k = 0; k < N + 2; k++) T[k] = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < N; j++) {
      const uint64_t t = (uint64_t)a[j] * b[i] + T[j] + carry;
      T[j] = (uint32_t)t;
      carry = t >> 32;
    }
    uint64_t t = (uint64_t)T[N] + carry;
    T[N] = (uint32_t)t;
    T[N + 1] = (uint32_t)(t >> 32);
    const uint32_t m = T[0] * C::INV;
    carry = ((uint64_t)m * C::P(0) + T[0]) >> 32;
#pragma unroll
    for (int j = 1; j < N; j++) {
      const uint64_t u = (uint64_t)m * C::P(j) + T[j] + carry;
      T[j - 1] = (uint32_t)u;
      carry = u >> 32;
    }
    t = (uint64_t)T[N] + carry;
    T[N - 1] = (uint32_t)t;
    T[N] = T[N + 1] + (uint32_t)(t >> 32);
  }
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = T[k];
  reduce_once<C>(r, T[N]);
}

// V1: separated operand scanning.  Phase A forms the full 2N-limb product with rows that do not depend on any Montgomery
// quotient digit (so consecutive rows can overlap), phase B runs the N reduction rows.  64-bit C arithmetic as above.
template <class C>
NMSM_HD void mont_mul_sos(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = C::N;
  uint32_t T[2 * N + 1];
#pragma unroll
  for (int k = 0; k < 2 * N + 1; k++) T[k] = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < N; j++) {
      const uint64_t t = (uint64_t)a[j] * b[i] + T[i + j] + carry;
      T[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    T[i + N] = (uint32_t)carry;
  }
  uint32_t top = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    const uint32_t m = T[i] * C::INV;
    uint64_t carry = 0;
#pragma unroll
    for (int j = 0; j < N; j++) {
      const uint64_t t = (uint64_t)m * C::P(j) + T[i + j] + carry;
      T[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    // propagate into limb i+N (and one further): the running top carry
    const uint64_t t = (uint64_t)T[i + N] + carry + top;
    T[i + N] = (uint32_t)t;
    top = (uint32_t)(t >> 32);
  }
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = T[N + k];
  reduce_once<C>(r, top);
}

// V4: four carry chains per row.  The operand a and the modulus p are split in halves, a = aL + 2^(32H) aH (H = N/2): the
// low-half products go to the (E, O) column arrays exactly as in mont_mul, the high-half products a_{H+j'} * w and
// p_{H+j'} * m go to a SECOND pair (EH, OH).  Inside a stage of H rows the second pair only ever holds limbs at positions
// >= (first row of the stage) + H, which no quotient digit m of that stage looks at, so its chains are independent of the
// first pair's; after rows H-1 and N-1 everything is merged into one array by plain carry-propagating additions.  Chain-end
// carries are collected in carry-word arrays (as mont_sqr does) and merged at the same points.  Every row then runs four
// independent chains of H/2 IMAD.WIDE instead of two chains of H: half the dependent depth for a lone warp, at the price of
// ~250 extra ALU instructions — for the latency-bound tails only, the throughput kernels keep mont_mul.
template <class C>
NMSM_HD void mont_mul_lat4(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = C::N, H = N / 2, S = 2 * N + 2;
  static_assert(N % 4 == 0, "N/2 must be even (parity of the split point)");
  uint32_t E[S], O[S], EH[S], OH[S], CA[S], CH[S];
#pragma unroll
  for (int k = 0; k < S; k++) E[k] = O[k] = EH[k] = OH[k] = CA[k] = CH[k] = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* P1 = (i & 1) ? O : E;    // slots aligned at position i
    uint32_t* P2 = (i & 1) ? E : O;    // slots aligned at position i + 1
    uint32_t* Q1 = (i & 1) ? OH : EH;  // second pair, same alignment (H is even)
    uint32_t* Q2 = (i & 1) ? EH : OH;
    const uint32_t w = b[i];
    // ---- multiply phase ----
    if (i > 0) P1[i] = add_cc(P1[i], P2[i]);  // leftover high half; carry continues into P2's chain at position i + 1
#pragma unroll
    for (int j = 1; j < H; j += 2) {  // low half, odd j
      P2[i + j] = (i == 0 && j == 1) ? mad_lo_cc(a[j], w, P2[i + j]) : madc_lo_cc(a[j], w, P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(a[j], w, P2[i + j + 1]);
    }
    CA[i + H + 1] = addc(CA[i + H + 1], 0);
#pragma unroll
    for (int j = 0; j < H; j += 2) {  // low half, even j
      P1[i + j] = (j == 0) ? mad_lo_cc(a[j], w, P1[i + j]) : madc_lo_cc(a[j], w, P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(a[j], w, P1[i + j + 1]);
    }
    CA[i + H] = addc(CA[i + H], 0);
#pragma unroll
    for (int j = 0; j < H; j += 2) {  // high half, even j'
      Q1[i + H + j] = (j == 0) ? mad_lo_cc(a[H + j], w, Q1[i + H + j]) : madc_lo_cc(a[H + j], w, Q1[i + H + j]);
      Q1[i + H + j + 1] = madc_hi_cc(a[H + j], w, Q1[i + H + j + 1]);
    }
    CH[i + N] = addc(CH[i + N], 0);
#pragma unroll
    for (int j = 1; j < H; j += 2) {  // high half, odd j'
      Q2[i + H + j] = (j == 1) ? mad_lo_cc(a[H + j], w, Q2[i + H + j]) : madc_lo_cc(a[H + j], w, Q2[i + H + j]);
      Q2[i + H + j + 1] = madc_hi_cc(a[H + j], w, Q2[i + H + j + 1]);
    }
    CH[i + N + 1] = addc(CH[i + N + 1], 0);
    // ---- Montgomery quotient digit: makes limb i vanish ----
    const uint32_t m = P1[i] * C::INV;
#pragma unroll
    for (int j = 1; j < H; j += 2) {
      P2[i + j] = (j == 1) ? mad_lo_cc(m, C::P(j), P2[i + j]) : madc_lo_cc(m, C::P(j), P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(m, C::P(j), P2[i + j + 1]);
    }
    CA[i + H + 1] = addc(CA[i + H + 1], 0);
#pragma unroll
    for (int j = 0; j < H; j += 2) {
      P1[i + j] = (j == 0) ? mad_lo_cc(m, C::P(j), P1[i + j]) : madc_lo_cc(m, C::P(j), P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(m, C::P(j), P1[i + j + 1]);
    }
    CA[i + H] = addc(CA[i + H], 0);
#pragma unroll
    for (int j = 0; j < H; j += 2) {
      Q1[i + H + j] = (j == 0) ? mad_lo_cc(m, C::P(H + j), Q1[i + H + j]) : madc_lo_cc(m, C::P(H + j), Q1[i + H + j]);
      Q1[i + H + j + 1] = madc_hi_cc(m, C::P(H + j), Q1[i + H + j + 1]);
    }
    CH[i + N] = addc(CH[i + N], 0);
#pragma unroll
    for (int j = 1; j < H; j += 2) {
      Q2[i + H + j] = (j == 1) ? mad_lo_cc(m, C::P(H + j), Q2[i + H + j]) : madc_lo_cc(m, C::P(H + j), Q2[i + H + j]);
      Q2[i + H + j + 1] = madc_hi_cc(m, C::P(H + j), Q2[i + H + j + 1]);
    }
    CH[i + N + 1] = addc(CH[i + N + 1], 0);
    // ---- stage boundary: merge the second pair and the carry words into the array the next row folds INTO ----
    if (i == H - 1 || i == N - 1) {
      uint32_t* X = ((i + 1) & 1) ? O : E;  // next row's P1 (for i = N-1 any of the two would do)
      const int lo = i + 1;                 // everything below is zero in all side arrays
      uint32_t* side[4] = {EH, OH, CA, CH};
#pragma unroll
      for (int t = 0; t < 4; t++) {
        X[lo] = add_cc(X[lo], side[t][lo]);
#pragma unroll
        for (int k = lo + 1; k < S; k++) X[k] = addc_cc(X[k], side[t][k]);
#pragma unroll
        for (int k = 0; k < S; k++) side[t][k] = 0;
      }
    }
  }
  // limbs N..2N of E + O
  r[0] = add_cc(E[N], O[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(E[N + k], O[N + k]);
  uint32_t top = addc(E[2 * N], O[2 * N]);
  reduce_once<C>(r, top);
}

}  // namespace nmsm
