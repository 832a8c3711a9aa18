// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Compiles the device headers (field.cuh / ec.cuh / msm_body.cuh) for the HOST with g++ and an
// emulated PTX carry flag (bigint.cuh), and drives the per-thread kernel bodies in plain loops.
// This lets `pytest -m "not gpu"` verify the limb arithmetic, the group formulas and the bucket
// bookkeeping of the CUDA path bit-for-bit against the oracle on a box without a GPU.  It is not a
// CPU fallback: the product package cannot load or call it.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "msm_body.cuh"
#include "ed25519_verify.cuh"
#include "codec.cuh"
#include "validate.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;

// plans are made for the SM count of the target GPU (H100 SXM: 132 SMs), as nmsm_init does from the device
static constexpr int EMU_SM_COUNT = 132;

// what k_accumulate runs per thread.  g_paired = 0 (the default build, NMSM_PAIRED=0): the plain mixed-addition loop;
// g_paired = 1: the paired accumulation of the NMSM_PAIRED=1 build for the short-Weierstrass curves (the warp-shared
// inversion of the kernel becomes a plain inversion of this thread's product) — both are parity-tested.
static int g_paired = 0;
extern "C" int emu_set_paired(int on) { int prev = g_paired; g_paired = on; return prev; }
template <class Cv>
static void emu_accumulate(uint32_t w, uint32_t t, const uint32_t* aff, const uint32_t* sorted, const uint32_t* offsets,
                           const MsmPlan& plan, uint32_t* buckets, uint32_t* heads, uint32_t* tails) {
  if (!g_paired) {
    accumulate_body<Cv>(w, t, aff, sorted, offsets, plan, buckets, heads, tails);
    return;
  }
  if constexpr (!Cv::G::IS_EDWARDS) {
    using F = typename Cv::G::Field;
    F suf[MAX_PAIRS];
    int npairs;
    const F run = accumulate_pairs_pass1<Cv>(w, t, aff, sorted, offsets, plan, suf, npairs);
    accumulate_pairs_pass2<Cv>(w, t, aff, sorted, offsets, plan, suf, npairs, inv(run), buckets, heads, tails);
  } else {
    accumulate_body<Cv>(w, t, aff, sorted, offsets, plan, buckets, heads, tails);
  }
}

template <class Cv>
static int emu_msm_t(const uint32_t* pts, const uint32_t* scalars, uint32_t n, int forced_c, int forced_L,
                     uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out, uint32_t* plan_out, int table_c = 0,
                     int groups = 1) {
  using G = typename Cv::G;
  // table_c != 0: fixed-base table route (nmsm_points_precompute + nmsm_msm_points)
  MsmPlan plan = table_c ? make_table_plan<Cv>(n, canonical_table_bits<Cv>(table_c), EMU_SM_COUNT) : make_plan<Cv>(n, forced_c, EMU_SM_COUNT);
  if (forced_L > 0) {
    plan.L = forced_L;
    plan.TPW = plan_tpw((uint64_t)n * split_of<Cv>() * (table_c ? plan.D : 1), plan.L);
  }
  plan_out[0] = plan.c; plan_out[1] = plan.W; plan_out[2] = plan.B; plan_out[3] = plan.L;
  const size_t terms = (size_t)n * split_of<Cv>();
  std::vector<uint32_t> aff(terms * G::AFF_WORDS * (table_c ? plan.D : 1));
  std::vector<unsigned int> counts(plan.G + 1, 0), cursor(plan.G + 1, 0);
  std::vector<uint32_t> offsets(plan.G + 1, 0);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  for (uint32_t i = 0; i < n; i++) prepare_body<Cv>(i, n, pts, aff.data(), err);
  if (table_c && err[0] == 0xffffffffu)
    for (int j = 1; j < plan.D; j++)
      for (uint32_t i = 0; i < terms; i++)
        table_level_body<Cv>(i, aff.data() + (size_t)(j - 1) * terms * G::AFF_WORDS,
                             aff.data() + (size_t)j * terms * G::AFF_WORDS, digit_width(plan, j - 1));
  for (uint32_t i = 0; i < n; i++) digits_body<Cv, false>(i, n, scalars, plan, counts.data(), nullptr, err);
  uint32_t run = 0;
  for (int g = 0; g < plan.G; g++) { offsets[g] = run; cursor[g] = run; run += counts[g]; }
  offsets[plan.G] = run;
  const uint32_t T = run;
  std::vector<uint32_t> sorted(T ? T : 1);
  for (uint32_t i = 0; i < n; i++) digits_body<Cv, true>(i, n, scalars, plan, cursor.data(), sorted.data(), err);
  (void)T;
  // segments: TPW per window (the launch geometry of k_accumulate: every (w, t) with t < TPW runs, most exit at once)
  const size_t nseg = (size_t)plan.W * plan.TPW;
  std::vector<uint32_t> buckets((size_t)plan.G * G::ACC_WORDS, 0xdeadbeefu);
  std::vector<uint32_t> heads(nseg * G::ACC_WORDS, 0xdeadbeefu), tails(nseg * G::ACC_WORDS, 0xdeadbeefu);
  const size_t nchunks = (size_t)plan.W * plan.chunks;
  std::vector<uint32_t> sums(nchunks * G::ACC_WORDS), wsums(nchunks * G::ACC_WORDS);
  const uint32_t ntile1 = (uint32_t)(nseg / STITCH_FAN), ntile2 = ntile1 / STITCH_FAN;
  std::vector<uint32_t> tile1((size_t)ntile1 * G::ACC_WORDS, 0xdeadbeefu), tile2((size_t)(ntile2 + 1) * G::ACC_WORDS, 0xdeadbeefu);
  std::vector<uint32_t> window_out((size_t)plan.W * G::ACC_WORDS), hacc(G::ACC_WORDS);
  // window groups, top windows first, exactly as engine.cuh submit_msm issues them
  if (groups < 1) groups = 1;
  if (groups > plan.W) groups = plan.W;
  const int per = (plan.W + groups - 1) / groups;
  bool first = true;
  for (int w_hi = plan.W; w_hi > 0; w_hi -= per) {
    const int w_lo = w_hi > per ? w_hi - per : 0;
    for (int w = w_lo; w < w_hi; w++)
      for (uint32_t t = 0; t < plan.TPW; t++) {
        // skip the (many) idle segments quickly: same early exit the body takes
        if ((uint64_t)offsets[(size_t)w * plan.B] + (uint64_t)t * plan.L >= offsets[(size_t)(w + 1) * plan.B] && t > 2) break;
        emu_accumulate<Cv>(w, t, aff.data(), sorted.data(), offsets.data(), plan, buckets.data(), heads.data(), tails.data());
      }
    const uint32_t a0 = (uint32_t)((uint64_t)w_lo * plan.TPW / STITCH_FAN), a1 = (uint32_t)((uint64_t)w_hi * plan.TPW / STITCH_FAN);
    for (uint32_t j = a0; j < a1; j++) stitch_tile_serial<Cv>(j, STITCH_FAN, offsets.data(), plan, heads.data(), tile1.data());
    for (uint32_t j = a0 / STITCH_FAN; j < a1 / STITCH_FAN; j++)
      stitch_tile_serial<Cv>(j, STITCH_FAN * STITCH_FAN, offsets.data(), plan, tile1.data(), tile2.data());
    for (uint32_t id = (uint32_t)w_lo * plan.chunks; id < (uint32_t)w_hi * plan.chunks; id++)
      reduce1_body<Cv, SerialOps<G>>(id, offsets.data(), buckets.data(), heads.data(), tails.data(), tile1.data(), tile2.data(), plan, sums.data(), wsums.data());
    for (int w = w_lo; w < w_hi; w++)  // serial statement of what k_reduce2 computes cooperatively
      reduce2_serial<Cv>(w, sums.data(), wsums.data(), plan, window_out.data());
    horner_step_body<Cv>(window_out.data(), plan, w_lo, w_hi, first, false, hacc.data());
    first = false;
  }
  fold_body<Cv>(hacc.data(), 1, out_xy, out_inf);  // k_combine<AFFINE_OUT>: fold of one accumulator + to-affine
  err_out[0] = err[0];
  err_out[1] = err[1];
  // cross-check 1: the classic single Horner over all windows (final_body) must agree
  {
    std::vector<uint32_t> xy1(G::IN_WORDS);
    uint32_t inf1 = 7;
    final_body<Cv, true>(window_out.data(), plan, xy1.data(), &inf1);
    if (inf1 != *out_inf || memcmp(xy1.data(), out_xy, G::IN_WORDS * 4) != 0) return -101;
  }
  // cross-check 2: shifted per-window results (what multi-GPU window owners compute) summed by the fold
  {
    std::vector<uint32_t> parts((size_t)plan.W * G::ACC_WORDS), xy1(G::IN_WORDS);
    uint32_t inf1 = 7;
    for (int w = 0; w < plan.W; w++) horner_step_body<Cv>(window_out.data(), plan, w, w + 1, true, true, parts.data() + (size_t)w * G::ACC_WORDS);
    fold_body<Cv>(parts.data(), plan.W, xy1.data(), &inf1);
    if (plan.stride == 0 && (inf1 != *out_inf || memcmp(xy1.data(), out_xy, G::IN_WORDS * 4) != 0)) return -102;
  }
  // also exercise the partial + fold route (multi-GPU path): must give the same answer
  std::vector<uint32_t> raw(2 * G::ACC_WORDS);
  final_body<Cv, false>(window_out.data(), plan, raw.data(), nullptr);
  typename G::Acc id = G::identity();
  save_acc<G>(raw.data() + G::ACC_WORDS, id);
  std::vector<uint32_t> xy2(G::IN_WORDS);
  uint32_t inf2 = 7;
  fold_body<Cv>(raw.data(), 2, xy2.data(), &inf2);
  if (inf2 != *out_inf || memcmp(xy2.data(), out_xy, G::IN_WORDS * 4) != 0) return -100;
  return 0;
}

// ---- sharded MSM with bucket exchange (engine.cuh submit_msm, shard != nullptr) ---------------------------------
// Stage 1 on every rank: local terms -> DENSE buckets of all windows, planned for the global term count.
template <class Cv>
static int emu_shard_buckets_t(const uint32_t* pts, const uint32_t* scalars, uint32_t n_local, uint32_t n_total,
                               uint32_t* buckets_out, uint32_t* plan_out, uint32_t* err_out) {
  using G = typename Cv::G;
  MsmPlan plan = make_plan<Cv>(n_total, 0, EMU_SM_COUNT, n_local ? n_local : 1);
  plan_out[0] = plan.c; plan_out[1] = plan.W; plan_out[2] = plan.B; plan_out[3] = G::ACC_WORDS;
  if (!buckets_out) return 0;  // plan query
  const size_t terms = (size_t)(n_local ? n_local : 1) * split_of<Cv>();
  std::vector<uint32_t> aff(terms * G::AFF_WORDS);
  std::vector<unsigned int> counts(plan.G + 1, 0), cursor(plan.G + 1, 0);
  std::vector<uint32_t> offsets(plan.G + 1, 0);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  for (uint32_t i = 0; i < n_local; i++) prepare_body<Cv>(i, n_local, pts, aff.data(), err);
  for (uint32_t i = 0; i < n_local; i++) digits_body<Cv, false>(i, n_local, scalars, plan, counts.data(), nullptr, err);
  uint32_t run = 0;
  for (int g = 0; g < plan.G; g++) { offsets[g] = run; cursor[g] = run; run += counts[g]; }
  offsets[plan.G] = run;
  std::vector<uint32_t> sorted(run ? run : 1);
  for (uint32_t i = 0; i < n_local; i++) digits_body<Cv, true>(i, n_local, scalars, plan, cursor.data(), sorted.data(), err);
  const size_t nseg = (size_t)plan.W * plan.TPW;
  std::vector<uint32_t> heads(nseg * G::ACC_WORDS, 0xdeadbeefu), tails(nseg * G::ACC_WORDS, 0xdeadbeefu);
  const uint32_t ntile1 = (uint32_t)(nseg / STITCH_FAN), ntile2 = ntile1 / STITCH_FAN;
  std::vector<uint32_t> tile1((size_t)ntile1 * G::ACC_WORDS, 0xdeadbeefu), tile2((size_t)(ntile2 + 1) * G::ACC_WORDS, 0xdeadbeefu);
  for (size_t k = 0; k < (size_t)plan.G * G::ACC_WORDS; k++) buckets_out[k] = 0xdeadbeefu;
  for (int w = 0; w < plan.W; w++)
    for (uint32_t t = 0; t < plan.TPW; t++) {
      if ((uint64_t)offsets[(size_t)w * plan.B] + (uint64_t)t * plan.L >= offsets[(size_t)(w + 1) * plan.B] && t > 2) break;
      emu_accumulate<Cv>(w, t, aff.data(), sorted.data(), offsets.data(), plan, buckets_out, heads.data(), tails.data());
    }
  for (uint32_t j = 0; j < ntile1; j++) stitch_tile_serial<Cv>(j, STITCH_FAN, offsets.data(), plan, heads.data(), tile1.data());
  for (uint32_t j = 0; j < ntile2; j++) stitch_tile_serial<Cv>(j, STITCH_FAN * STITCH_FAN, offsets.data(), plan, tile1.data(), tile2.data());
  for (uint32_t g = 0; g < (uint32_t)plan.G; g++)
    bucket_finalize_body<Cv>(g, offsets.data(), buckets_out, heads.data(), tails.data(), tile1.data(), tile2.data(), plan);
  err_out[0] = err[0];
  err_out[1] = err[1];
  return 0;
}
// Stage 2 on the owner of window w: fold the peers' partial buckets, reduce the window, weight it by 2^(c w).
// `own` = this rank's dense buckets of window w (B accumulators, modified in place), `recv` = npeers such arrays.
template <class Cv>
static int emu_owner_window_t(uint32_t n_total, int w, uint32_t* own, const uint32_t* recv, int npeers, uint32_t* out_acc) {
  using G = typename Cv::G;
  MsmPlan plan = make_plan<Cv>(n_total, 0, EMU_SM_COUNT, 1);
  const size_t WB = (size_t)plan.B * G::ACC_WORDS;
  for (uint32_t b = 0; b < (uint32_t)plan.B; b++) bucket_fold_body<Cv>(b, own, recv, npeers, WB);
  // the kernels index buckets / chunks / window sums globally: stage the window at its global position
  std::vector<uint32_t> all((size_t)plan.W * WB, 0xdeadbeefu);
  memcpy(all.data() + (size_t)w * WB, own, WB * 4);
  const size_t nchunks = (size_t)plan.W * plan.chunks;
  std::vector<uint32_t> sums(nchunks * G::ACC_WORDS), wsums(nchunks * G::ACC_WORDS), window_out((size_t)plan.W * G::ACC_WORDS);
  for (uint32_t id = (uint32_t)w * plan.chunks; id < (uint32_t)(w + 1) * plan.chunks; id++)
    reduce1_dense_body<Cv>(id, all.data(), plan, sums.data(), wsums.data());
  reduce2_serial<Cv>(w, sums.data(), wsums.data(), plan, window_out.data());
  horner_step_body<Cv>(window_out.data(), plan, w, w + 1, true, true, out_acc);
  return 0;
}

// multi-GPU building blocks: raw accumulator of a shard, and the fold of several accumulators
template <class Cv>
static int emu_partial_t(const uint32_t* pts, const uint32_t* scalars, uint32_t n, uint32_t* out_acc) {
  using G = typename Cv::G;
  if (n == 0) {
    typename G::Acc id = G::identity();
    save_acc<G>(out_acc, id);
    return 0;
  }
  std::vector<uint32_t> xy(G::IN_WORDS);
  uint32_t inf, err[2], plan[4];
  // run the full pipeline and lift its affine result back to a raw accumulator
  int rc = emu_msm_t<Cv>(pts, scalars, n, 0, 0, xy.data(), &inf, err, plan);
  if (rc) return rc;
  typename G::Acc acc = G::identity();
  if (!inf) {
    typename G::Affine a = G::prepare(xy.data());
    acc = G::from_affine(a);
  }
  save_acc<G>(out_acc, acc);
  return 0;
}
template <class Cv>
static int emu_fold_t(const uint32_t* accs, int count, uint32_t* out_xy, uint32_t* out_inf) {
  fold_body<Cv>(accs, count, out_xy, out_inf);
  return 0;
}

template <class Cv>
static int emu_mul_t(const uint32_t* pts, const uint32_t* scalars, uint32_t n, int allow_zero, uint32_t* out_xy,
                     uint32_t* out_inf, uint32_t* err_out) {
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  for (uint32_t i = 0; i < n; i++) mul_body<Cv>(i, pts, scalars, allow_zero, out_xy, out_inf, err);
  err_out[0] = err[0];
  err_out[1] = err[1];
  return 0;
}

// Fixed-point multiplication table (nmsm_point_table_*) with TB-bit digits: the production bodies, small table.
template <class Cv, int TB>
static int emu_point_table_t(const uint32_t* point_xy, const uint32_t* scalars, uint32_t n, int allow_zero,
                             uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out) {
  using G = typename Cv::G;
  constexpr int LV = point_table_levels<Cv, TB>();
  constexpr uint32_t HALF = 1u << (TB - 1);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  std::vector<uint32_t> aff((size_t)split_of<Cv>() * G::AFF_WORDS);
  prepare_body<Cv>(0, 1, point_xy, aff.data(), err);
  const size_t level_words = (size_t)HALF * G::AFF_WORDS;
  std::vector<uint32_t> tbl(level_words * LV);
  for (uint32_t i = 0; i < HALF; i++) table_base_body<Cv, TB>(i, aff.data(), tbl.data());
  for (int j = 1; j < LV; j++)
    for (uint32_t i = 0; i < HALF; i++)
      table_level_body<Cv>(i, tbl.data() + (size_t)(j - 1) * level_words, tbl.data() + (size_t)j * level_words, TB);
  for (uint32_t i = 0; i < n; i++) {
    typename G::Acc acc;
    out_inf[i] = 9;
    if (!table_mul_body<Cv, TB>(i, tbl.data(), scalars, allow_zero, acc, err)) continue;
    nl_to_affine<G>(acc, out_xy + (size_t)i * G::IN_WORDS, out_inf + i);
  }
  err_out[0] = err[0];
  err_out[1] = err[1];
  return 0;
}

template <class Cv>
static int emu_torsion_t(const uint32_t* pts, uint32_t n, uint8_t* out_ok, uint32_t* err_out) {
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  for (uint32_t i = 0; i < n; i++) torsion_body<Cv>(i, pts, out_ok, err);
  err_out[0] = err[0];
  err_out[1] = err[1];
  return 0;
}

// plan introspection for tests: out = {c, W, B, L, K, chunks, D, wb, r, stride, auto_c}
template <class Cv>
static int emu_plan_t(uint32_t n, int table_c_req, uint32_t* out) {
  MsmPlan p = table_c_req ? make_table_plan<Cv>(n, canonical_table_bits<Cv>(table_c_req), EMU_SM_COUNT) : make_plan<Cv>(n, 0, EMU_SM_COUNT);
  out[0] = p.c; out[1] = p.W; out[2] = p.B; out[3] = p.L; out[4] = p.K; out[5] = p.chunks; out[6] = p.D;
  out[7] = p.wb; out[8] = p.r; out[9] = p.stride;
  out[10] = choose_table_bits<Cv>(n, EMU_SM_COUNT, 64e9);
  out[11] = glv_bits<Cv>() + 1;
  return 0;
}

#define DISPATCH(curve, EXPR)                                        \
  switch (curve) {                                                   \
    case 0: { using Cv = CurveSecp256k1; return EXPR; }              \
    case 1: { using Cv = CurveEd25519; return EXPR; }                \
    case 2: { using Cv = CurveBn254G1; return EXPR; }                \
    case 3: { using Cv = CurveBn254G2; return EXPR; }                \
    case 4: { using Cv = CurveBls381G1; return EXPR; }               \
    case 5: { using Cv = CurveBls381G2; return EXPR; }               \
    case 6: { using Cv = CurveBls381G1Any; return EXPR; }            \
    case 7: { using Cv = CurveBls381G2Any; return EXPR; }            \
    default: return -1;                                              \
  }

template <class P>
static void field_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  Fp<P> x, y, z;
  for (int i = 0; i < P::N; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  switch (op) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 3: z = inv_xgcd(x); break;                                                  // the fallback path
    case 10: z = inv(x); break;                                                      // what the kernels call (divsteps)
    case 4: z = Fp<P>::from_canonical(a); break;
    case 5: x.to_canonical(z.v); break;
    case 6: z = sqr(x); break;
    case 8: z = DivstepsInv<P>::inverse(x); break;                                  // Montgomery in / out
    case 9: if (!DivstepsInv<P>::inverse_words(a, z.v)) z = Fp<P>::zero(); break;    // plain integers
    case 11: z = Fp<P>::zero(); z.v[0] = Fp<P>::canonical_in_range(a) ? 1u : 0u; break;
    default: z = -x; break;
  }
  for (int i = 0; i < P::N; i++) r[i] = z.v[i];
}

// op 0: T = a * b as 2N words (any N-limb a, b); op 1: T / R mod p of a 2N-word T < p R / 2 (field.cuh mul_wide,
// mont_reduce_wide)
template <class P>
static void wide_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (op == 0) mul_wide<P>(r, a, b);
  else mont_reduce_wide<P>(r, a);
}

static int emu_ed_verify(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                         const uint8_t* z16, int* out_ok, long long* out_bad) {
  using Cv = CurveEd25519;
  using G = Cv::G;
  *out_ok = 0;
  *out_bad = -1;
  if (n == 0) { *out_ok = 1; return 0; }
  const uint32_t terms = 2 * n + 1;
  std::vector<uint32_t> pts((size_t)terms * 16), sc((size_t)terms * 8), zs((size_t)n * 8);
  unsigned int bad = 0xffffffffu;
  for (uint32_t i = 0; i < n; i++) ed_terms_body(i, n, sigs, pks, msgs, off, z16, pts.data(), sc.data(), zs.data(), &bad);
  ed_finish_serial(n, zs.data(), pts.data(), sc.data());
  std::vector<uint32_t> acc_words(G::ACC_WORDS);
  int rc = emu_partial_t<Cv>(pts.data(), sc.data(), terms, acc_words.data());
  if (rc) return rc;
  G::Acc acc = load_acc<G>(acc_words.data());
  for (int j = 0; j < 3; j++) G::dbl(acc);
  if (bad != 0xffffffffu) { *out_bad = bad; return 0; }
  *out_ok = G::is_identity(acc) ? 1 : 0;
  return 0;
}

// Fp2 operations on Montgomery-form operands (a, b, r: c0 limbs then c1 limbs), both statements of the multiplication:
// form 0 = three reduced base multiplications (tower.ts:420-431 order), form 1 = Karatsuba with lazy reduction,
// form 2 = operator*, form 3 = sqr, form 4 = inv
template <class P>
static void fp2_mul_forms(int form, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  Fp2<P> x, y, z;
  for (int i = 0; i < P::N; i++) {
    x.c0.v[i] = a[i]; x.c1.v[i] = a[P::N + i];
    y.c0.v[i] = b[i]; y.c1.v[i] = b[P::N + i];
  }
  if (form == 1) {
    z = Fp2<P>::mul_lazy(x, y);
  } else if (form == 2) {
    z = x * y;
  } else if (form == 3) {
    z = sqr(x);
  } else if (form == 4) {
    z = inv(x);
  } else {
    Fp<P> t1 = x.c0 * y.c0, t2 = x.c1 * y.c1;
    z = Fp2<P>{t1 - t2, (x.c0 + x.c1) * (y.c0 + y.c1) - (t1 + t2)};
  }
  for (int i = 0; i < P::N; i++) { r[i] = z.c0.v[i]; r[P::N + i] = z.c1.v[i]; }
}
extern "C" {
int emu_ed25519_decompress(const uint8_t* enc, uint32_t* out_xy) { return ed_decompress(enc, out_xy) ? 1 : 0; }
int emu_sha512_rAM(const uint8_t* r, const uint8_t* a, const uint8_t* msg, uint64_t mlen, uint8_t* digest) {
  sha512_rAM(r, a, msg, mlen, digest);
  return 0;
}
int emu_ed25519_verify_batch(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                             const uint8_t* z16, int* out_ok, long long* out_bad) {
  return emu_ed_verify(sigs, pks, msgs, off, n, z16, out_ok, out_bad);
}
// Fp2 square root over BLS12-381 Fp (codec.cuh fp2_sqrt): canonical c0 || c1 words in and out; returns 1 if a root exists
int emu_fp2_sqrt(const uint32_t* in, uint32_t* out) {
  Fp2<FpBls381> n = Fp2<FpBls381>::from_canonical(in), r;
  if (!fp2_sqrt<FpBls381>(n, r)) return 0;
  r.to_canonical(out);
  return 1;
}
int emu_decode(int curve, const uint8_t* enc, uint32_t* out_xy) {
  if (curve == 0) return sec1_decode_secp256k1(enc, out_xy);
  if (curve == 4) return zcash_decode_bls12_381_g1(enc, out_xy);
  if (curve == 5) return zcash_decode_bls12_381_g2(enc, out_xy);
  if (curve == 1) return ed25519_decode(enc, out_xy);
  return -1;
}
// GLV split of one scalar (BLS12-381 G1): out = m1[4], m2[4], neg1, neg2
int emu_glv_split(const uint32_t* k, uint32_t* out) {
  bool n1, n2;
  glv_split<Bls381G1Glv>(k, out, n1, out + 4, n2);
  out[8] = n1;
  out[9] = n2;
  return 0;
}
// psi-GLS split of one scalar (BLS12-381 G2): out = mag[4] as (lo, hi) word pairs, then neg[4]
int emu_gls_split(const uint32_t* k, uint32_t* out) {
  uint64_t mag[4];
  bool neg[4];
  gls_split<Bls381G2Gls>(k, mag, neg);
  for (int j = 0; j < 4; j++) {
    out[2 * j] = (uint32_t)mag[j];
    out[2 * j + 1] = (uint32_t)(mag[j] >> 32);
    out[8 + j] = neg[j];
  }
  return 0;
}
// lattice GLV split (curve 0 = secp256k1, 2 = bn254 G1): out = m1[5], m2[5], neg1, neg2
int emu_glv_split_lattice(int curve, const uint32_t* k, uint32_t* out) {
  bool n1, n2;
  if (curve == 0) glv_split_lattice<Secp256k1Glv>(k, out, n1, out + 5, n2);
  else glv_split_lattice<Bn254G1Glv>(k, out, n1, out + 5, n2);
  out[10] = n1;
  out[11] = n2;
  return 0;
}
int emu_point_table(int curve, int table_bits, const uint32_t* point_xy, const uint32_t* scalars, uint32_t n,
                    int allow_zero, uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out) {
  if (table_bits == 5) {
    DISPATCH(curve, (emu_point_table_t<Cv, 5>(point_xy, scalars, n, allow_zero, out_xy, out_inf, err_out)));
  }
  DISPATCH(curve, (emu_point_table_t<Cv, 8>(point_xy, scalars, n, allow_zero, out_xy, out_inf, err_out)));
}
int emu_torsion(int curve, const uint32_t* pts, uint32_t n, uint8_t* out_ok, uint32_t* err_out) {
  DISPATCH(curve, emu_torsion_t<Cv>(pts, n, out_ok, err_out));
}
int emu_plan(int curve, uint32_t n, int table_c_req, uint32_t* out) { DISPATCH(curve, emu_plan_t<Cv>(n, table_c_req, out)); }
int emu_msm_table(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n, int table_c, int forced_L,
                  uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out, uint32_t* plan_out) {
  DISPATCH(curve, emu_msm_t<Cv>(pts, scalars, n, 0, forced_L, out_xy, out_inf, err_out, plan_out, table_c));
}
int emu_msm(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n, int forced_c, int forced_L,
            uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out, uint32_t* plan_out) {
  DISPATCH(curve, emu_msm_t<Cv>(pts, scalars, n, forced_c, forced_L, out_xy, out_inf, err_out, plan_out));
}
int emu_msm_groups(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n, int forced_c, int forced_L, int groups,
                   uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out, uint32_t* plan_out) {
  DISPATCH(curve, emu_msm_t<Cv>(pts, scalars, n, forced_c, forced_L, out_xy, out_inf, err_out, plan_out, 0, groups));
}
int emu_ed25519_decompress_strict(const uint8_t* enc, uint32_t* out_xy) { return ed_decompress(enc, out_xy, false) ? 1 : 0; }
int emu_on_curve(int curve, const uint32_t* xy) { DISPATCH(curve, point_on_curve<Cv>(xy)); }
int emu_mul_batch(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n, int allow_zero,
                  uint32_t* out_xy, uint32_t* out_inf, uint32_t* err_out) {
  DISPATCH(curve, emu_mul_t<Cv>(pts, scalars, n, allow_zero, out_xy, out_inf, err_out));
}
int emu_msm_partial(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n, uint32_t* out_acc) {
  DISPATCH(curve, emu_partial_t<Cv>(pts, scalars, n, out_acc));
}
int emu_shard_buckets(int curve, const uint32_t* pts, const uint32_t* scalars, uint32_t n_local, uint32_t n_total,
                      uint32_t* buckets_out, uint32_t* plan_out, uint32_t* err_out) {
  DISPATCH(curve, emu_shard_buckets_t<Cv>(pts, scalars, n_local, n_total, buckets_out, plan_out, err_out));
}
int emu_owner_window(int curve, uint32_t n_total, int w, uint32_t* own, const uint32_t* recv, int npeers, uint32_t* out_acc) {
  DISPATCH(curve, emu_owner_window_t<Cv>(n_total, w, own, recv, npeers, out_acc));
}
int emu_fold(int curve, const uint32_t* accs, int count, uint32_t* out_xy, uint32_t* out_inf) {
  DISPATCH(curve, emu_fold_t<Cv>(accs, count, out_xy, out_inf));
}
int emu_fp2_mul(int field, int form, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field == 2) { fp2_mul_forms<FpBn254>(form, a, b, r); return 0; }
  if (field == 3) { fp2_mul_forms<FpBls381>(form, a, b, r); return 0; }
  return -1;
}
// field: 0 secp256k1 p, 1 ed25519 p, 2 bn254 p, 3 bls12-381 p, 4 secp256k1 n, 5 ed25519 l, 6 bn254 r, 7 bls12-381 r
int emu_field(int field, int op, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  switch (field) {
    case 0: field_op<FpSecp256k1>(op, a, b, r); return 0;
    case 1: field_op<FpEd25519>(op, a, b, r); return 0;
    case 2: field_op<FpBn254>(op, a, b, r); return 0;
    case 3: field_op<FpBls381>(op, a, b, r); return 0;
    case 4: field_op<FnSecp256k1Mod>(op, a, b, r); return 0;
    case 5: field_op<FnEd25519Mod>(op, a, b, r); return 0;
    case 6: field_op<FrBn254>(op, a, b, r); return 0;
    case 7: field_op<FrBls381>(op, a, b, r); return 0;
  }
  return -1;
}
// batched forms of emu_field / field_op, wide_op and emu_fp2_mul: n cases laid out back to back, the interface of
// tests/devemu's dev_field / dev_wide / dev_fp2
int emu_field_n(int field, int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field < 0 || field > 7) return -1;
  const size_t N = field == 3 ? 12 : 8;
  for (uint32_t i = 0; i < n; i++) emu_field(field, op, a + i * N, b + i * N, r + i * N);
  return 0;
}
int emu_wide_n(int field, int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field != 2 && field != 3) return -1;
  const size_t N = field == 3 ? 12 : 8, wa = op == 0 ? N : 2 * N, wr = op == 0 ? 2 * N : N;
  for (uint32_t i = 0; i < n; i++) {
    if (field == 2) wide_op<FpBn254>(op, a + i * wa, b + i * N, r + i * wr);
    else wide_op<FpBls381>(op, a + i * wa, b + i * N, r + i * wr);
  }
  return 0;
}
int emu_fp2_n(int field, int form, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field != 2 && field != 3) return -1;
  const size_t W = field == 3 ? 24 : 16;
  for (uint32_t i = 0; i < n; i++) emu_fp2_mul(field, form, a + i * W, b + i * W, r + i * W);
  return 0;
}
}
