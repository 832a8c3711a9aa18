// BLS12-381 aggregate verification (SURVEY §8 row f3): FastAggregateVerify and noble's verifyBatch with per-message
// key sums (abstract/bls.ts verifyBatch).  Check j has one signature and groups [group_off[j], group_off[j+1]); group g
// has one message and keys [key_off[g], key_off[g+1]):
//   check j:  e(-G1, sig_j) prod_g e(S_g, H(m_g)) == 1,   S_g = sum of group g's keys
// Keys are affine G1 points the caller has decoded and subgroup-checked (the identity is (0, 0)); here they are only
// range- and curve-checked.  Pair layout: check j owns pairs [group_off[j] + j, group_off[j+1] + j + 1), its groups'
// (S_g, H(m_g)) first, then (-G1, sig_j); pairing_checks_run<BlsPairing> runs them as any other pairing check.
//   k_bls_key_tiles    one warp per tile of at most a tile size of keys of one group: lanes add strided keys with the
//                      complete mixed addition, then combine by shuffles with the complete addition (a group may repeat
//                      a key or hold P and -P); range and curve checks, identity keys mark the tile bad
//   k_bls_key_groups   one thread per group: folds its tile partials, S_g affine through one warp-shared inversion,
//                      writes (S_g, H(m_g)) into the group's pair (two identities when the group is bad) and group_ok
//   k_bls_agg_prepare  one thread per check: signature decode and G2 subgroup check, the AND of its group_ok bytes and
//                      the non-empty rules into pre_ok, the pair (-G1, sig); a rejected check's pairs are all zeroed so
//                      that their Miller loops are skipped
// Bodies are host/device so tests/hostemu can run them; bls_agg_serial is the kernels' work in order.
#pragma once
#include <vector>

#include "pairing.cuh"

namespace nmsm {

using BlsG1 = CurveBls381G1Any::G;
static constexpr int BLS_ACC_WORDS = BlsG1::ACC_WORDS;  // 48 words: one XYZZ tile partial
static constexpr uint32_t BLS_KEY_LANES = 32;           // lanes per tile (one warp)

// tile t: keys [k0, k1) of one group, k0 < k1
struct BlsKeyTile {
  uint32_t k0, k1;
};

// The tile table of n_groups groups (host): a group of nk keys gets ceil(nk / s) tiles of s = max(tile, ceil(nk / cap))
// keys, so a small group costs one tile and a huge one spreads over at most cap warps (which bounds the serial fold of
// k_bls_key_groups).  An empty group gets no tile.  tile_off: n_groups + 1 entries.
inline void bls_key_tiles(const uint64_t* key_off, uint64_t n_groups, uint64_t tile, uint64_t cap,
                          std::vector<BlsKeyTile>& tiles, std::vector<uint32_t>& tile_off) {
  tiles.clear();
  tile_off.resize(n_groups + 1);
  for (uint64_t g = 0; g < n_groups; g++) {
    tile_off[g] = (uint32_t)tiles.size();
    const uint64_t a = key_off[g], b = key_off[g + 1], nk = b - a;
    const uint64_t s = nk > tile * cap ? (nk + cap - 1) / cap : tile;
    for (uint64_t k = a; k < b; k += s) tiles.push_back(BlsKeyTile{(uint32_t)k, (uint32_t)(k + s < b ? k + s : b)});
  }
  tile_off[n_groups] = (uint32_t)tiles.size();
}

// lane `lane` of tile t: the sum of keys k0 + lane, k0 + lane + 32, ... below k1.  A key with a coordinate >= p or off
// the curve sets err[0] to the smallest such index; it and an identity key make the lane bad.
NMSM_HD BlsG1::Acc bls_key_lane(const BlsKeyTile& t, uint32_t lane, const uint32_t* keys, bool& bad, unsigned int* err) {
  BlsG1::Acc acc = BlsG1::identity();
  for (uint32_t k = t.k0 + lane; k < t.k1; k += BLS_KEY_LANES) {
    uint32_t xy[24];
    load_words<24>(xy, keys + (size_t)k * 24);
    if (!point_on_curve<CurveBls381G1Any>(xy)) {
      atomic_min_u32(&err[0], k);
      bad = true;
    } else if (words_zero(xy, 24)) {
      bad = true;
    } else {
      BlsG1::madd(acc, BlsG1::prepare(xy));
    }
  }
  return acc;
}

NMSM_HD void bls_acc_load(BlsG1::Acc& p, const uint32_t* src) {
  uint32_t* d = reinterpret_cast<uint32_t*>(&p);
  load_words<BLS_ACC_WORDS>(d, src);
}

// k_bls_key_groups, group g: the fold of its tile partials; ok = at least one tile, no bad tile and S_g != O
NMSM_HD BlsG1::Acc bls_group_sum(uint32_t g, const uint32_t* tile_off, const uint32_t* partials,
                                 const uint8_t* tile_bad, bool& ok) {
  BlsG1::Acc s = BlsG1::identity(), q;
  ok = tile_off[g] < tile_off[g + 1];
  for (uint32_t t = tile_off[g]; t < tile_off[g + 1]; t++) {
    bls_acc_load(q, partials + (size_t)t * BLS_ACC_WORDS);
    BlsG1::add(s, q);
    ok = ok && !tile_bad[t];
  }
  ok = ok && !BlsG1::is_identity(s);
  return s;
}

// the pair of group g (pair index pair): (S_g, H(m_g)) from s and zi = ZZZ^-1, or two identities when !ok
NMSM_HD void bls_group_store(uint32_t g, uint32_t pair, bool ok, const BlsG1::Acc& s, const BlsF& zi,
                             const uint32_t* h, uint32_t* g1, uint32_t* g2, uint8_t* group_ok) {
  uint32_t xy[24], hq[48], inf;
  for (int k = 0; k < 24; k++) xy[k] = 0u;
  for (int k = 0; k < 48; k++) hq[k] = 0u;
  if (ok) {
    BlsG1::to_affine_canonical_with_inv(s, zi, xy, &inf);
    load_words<48>(hq, h + (size_t)g * 48);
  }
  store_words<24>(g1 + (size_t)pair * 24, xy);
  store_words<48>(g2 + (size_t)pair * 48, hq);
  group_ok[g] = ok ? 1 : 0;
}

// k_bls_agg_prepare, check j: pre_ok[j] = at least one group, every group_ok, sig decodes, is not the identity and is
// in G2.  Writes the pair (-G1, sig) at group_off[j+1] + j, and zeroes all of the check's pairs when it is rejected.
NMSM_HD void bls_agg_prepare_body(uint32_t j, const uint8_t* sigs96, const uint64_t* group_off, const uint8_t* group_ok,
                                  uint32_t* g1, uint32_t* g2, uint8_t* pre_ok) {
  const uint64_t ga = group_off[j], gb = group_off[j + 1];
  bool ok = ga < gb;
  for (uint64_t g = ga; ok && g < gb; g++) ok = group_ok[g] != 0;
  uint32_t sig[48];
  ok = ok && zcash_decode_bls12_381_g2(sigs96 + (size_t)j * 96, sig) == 1;
  ok = ok && bls_in_subgroup<CurveBls381G2Any>(sig);
  const uint64_t last = gb + j;
  for (int k = 0; k < 24; k++) g1[last * 24 + k] = ok ? bls_neg_g1(k) : 0u;
  for (int k = 0; k < 48; k++) g2[last * 48 + k] = ok ? sig[k] : 0u;
  if (!ok)
    for (uint64_t q = ga + j; q < last; q++) {
      for (int k = 0; k < 24; k++) g1[q * 24 + k] = 0u;
      for (int k = 0; k < 48; k++) g2[q * 48 + k] = 0u;
    }
  pre_ok[j] = ok ? 1 : 0;
}

// ---- serial statement (tests/hostemu): the kernels' work in order with tiles of `tile` keys (at most `cap` per group)
// and Miller chunks of `chunk` pairs.  h: the groups' hashed messages (n_groups x 48 words, k_bls_hash_to_g2's
// output); W: (chunk + 2) * BLS_F12_WORDS words.  err[0]: smallest bad key index; err[1..2]: the pair validation's.
inline void bls_agg_serial(uint64_t n_checks, const uint8_t* sigs96, const uint64_t* group_off, const uint32_t* keys,
                           const uint64_t* key_off, const uint32_t* h, uint64_t tile, uint64_t cap, uint64_t chunk,
                           uint32_t* W, uint8_t* out_ok, unsigned int* err) {
  const uint64_t n_groups = group_off[n_checks], n_pairs = n_groups + n_checks;
  std::vector<BlsKeyTile> tiles;
  std::vector<uint32_t> tile_off;
  bls_key_tiles(key_off, n_groups, tile, cap, tiles, tile_off);
  std::vector<uint32_t> partials(tiles.size() * BLS_ACC_WORDS + 1), g1(n_pairs * 24), g2(n_pairs * 48);
  std::vector<uint8_t> tile_bad(tiles.size() + 1), group_ok(n_groups + 1), pre_ok(n_checks);
  std::vector<uint64_t> pair_off(n_checks + 1);
  for (size_t t = 0; t < tiles.size(); t++) {  // k_bls_key_tiles: the lanes, then the shuffle tree
    BlsG1::Acc lane[BLS_KEY_LANES];
    bool bad = false;
    for (uint32_t l = 0; l < BLS_KEY_LANES; l++) lane[l] = bls_key_lane(tiles[t], l, keys, bad, err);
    for (uint32_t d = BLS_KEY_LANES / 2; d; d >>= 1)
      for (uint32_t l = 0; l < d; l++) BlsG1::add(lane[l], lane[l + d]);
    BlsG1::store_acc(partials.data() + t * BLS_ACC_WORDS, lane[0]);
    tile_bad[t] = bad ? 1 : 0;
  }
  for (uint64_t j = 0; j < n_checks; j++)  // k_bls_key_groups
    for (uint64_t g = group_off[j]; g < group_off[j + 1]; g++) {
      bool ok;
      const BlsG1::Acc s = bls_group_sum((uint32_t)g, tile_off.data(), partials.data(), tile_bad.data(), ok);
      bls_group_store((uint32_t)g, (uint32_t)(g + j), ok, s, inv(ok ? s.ZZZ : BlsF::one()), h, g1.data(), g2.data(),
                      group_ok.data());
    }
  for (uint64_t j = 0; j < n_checks; j++) {  // k_bls_agg_prepare
    bls_agg_prepare_body((uint32_t)j, sigs96, group_off, group_ok.data(), g1.data(), g2.data(), pre_ok.data());
    pair_off[j + 1] = group_off[j + 1] + j + 1;
  }
  pair_off[0] = 0;
  pairing_check_serial<BlsPairing>(n_checks, pair_off.data(), g1.data(), g2.data(), pre_ok.data(), chunk, W, out_ok,
                                   err + 1);
}

}  // namespace nmsm
