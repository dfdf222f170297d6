// Host-side checks of the masked arg-min kernel's schedule (expanded_tc.cuh EPI_MINLOC_MASKED, masked_nn.cuh); no GPU
// needed.
//   classify          reads "m n G", G group ends and m rows of G 0/1 characters from stdin and prints the class of
//                     every (64-row slab, 128-column half) tile from masked_tile_class, one row of digits per slab
//                     (compared with a numpy restatement by tests/test_masked_nn.py)
//   replay            replays the producer and the two consumer warpgroups of expanded_tc_kernel<kResident,
//                     EPI_MINLOC_MASKED> over random class bytes, resident and streaming, and checks the invariants of
//                     DESIGN.md section 2 K3m: the same stage sequence on both sides, every loaded stage released by
//                     both warpgroups exactly once, the y block of every loaded item waited for and handed back by
//                     both, and nothing for a skipped item.  (Counts and order per warpgroup: that every warp of a
//                     warpgroup waits for each stage and the warpgroup meets before a NONE half's hand-back is the
//                     per-warp side of the protocol, DESIGN.md K3m.)
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>
#include "../../raft_b200/csrc/masked_nn.cuh"

using namespace b2d;

static int classify()
{
  long long m, n, G;
  if (std::scanf("%lld %lld %lld", &m, &n, &G) != 3) return 2;
  std::vector<int> gi(G);
  for (auto& v : gi) if (std::scanf("%d", &v) != 1) return 2;
  const long long W = (m + 31) / 32;
  std::vector<unsigned> bits(static_cast<size_t>(W * G + 1), 0u);
  std::vector<char> row(G + 2);
  for (long long i = 0; i < m; ++i) {
    if (G == 0) continue;
    if (std::scanf("%s", row.data()) != 1) return 2;
    for (long long g = 0; g < G; ++g)
      if (row[g] == '1') bits[(i / 32) * G + g] |= 1u << (i % 32);
  }
  for (long long s = 0; s < (m + 63) / 64; ++s) {
    for (long long h = 0; h < (n + 127) / 128; ++h) std::printf("%d", masked_tile_class(bits.data(), gi.data(), G, m, n, s, h));
    std::printf("\n");
  }
  return 0;
}

// one (tile, k-block) stage load of the producer, and what the consumers did with it
struct Stage {
  int item, mt, h, kb;
  int waits[2] = {0, 0}, releases[2] = {0, 0};
};

static int replay_case(bool resident, int nkb, int tiles_m, int nblocks, int n_last_half, int chunk, int grid, std::mt19937& rng,
                       double p_dead)
{
  int bad = 0;
  // class bytes: a tile is dead with probability p_dead, otherwise random classes per (slab, half); a y block's second
  // half exists only if the block is not the last one or n_last_half
  std::vector<uint8_t> cls(static_cast<size_t>(nblocks) * tiles_m);
  std::uniform_real_distribution<double> u(0, 1);
  for (int nb = 0; nb < nblocks; ++nb)
    for (int mt = 0; mt < tiles_m; ++mt) {
      unsigned b = 0;
      const int nh = (nb < nblocks - 1 || n_last_half) ? 2 : 1;
      if (u(rng) >= p_dead)
        for (int h = 0; h < nh; ++h)
          for (int s = 0; s < 2; ++s) b |= static_cast<unsigned>(rng() % 3) << (2 * (2 * h + s));
      cls[static_cast<size_t>(nb) * tiles_m + mt] = static_cast<uint8_t>(b);
    }
  const int chunks_m = (tiles_m + chunk - 1) / chunk;
  const long long n_items = static_cast<long long>(nblocks) * chunks_m;
  for (int cta = 0; cta < grid; ++cta) {
    // ---- producer (the masked loop of expanded_tc_kernel) ----
    std::vector<Stage> loads;
    std::vector<int> b_loads;   // it_local of every y block load
    uint32_t it_local = 0;
    for (long long item = cta; item < n_items; item += grid) {
      const int n_blk = static_cast<int>(item % nblocks), ch = static_cast<int>(item / nblocks);
      const int mt0 = ch * chunk, mt1 = std::min(mt0 + chunk, tiles_m);
      const int nh  = (n_blk < nblocks - 1 || n_last_half) ? 2 : 1;
      bool b_loaded = false;
      for (int mt = mt0; mt < mt1; ++mt) {
        const unsigned tcls = cls[static_cast<size_t>(n_blk) * tiles_m + mt];
        if (tcls == 0u) continue;
        for (int h = 0; h < (resident ? 1 : nh); ++h) {
          if (!resident && !mask_half_live(tcls, h)) continue;
          for (int kb = 0; kb < nkb; ++kb) {
            if (resident && !b_loaded && kb == 0) b_loads.push_back(static_cast<int>(it_local));
            loads.push_back(Stage{static_cast<int>(item), mt, h, kb});
          }
          b_loaded = true;
        }
      }
      if (b_loaded) ++it_local;
    }
    // ---- consumer warpgroups (the masked paths of the consumer loop) ----
    std::vector<int> a_end(2);
    std::map<int, int> bwait_item[2], brel_item[2];   // it_local -> count
    // liveness of the ring: the producer refills position P - stages as position P, so a warpgroup must have handed
    // P - stages back before it waits for P
    const int stages = resident ? TC_STAGES_RES : TC_STAGES_STR;
    for (int wg = 0; wg < 2; ++wg) {
      std::vector<char> released(loads.size() + 1, 0);
      auto wait_at = [&](uint32_t it) {
        if (it >= static_cast<uint32_t>(stages) && it - stages < released.size() && !released[it - stages]) ++bad;
      };
      auto release_at = [&](uint32_t it) { if (it < released.size()) released[it] = 1; };
      uint32_t a_it = 0, itl = 0;
      for (long long item = cta; item < n_items; item += grid, ++itl) {
        const int n_blk = static_cast<int>(item % nblocks), ch = static_cast<int>(item / nblocks);
        const int mt0 = ch * chunk, mt1 = std::min(mt0 + chunk, tiles_m);
        const int nh  = (n_blk < nblocks - 1 || n_last_half) ? 2 : 1;
        const uint8_t* c = cls.data() + static_cast<size_t>(n_blk) * tiles_m;
        int mt_last = -1;
        for (int mt = mt0; mt < mt1; ++mt) if (c[mt] != 0u) mt_last = mt;
        if (mt_last < 0) { --itl; continue; }
        bool b_first = true;
        for (int mt = mt0; mt < mt1; ++mt) {
          const unsigned tcls = c[mt];
          if (tcls == 0u) continue;
          for (int h = 0; h < nh; ++h) {
            const int hcls = mask_class_of(tcls, h, wg);
            const bool release = !resident || h == nh - 1;
            auto stage_at = [&](uint32_t it) -> Stage* {
              if (it >= loads.size()) { ++bad; return nullptr; }
              Stage* st = &loads[it];
              if (st->item != item || st->mt != mt || (!resident && st->h != h)) ++bad;   // the same stage sequence
              return st;
            };
            if (hcls == MASK_NONE) {
              if (!resident && !mask_half_live(tcls, h)) continue;
              if (release) {
                for (int kb = 0; kb < nkb; ++kb) {   // wait, meet, hand back: one stage at a time
                  wait_at(a_it + kb);
                  release_at(a_it + kb);
                  if (Stage* st = stage_at(a_it + kb)) { st->waits[wg]++; st->releases[wg]++; if (st->kb != kb) ++bad; }
                }
                a_it += nkb;
                if (resident && mt == mt_last) brel_item[wg][static_cast<int>(itl)]++;
              }
              continue;
            }
            for (int kb = 0; kb < nkb; ++kb) {   // live: wait for kb, then hand back kb - 1 (the last after the loop)
              if (resident && b_first && kb == 0) bwait_item[wg][static_cast<int>(itl)]++;
              wait_at(a_it + kb);
              if (release && kb > 0) release_at(a_it + kb - 1);
              if (Stage* st = stage_at(a_it + kb)) { st->waits[wg]++; if (release) st->releases[wg]++; if (st->kb != kb) ++bad; }
            }
            if (release) release_at(a_it + nkb - 1);
            b_first = false;
            if (release) {
              a_it += nkb;
              if (resident && mt == mt_last && h == nh - 1) brel_item[wg][static_cast<int>(itl)]++;
            }
          }
        }
      }
      a_end[wg] = static_cast<int>(a_it);
      if (itl != it_local) ++bad;   // both sides count the same loaded items
    }
    // ---- invariants ----
    for (int wg = 0; wg < 2; ++wg)
      if (a_end[wg] != static_cast<int>(loads.size())) ++bad;   // a_it counts exactly the loaded stages
    for (const Stage& st : loads)
      for (int wg = 0; wg < 2; ++wg)
        if (st.releases[wg] != 1 || st.waits[wg] < 1) ++bad;   // waited for, and released once by each warpgroup
    if (resident)
      for (int it : b_loads)
        for (int wg = 0; wg < 2; ++wg) {
          if (brel_item[wg][it] != 1) ++bad;                    // the y block handed back once per loaded item
          if (bwait_item[wg][it] > 1) ++bad;                    // and waited for at most once (not at all: no MMAs)
        }
    if (resident && static_cast<int>(b_loads.size()) != static_cast<int>(it_local)) ++bad;
  }
  return bad;
}

static int replay()
{
  std::mt19937 rng(12345);
  int bad = 0, cases = 0;
  for (bool resident : {true, false})
    for (int nkb : resident ? std::vector<int>{1, 2, 3, 4} : std::vector<int>{5, 7, 10})
      for (double p_dead : {0.0, 0.5, 0.9, 1.0})
        for (int rep = 0; rep < 6; ++rep) {
          const int tiles_m = 1 + static_cast<int>(rng() % 40), nblocks = 1 + static_cast<int>(rng() % 9);
          const int chunk = 1 + static_cast<int>(rng() % 8), grid = 1 + static_cast<int>(rng() % 5);
          const int b = replay_case(resident, nkb, tiles_m, nblocks, static_cast<int>(rng() % 2), chunk, grid, rng, p_dead);
          if (b) std::printf("case resident=%d nkb=%d tiles_m=%d blocks=%d: %d violations\n", resident, nkb, tiles_m, nblocks, b);
          bad += b;
          ++cases;
        }
  std::printf(bad ? "FAIL %d (%d cases)\n" : "PASS (%d cases)\n", bad ? bad : cases, cases);
  return bad ? 1 : 0;
}

int main(int argc, char** argv)
{
  if (argc > 1 && std::strcmp(argv[1], "classify") == 0) return classify();
  return replay();
}
