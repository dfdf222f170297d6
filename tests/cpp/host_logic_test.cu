// Host-side checks of the scheduling helpers the kernels share with the launch code (no GPU needed):
// block selection by residue range (expanded_tc.cuh sel_to_blk / sel_count) -- the exact sample pass,
// the trial screen and the main screen of the screened search must partition the y blocks;
// the dispatch plan of a dense pairwise call (dispatch_plan.cuh) at every boundary of k, n, ldd and the alignments.
#include <cstdio>
#include <set>
#include <string>
#include <vector>
#include "../../raft_b200/csrc/expanded_tc.cuh"
#include "../../raft_b200/csrc/dispatch_plan.cuh"

// launches of the plan as "nkb:acc_mode:resident" words
static std::string plan_text(int post, int64_t m, int64_t n, int64_t k, uintptr_t dist, int64_t ldd)
{
  const b2d::TcStorePlan pl = b2d::tc_store_plan(post, m, n, k, dist, ldd);
  std::string t = pl.tma_store ? "tma" : (pl.vec2 ? "vec2" : "scalar");
  int next = 0;
  for (int i = 0; i < pl.launches; ++i) {
    const b2d::TcStoreLaunch l = b2d::tc_store_launch(pl, i);
    if (l.kb0 != next) return "gap";
    next += l.nkb;
    t += " " + std::to_string(l.nkb) + ":" + std::to_string(l.acc_mode) + ":" + (l.resident ? "res" : "str");
  }
  return next == pl.nkb_total ? t : "short";
}

static int check_plans()
{
  using namespace b2d;
  struct Row { int post; int64_t m, n, k; uintptr_t dist; int64_t ldd; const char* want; };
  const uintptr_t A = 0x1000;   // a 16-byte aligned address
  const Row rows[] = {
    // k: resident | streaming | chunked, and the remainder chunk's kernel
    {POST_CLAMP, 300, 256, 1, A, 256, "tma 1:0:res"},
    {POST_CLAMP, 300, 256, 128, A, 256, "tma 4:0:res"},
    {POST_CLAMP, 300, 256, 129, A, 256, "tma 5:0:str"},
    {POST_CLAMP, 300, 256, 320, A, 256, "tma 10:0:str"},
    {POST_CLAMP, 300, 256, 321, A, 256, "vec2 8:1:str 3:3:res"},
    {POST_CLAMP, 300, 256, 384, A, 256, "vec2 8:1:str 4:3:res"},
    {POST_CLAMP, 300, 256, 385, A, 256, "vec2 8:1:str 5:3:str"},
    {POST_CLAMP, 300, 256, 512, A, 256, "vec2 8:1:str 8:3:str"},
    {POST_CLAMP, 300, 256, 513, A, 256, "vec2 8:1:str 8:2:str 1:3:res"},
    {POST_NONE, 300, 256, 1024, A, 256, "vec2 8:1:str 8:2:str 8:2:str 8:3:str"},
    {POST_POLY, 300, 256, 321, A, 256, "vec2 8:1:str 3:3:res"},
    // the ratio metrics are never chunked
    {POST_JACCARD, 300, 256, 321, A, 256, "tma 11:0:str"},
    {POST_DICE, 300, 256, 1024, A, 256, "tma 32:0:str"},
    // TMA stores: n % 4, ldd % 4, base % 16, and the 32-bit coordinates
    {POST_CLAMP, 300, 252, 64, A, 252, "tma 2:0:res"},
    {POST_CLAMP, 300, 254, 64, A, 256, "vec2 2:0:res"},
    {POST_CLAMP, 300, 253, 64, A, 256, "vec2 2:0:res"},
    {POST_CLAMP, 300, 256, 64, A, 258, "vec2 2:0:res"},
    {POST_CLAMP, 300, 256, 64, A, 257, "scalar 2:0:res"},
    {POST_CLAMP, 300, 256, 64, A + 8, 256, "vec2 2:0:res"},
    {POST_CLAMP, 300, 256, 64, A + 4, 256, "scalar 2:0:res"},
    {POST_CLAMP, 300, 256, 64, A + 12, 256, "scalar 2:0:res"},
    {POST_CLAMP, 300, 256, 160, A + 4, 256, "scalar 5:0:str"},
    {POST_CLAMP, 300, 256, 160, A, 258, "vec2 5:0:str"},
    {POST_CLAMP, 300, 256, 400, A, 257, "scalar 8:1:str 5:3:str"},
    {POST_CLAMP, 300, 256, 400, A + 4, 256, "scalar 8:1:str 5:3:str"},
    {POST_CLAMP, 0x80000000ll, 4, 32, A, 4, "vec2 1:0:res"},
    {POST_CLAMP, 0x7fffffffll, 4, 32, A, 4, "tma 1:0:res"},
  };
  int bad = 0;
  for (const Row& r : rows) {
    const std::string got = plan_text(r.post, r.m, r.n, r.k, r.dist, r.ldd);
    if (got != r.want) {
      std::printf("plan post %d m %lld n %lld k %lld dist %#llx ldd %lld: %s, expected %s\n", r.post, (long long)r.m,
                  (long long)r.n, (long long)r.k, (unsigned long long)r.dist, (long long)r.ldd, got.c_str(), r.want);
      ++bad;
    }
  }
  // every k: the chunks tile the k-blocks, 8 each but the last; the first stores, the last finishes
  for (int64_t k = 1; k <= 4100; ++k) {
    const TcStorePlan pl = tc_store_plan(POST_CLAMP, 10, 10, k, A, 10);
    if (pl.chunked != (k > 320) || pl.launches != (k > 320 ? (tc_k_blocks(k) + 7) / 8 : 1)) ++bad;
    if (plan_text(POST_CLAMP, 10, 10, k, A, 10).size() < 6) ++bad;
    for (int i = 0; i < pl.launches; ++i) {
      const TcStoreLaunch l = tc_store_launch(pl, i);
      const int want = !pl.chunked ? 0 : i == 0 ? 1 : i == pl.launches - 1 ? 3 : 2;
      if (l.acc_mode != want || l.nkb < 1 || (i + 1 < pl.launches && l.nkb != 8) || l.resident != (l.nkb <= 4)) ++bad;
    }
  }
  // unexpanded kernels: 16-byte loads need unit column stride, k % 4, pitch % 4 and a 16-byte aligned base
  struct Vec { int64_t rs, cs, k; uintptr_t base; int want; };
  const Vec vecs[] = {{32, 1, 32, A, 1}, {36, 1, 32, A, 1}, {33, 1, 32, A, 0}, {34, 1, 32, A, 0}, {32, 1, 31, A, 0},
                      {32, 1, 30, A, 0}, {32, 1, 32, A + 4, 0}, {32, 1, 32, A + 8, 0}, {32, 1, 32, A + 16, 1},
                      {1, 32, 32, A, 0}, {4, 1, 4, A, 1}, {8, 1, 5, A, 0}, {1, 1, 1, A, 0}};
  for (const Vec& v : vecs)     // each operand on its own, against one that vectorises and one that does not
    for (int other = 0; other < 2; ++other) {
      const int64_t ors = other ? 32 : 33;
      const UxPlan a = ux_plan(v.rs, v.cs, v.base, ors, 1, A, v.k), b = ux_plan(ors, 1, A, v.rs, v.cs, v.base, v.k);
      const int ov = other && v.k % 4 == 0;
      if (a.vec_x != v.want || a.vec_y != ov || a.tma != (v.want && ov) || b.vec_y != v.want || b.vec_x != ov ||
          b.tma != a.tma) {
        std::printf("ux_plan rs %lld cs %lld k %lld base %#llx != %d\n", (long long)v.rs, (long long)v.cs, (long long)v.k,
                    (unsigned long long)v.base, v.want);
        ++bad;
      }
    }
  return bad;
}

int main()
{
  int bad = check_plans();
  for (int tiles_n = 0; tiles_n <= 300; ++tiles_n)
    for (int S : {2, 3, 8, 32}) {
      std::vector<std::pair<int, int>> ranges = {{0, 1}, {1, 2}, {2, S}};
      if (S == 2) ranges = {{0, 1}, {1, 2}};
      std::set<int> seen;
      for (auto [lo, hi] : ranges) {
        const int cnt = b2d::sel_count(tiles_n, S, lo, hi);
        int prev = -1;
        for (int s = 0; s < cnt; ++s) {
          const int b = b2d::sel_to_blk(s, S, lo, hi);
          if (b <= prev || b < 0 || b >= tiles_n || b % S < lo || b % S >= hi || !seen.insert(b).second) ++bad;
          prev = b;
        }
        // the next index would fall outside
        if (b2d::sel_to_blk(cnt, S, lo, hi) < tiles_n) ++bad;
      }
      if (static_cast<int>(seen.size()) != tiles_n) ++bad;
    }
  // S <= 1: identity
  for (int s = 0; s < 10; ++s) if (b2d::sel_to_blk(s, 0, 0, 0) != s || b2d::sel_count(s, 1, 0, 0) != s) ++bad;
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
