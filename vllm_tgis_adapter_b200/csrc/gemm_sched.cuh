// The work schedule of the persistent GEMM (gemm_wgmma.cu): which (tile, k-block) units every CTA runs, in which order,
// and how the partials of a split tile are reduced.  One description, host- and device-callable: the kernel's TMA
// producer, its MMA consumers and its split-tile fix-up all read it, and tgis_k_gemm_schedule (test_api.cu) lists it on
// the host, so the tests check exactly what the kernel runs.
#pragma once

namespace tgis {

// Prefill-shaped launches (more than one token tile): "data-parallel waves + stream-K tail".  Linear tile index i
// (see tile_decode) -> the first dp_waves * ncta tiles are whole tiles dealt round-robin, wave w = tiles
// [w * ncta, (w+1) * ncta): at any moment the ncta CTAs work on ONE compact 8 x (ncta / 8) rectangle of (weight tile, token
// tile) pairs, so both operands of a wave stay in L2 (with contiguous per-CTA ranges the CTAs drift apart, the working
// set is every weight tile + every activation tile, far more than L2 holds).  The remaining < ncta tiles are cut
// stream-K style.  Decode-shaped launches have dp_waves = 0.
//
// Decode-shaped launches with at least one tile per CTA (gate_up: 224 tiles, lm_head: 1002) use the same two
// regions in the OPPOSITE order ("sk_first"): every CTA first works through its < 1 tile share of the stream-K region --
// the shared tiles, whose last-arriver fix-up (atomic + L2 round trip + ordered sum) then runs in the epilogue warps
// UNDER the main loop of the following whole tile -- and ends on a whole tile with a direct epilogue.  With the pure
// stream-K cut most CTAs END on a shared tile piece, and the fix-ups (4-6.5 us at 32 tokens, growing with T) are the
// launch's tail.  Same tiles, same split points inside a shared tile's k-range order, same rank-ordered sums.
//
// Invariant of the fix-up: every CTA owns at least one unit of a non-empty stream-K region, so the CTAs whose ranges
// meet a split tile -- c_first .. c_last of split_owners() -- are exactly its contributors, and the last of the
// c_last - c_first + 1 arrivals reduces the tile and puts its counter back to 0.  A stream-K region of fewer units than
// CTAs would leave CTAs with empty ranges inside that span (arrivals that never come: the tile is never written and its
// counter stays raised for the next GEMM), so its tiles are dealt as one more, partial whole-tile wave instead: CTA c <
// dp_extra takes tile dp_waves * ncta + c, and no tile is split.
struct GemmSched {
  int n_tiles, t_tiles, KB, ncta;
  int dp_waves;        // whole-tile waves every CTA runs
  int dp_extra;        // CTAs 0 .. dp_extra - 1 run one more whole tile (wave dp_waves)
  int sk_tile0;        // first tile of the stream-K region
  long long sk_total;  // (tile, k-block) units in the stream-K region: 0, or at least ncta
  bool sk_first;       // stream-K region before the whole-tile waves
  __host__ __device__ GemmSched(int n_tiles_, int t_tiles_, int KB_, int ncta_, bool sk_first_)
      : n_tiles(n_tiles_), t_tiles(t_tiles_), KB(KB_), ncta(ncta_) {
    const int tiles = n_tiles * t_tiles;
    sk_first = sk_first_ && t_tiles == 1 && tiles >= ncta;
    dp_waves = (t_tiles > 1 || sk_first) ? tiles / ncta : 0;
    dp_extra = 0;
    sk_tile0 = dp_waves * ncta;
    sk_total = (long long)(tiles - sk_tile0) * KB;
    if (sk_total > 0 && sk_total < ncta) {
      dp_extra = tiles - sk_tile0;
      sk_tile0 = tiles;
      sk_total = 0;
    }
  }
  __host__ __device__ int whole_tiles(int cta) const { return dp_waves + (cta < dp_extra ? 1 : 0); }
  // CTA cta's contiguous range [sk_begin, sk_end) of the stream-K region's (tile, k-block) space
  __host__ __device__ long long sk_begin(int cta) const { return (sk_total * cta) / ncta; }
  __host__ __device__ long long sk_end(int cta) const { return (sk_total * (cta + 1)) / ncta; }
  // the CTA whose range holds stream-K unit p (sk_total > 0)
  __host__ __device__ int unit_owner(long long p) const { return (int)(((p + 1) * ncta - 1) / sk_total); }
  // the contributors of stream-K tile `tile`, in the order the fix-up sums their partials
  __host__ __device__ void split_owners(int tile, int& c_first, int& c_last) const {
    const long long p0 = (long long)(tile - sk_tile0) * KB;
    c_first = unit_owner(p0);
    c_last = unit_owner(p0 + KB - 1);
  }
  // the workspace slot contributor c wrote its partial of stream-K tile `tile` to: 0 when its range starts in that
  // tile (its first stream-K unit), else 1 (its last)
  __host__ __device__ int partial_slot(int c, int tile) const {
    return (int)(sk_begin(c) / KB) == tile - sk_tile0 ? 0 : 1;
  }
};

// linear tile index -> (weight tile, token tile).  One token tile: identity.  Otherwise blocks of 8 weight tiles, token
// tile next, weight tile fastest: ncta consecutive indices = 8 weight tiles x ncta / 8 token tiles.
__host__ __device__ __forceinline__ void tile_decode(const GemmSched& sc, int tile, int& n_tile, int& t_tile) {
  if (sc.t_tiles == 1) {
    n_tile = tile;
    t_tile = 0;
    return;
  }
  constexpr int NB = 8;
  const int full = NB * sc.t_tiles;
  const int nb = tile / full, rem = tile - nb * full;
  const int left = sc.n_tiles - nb * NB;
  const int nb_n = left < NB ? left : NB;
  t_tile = rem / nb_n;
  n_tile = nb * NB + rem - t_tile * nb_n;
}

// One CTA's units in the order it runs them: its whole tiles (wave w: tile w * ncta + cta), then its stream-K range cut
// at tile boundaries; sk_first: the stream-K range first.  slot = the workspace slot a partial unit's sum goes to.
struct UnitIter {
  long long pos, end;
  int kb_per_tile, wave, waves, cta, ncta, sk_tile0;
  bool first, sk_first;
  __host__ __device__ UnitIter(const GemmSched& sc, int cta_)
      : pos(sc.sk_begin(cta_)), end(sc.sk_end(cta_)), kb_per_tile(sc.KB), wave(0), waves(sc.whole_tiles(cta_)),
        cta(cta_), ncta(sc.ncta), sk_tile0(sc.sk_tile0), first(true), sk_first(sc.sk_first) {}
  // units in total, in k-blocks
  __host__ __device__ long long kblocks() const { return (long long)waves * kb_per_tile + (end - pos); }
  __host__ __device__ bool next(int& tile, int& kb0, int& kb1, int& slot) {
    if (wave < waves && (!sk_first || pos >= end)) {
      tile = wave * ncta + cta;
      kb0 = 0;
      kb1 = kb_per_tile;
      slot = 0;
      ++wave;
      return true;
    }
    if (pos >= end) return false;
    tile = sk_tile0 + (int)(pos / kb_per_tile);
    kb0 = (int)(pos % kb_per_tile);
    long long rem = end - pos;
    int room = kb_per_tile - kb0;
    int take = rem < room ? (int)rem : room;
    kb1 = kb0 + take;
    slot = first ? 0 : 1;
    first = false;
    pos += take;
    return true;
  }
};

}  // namespace tgis
