// pf_attn_sched.cu — host-side schedule / mask builders for groups of q tiles (include/pf_b200.h pf_attn_build_pair_* and
// pf_attn_build_group_*): the merged kv-tile lists and the 128 x 128 allow-bit blocks of the partial tiles.  They are part of
// the plan a caller builds once per shape; the sm_90a attention kernel (pf_attn.cu) works from the per-tile schedule and
// evaluates the element mask from seg / time itself, so it reads none of them.
#include <algorithm>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

namespace pf {

// Host: the 128 x 128 allow bits of one (q tile, kv tile) block: bit i of word w of row r = q row qt*128 + r may attend kv column
// kt*128 + 32 w + i  <=>  both inside the sequence, same segment, time_kv <= time_q (mask definition F:318-350).  A plan of the
// 768p run holds a few hundred such blocks; four columns per SSE2 compare (a scalar loop was 0.2 ms per block).
inline void attn_build_mask_block(const int32_t* sg, const int32_t* tm, int seq, int qt, int kt, uint32_t* blk) {
  alignas(16) int32_t sgk[128], tmk[128];
  uint32_t valid[4] = {0u, 0u, 0u, 0u};
  for (int c = 0; c < 128; ++c) {
    const int kv = kt * 128 + c;
    const bool in = kv < seq;
    sgk[c] = in ? sg[kv] : 0;
    tmk[c] = in ? tm[kv] : 0;
    if (in) valid[c >> 5] |= 1u << (c & 31);
  }
  for (int r = 0; r < 128; ++r) {
    const int q = qt * 128 + r;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (q < seq) {
      const int32_t sq = sg[q], tq = tm[q];
#if defined(__SSE2__)
      const __m128i sq4 = _mm_set1_epi32(sq), tq4 = _mm_set1_epi32(tq);
      for (int c = 0; c < 128; c += 4) {
        const __m128i eq = _mm_cmpeq_epi32(_mm_load_si128(reinterpret_cast<const __m128i*>(sgk + c)), sq4);
        const __m128i gt = _mm_cmpgt_epi32(_mm_load_si128(reinterpret_cast<const __m128i*>(tmk + c)), tq4);
        const uint32_t m = static_cast<uint32_t>(_mm_movemask_ps(_mm_castsi128_ps(_mm_andnot_si128(gt, eq))));
        w[c >> 5] |= m << (c & 31);
      }
#else
      for (int c = 0; c < 128; ++c) w[c >> 5] |= static_cast<uint32_t>(sgk[c] == sq && tmk[c] <= tq) << (c & 31);
#endif
      for (int k = 0; k < 4; ++k) w[k] &= valid[k];
    }
    for (int k = 0; k < 4; ++k) blk[r * 4 + k] = w[k];
  }
}

}  // namespace pf

extern "C" int pf_attn_build_pair_schedule(const int32_t* tile_sched, int32_t batch, int32_t seq, int32_t sched_stride,
                                           int32_t* out) {
  using namespace pf;
  PF_REQUIRE(tile_sched && out && batch > 0 && seq > 0, "pf_attn_build_pair_schedule: bad arguments");
  const int q_tiles = (seq + 127) / 128;
  PF_REQUIRE(sched_stride >= 1 + q_tiles, "pf_attn_build_pair_schedule: stride %d too small", sched_stride);
  const int n_pairs = (q_tiles + 1) / 2;
  for (int b = 0; b < batch; ++b) {
    for (int p = 0; p < n_pairs; ++p) {
      const int hi = q_tiles - 1 - 2 * p, lo = hi - 1;
      const int32_t* rh = tile_sched + (static_cast<size_t>(b) * q_tiles + hi) * sched_stride;
      const int32_t* rl = lo >= 0 ? tile_sched + (static_cast<size_t>(b) * q_tiles + lo) * sched_stride : nullptr;
      int32_t* row = out + (static_cast<size_t>(b) * n_pairs + p) * sched_stride;
      const int nh = rh[0], nl = rl ? rl[0] : 0;
      int ih = 0, il = 0, cnt = 0;
      while (ih < nh || il < nl) {
        const int eh = ih < nh ? rh[1 + ih] : 0x7fffffff, el = il < nl ? rl[1 + il] : 0x7fffffff;
        const int kh = eh >> 1, kl = el >> 1;
        const int kt = std::min(kh, kl);
        int fl = 0, fh = 0;
        if (kl == kt) { fl = 1 | ((el & 1) << 1); ++il; }
        if (kh == kt) { fh = 1 | ((eh & 1) << 1); ++ih; }
        row[1 + cnt] = (kt << 4) | fl | (fh << 2);
        ++cnt;
      }
      row[0] = cnt;
      for (int i = 1 + cnt; i < sched_stride; ++i) row[i] = 0;
    }
  }
  return 0;
}

extern "C" int64_t pf_attn_build_pair_masks(const int32_t* seg, const int32_t* time, const int32_t* pair_sched, int32_t batch,
                                            int32_t seq, int32_t sched_stride, int32_t* mask_index, uint32_t* mask_bits,
                                            int64_t capacity_blocks) {
  using namespace pf;
  if (!seg || !time || !pair_sched || !mask_index || batch <= 0 || seq <= 0) {
    set_error("pf_attn_build_pair_masks: bad arguments");
    return -1;
  }
  const int q_tiles = (seq + 127) / 128;
  const int n_pairs = (q_tiles + 1) / 2;
  int64_t blocks = 0;
  for (int b = 0; b < batch; ++b) {
    const int32_t* sg = seg + static_cast<size_t>(b) * seq;
    const int32_t* tm = time + static_cast<size_t>(b) * seq;
    for (int p = 0; p < n_pairs; ++p) {
      const int32_t* row = pair_sched + (static_cast<size_t>(b) * n_pairs + p) * sched_stride;
      int32_t* mi = mask_index + (static_cast<size_t>(b) * n_pairs + p) * 2 * sched_stride;
      for (int i = 0; i < 2 * sched_stride; ++i) mi[i] = -1;
      const int hi = q_tiles - 1 - 2 * p;
      for (int e = 0; e < row[0]; ++e) {
        const int ent = row[1 + e], kt = ent >> 4;
        for (int x = 0; x < 2; ++x) {
          const int fl = (ent >> (2 * x)) & 3;
          if (fl != 3) continue;                       // needs bits only when the tile owns the entry AND is partial
          const int qt = x ? hi : hi - 1;
          if (mask_bits != nullptr && blocks < capacity_blocks) {
            attn_build_mask_block(sg, tm, seq, qt, kt, mask_bits + static_cast<size_t>(blocks) * 128 * 4);
          }
          mi[2 * e + x] = static_cast<int32_t>(blocks);
          ++blocks;
        }
      }
    }
  }
  return blocks;
}

// Host helpers, generalised from the pair forms: group = q tiles per CTA (2 or 3), counted from the END of the sequence (group g
// = tiles q_tiles - group (g + 1) .. q_tiles - 1 - group g; the first group may miss its leading tiles).  Entry =
// (kv_tile << 8) | flags, flags = 2 bits per tile X at bit 2 X (X = 0 the lowest tile): bit0 the tile has an allowed pair in
// this kv tile, bit1 it needs the element mask.
extern "C" int pf_attn_build_group_schedule(const int32_t* tile_sched, int32_t batch, int32_t seq, int32_t sched_stride,
                                            int32_t group, int32_t* out) {
  using namespace pf;
  PF_REQUIRE(tile_sched && out && batch > 0 && seq > 0, "pf_attn_build_group_schedule: bad arguments");
  PF_REQUIRE(group >= 2 && group <= 4, "pf_attn_build_group_schedule: group %d not in [2, 4]", group);
  const int q_tiles = (seq + 127) / 128;
  PF_REQUIRE(sched_stride >= 1 + q_tiles, "pf_attn_build_group_schedule: stride %d too small", sched_stride);
  const int n_groups = (q_tiles + group - 1) / group;
  for (int b = 0; b < batch; ++b) {
    for (int g = 0; g < n_groups; ++g) {
      const int top = q_tiles - 1 - group * g;
      const int32_t* rows[4] = {nullptr, nullptr, nullptr, nullptr};
      int cnt_in[4] = {0, 0, 0, 0}, pos[4] = {0, 0, 0, 0};
      for (int x = 0; x < group; ++x) {
        const int qt = top - (group - 1 - x);
        if (qt >= 0) {
          rows[x] = tile_sched + (static_cast<size_t>(b) * q_tiles + qt) * sched_stride;
          cnt_in[x] = rows[x][0];
        }
      }
      int32_t* row = out + (static_cast<size_t>(b) * n_groups + g) * sched_stride;
      int cnt = 0;
      for (;;) {
        int kt = 0x7fffffff;
        for (int x = 0; x < group; ++x)
          if (pos[x] < cnt_in[x]) kt = std::min(kt, rows[x][1 + pos[x]] >> 1);
        if (kt == 0x7fffffff) break;
        int flags = 0;
        for (int x = 0; x < group; ++x)
          if (pos[x] < cnt_in[x] && (rows[x][1 + pos[x]] >> 1) == kt) {
            flags |= (1 | ((rows[x][1 + pos[x]] & 1) << 1)) << (2 * x);
            ++pos[x];
          }
        row[1 + cnt] = (kt << 8) | flags;
        ++cnt;
      }
      row[0] = cnt;
      for (int i = 1 + cnt; i < sched_stride; ++i) row[i] = 0;
    }
  }
  return 0;
}

extern "C" int64_t pf_attn_build_group_masks(const int32_t* seg, const int32_t* time, const int32_t* group_sched, int32_t batch,
                                             int32_t seq, int32_t sched_stride, int32_t group, int32_t* mask_index,
                                             uint32_t* mask_bits, int64_t capacity_blocks, const int32_t* pair_sched,
                                             const int32_t* pair_mask_index) {
  using namespace pf;
  if (!seg || !time || !group_sched || !mask_index || batch <= 0 || seq <= 0 || group < 2 || group > 4) {
    set_error("pf_attn_build_group_masks: bad arguments");
    return -1;
  }
  const int q_tiles = (seq + 127) / 128;
  const int n_groups = (q_tiles + group - 1) / group;
  const int n_pairs = (q_tiles + 1) / 2;
  const bool share = pair_sched != nullptr && pair_mask_index != nullptr;   // reuse the pair schedule's blocks: same (q tile, kv tile) masks
  int64_t blocks = 0;
  for (int b = 0; b < batch; ++b) {
    const int32_t* sg = seg + static_cast<size_t>(b) * seq;
    const int32_t* tm = time + static_cast<size_t>(b) * seq;
    for (int g = 0; g < n_groups; ++g) {
      const int32_t* row = group_sched + (static_cast<size_t>(b) * n_groups + g) * sched_stride;
      int32_t* mi = mask_index + (static_cast<size_t>(b) * n_groups + g) * group * sched_stride;
      for (int i = 0; i < group * sched_stride; ++i) mi[i] = -1;
      const int top = q_tiles - 1 - group * g;
      for (int e = 0; e < row[0]; ++e) {
        const int ent = row[1 + e], kt = ent >> 8;
        for (int x = 0; x < group; ++x) {
          const int fl = (ent >> (2 * x)) & 3;
          if (fl != 3) continue;                       // needs bits only when the tile owns the entry AND is partial
          const int qt = top - (group - 1 - x);
          if (share) {
            // q tile qt is tile x_p of pair p; its partial (qt, kt) block was numbered by pf_attn_build_pair_masks
            const int p = (q_tiles - 1 - qt) / 2;
            const int x_p = (qt == q_tiles - 1 - 2 * p) ? 1 : 0;
            const int32_t* prow = pair_sched + (static_cast<size_t>(b) * n_pairs + p) * sched_stride;
            int lo = 0, hi = prow[0] - 1, at = -1;
            while (lo <= hi) {
              const int mid = (lo + hi) / 2, k2 = prow[1 + mid] >> 4;
              if (k2 == kt) { at = mid; break; }
              if (k2 < kt) lo = mid + 1; else hi = mid - 1;
            }
            const int32_t blk = at < 0 ? -1 : pair_mask_index[(static_cast<size_t>(b) * n_pairs + p) * 2 * sched_stride + 2 * at + x_p];
            if (blk < 0) {
              set_error("pf_attn_build_group_masks: no pair block for q tile %d, kv tile %d (batch %d)", qt, kt, b);
              return -1;
            }
            mi[group * e + x] = blk;
            blocks = std::max<int64_t>(blocks, static_cast<int64_t>(blk) + 1);
            continue;
          }
          if (mask_bits != nullptr && blocks < capacity_blocks) {
            attn_build_mask_block(sg, tm, seq, qt, kt, mask_bits + static_cast<size_t>(blocks) * 128 * 4);
          }
          mi[group * e + x] = static_cast<int32_t>(blocks);
          ++blocks;
        }
      }
    }
  }
  return blocks;
}

// Host helper: the kv-major transpose of the q-tile schedule (pf_b200.h pf_attn_build_kv_schedule).  Walking the q tiles in
// increasing order appends each q tile to the rows of the kv tiles it names, so every kv row comes out sorted by q tile.
extern "C" int pf_attn_build_kv_schedule(const int32_t* tile_sched, int32_t batch, int32_t seq, int32_t sched_stride,
                                         int32_t* out) {
  using namespace pf;
  PF_REQUIRE(tile_sched && out && batch > 0 && seq > 0, "pf_attn_build_kv_schedule: bad arguments");
  const int tiles = (seq + 127) / 128;
  PF_REQUIRE(sched_stride >= 1 + tiles, "pf_attn_build_kv_schedule: stride %d too small", sched_stride);
  for (int b = 0; b < batch; ++b) {
    int32_t* rows = out + static_cast<size_t>(b) * tiles * sched_stride;
    for (int i = 0; i < tiles * sched_stride; ++i) rows[i] = 0;
    for (int qt = 0; qt < tiles; ++qt) {
      const int32_t* row = tile_sched + (static_cast<size_t>(b) * tiles + qt) * sched_stride;
      PF_REQUIRE(row[0] >= 0 && row[0] <= tiles, "pf_attn_build_kv_schedule: bad count %d (batch %d, q tile %d)", row[0], b, qt);
      for (int e = 0; e < row[0]; ++e) {
        const int kt = row[1 + e] >> 1;
        PF_REQUIRE(kt >= 0 && kt < tiles, "pf_attn_build_kv_schedule: kv tile %d out of range (batch %d, q tile %d)", kt, b, qt);
        int32_t* kr = rows + static_cast<size_t>(kt) * sched_stride;
        // a well-formed q schedule names a kv tile at most once per q row, so a kv row never holds more than `tiles` entries
        PF_REQUIRE(kr[0] < tiles && kr[0] < sched_stride - 1 && (kr[0] == 0 || (kr[kr[0]] >> 1) != qt),
                   "pf_attn_build_kv_schedule: kv tile %d named more than once by a q tile (batch %d, q tile %d)", kt, b, qt);
        kr[1 + kr[0]] = (qt << 1) | (row[1 + e] & 1);
        ++kr[0];
      }
    }
  }
  return 0;
}
