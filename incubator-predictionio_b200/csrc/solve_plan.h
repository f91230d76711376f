// solve_plan.h -- which kernels an ALS half-step runs, and with what geometry.  Pure host C++17: no CUDA header and no
// handle, so the rules can be checked without a GPU (tests/test_solve_plan.py compiles this header alone).  pio_als.cu
// reads the switches once per handle (read_solve_switches), plans each side once per ingest (plan_side) and each
// half-step before it launches (plan_half_step), then executes the plan.  Kernels (DESIGN.md 4.1-4.4, 4.8):
//
//   KP 16 / 32       FP32    als_solve_kernel, rows above HEAVY_T cut into PART-rating parts + als_finish_kernel
//   KP 64 default    PAIR    als_solve_pair_kernel, rows above PAIR_SEG_T cut into PAIR_PART-rating parts of the
//                            same kernel + als_finish_pair_kernel; long rows on the auxiliary stream, whole rows in
//                            n_pieces launches on the main stream (each piece's all-gather starts when it is done)
//   KP 64 MMA=1      MMA     mm::als_solve_mma_kernel, rows above HEAVY_T_TC as FP32 parts + als_finish_kernel
//   KP 64 MMA=0      FP32    as KP 16 / 32
//   KP 64 TC=1       WGMMA   tc::als_solve_tc_kernel (+ als_solve_packed_kernel in split mode), long rows as MMA
//   KP 128           LS128   every row in parts: als_solve_kernel on LS128_TILE_ROWS rows' parts at a time, then
//                            als_finish_ls128_kernel on those rows
#pragma once
#include <stdlib.h>

#include <vector>

namespace pio {

constexpr int HEAVY_T = 4096;      // FP32 kernel: rows with more ratings than this are cut into parts (als_finish_kernel)
constexpr int HEAVY_T_TC = 8192;   // same threshold when the mma.sync or wgmma kernel handles the shorter rows
constexpr int PART = 2016;         // ratings per part (a multiple of every CH and of the wgmma stage size 24)
constexpr int PAIR_SEG_T = 1024;   // pair kernel: rows with more ratings than this are cut into parts ...
constexpr int PAIR_PART = 512;     // ... of this many ratings: two-level summation keeps long rows inside the parity bound
constexpr int TC_TILE_ROWS = 1 << 20;    // wgmma split mode: rows whose normal equations are buffered at once (9.1 KB per row)
constexpr int LS128_TILE_ROWS = 32768;   // KP 128: rows per work-list launch (bounds the partial buffer)

// Launch geometry of the kernels (pio_als.cu static_asserts each against the kernel headers)
constexpr int fp32_rows_per_cta(int kp) { return kp <= 32 ? 25 : kp == 64 ? 7 : 2; }   // SolveCfg::NG
constexpr int FINISH_ROWS_PER_CTA = 4;          // als_finish_kernel: one warp per row, 128 threads
constexpr int MMA_ROWS_PER_CTA = 4;             // mm::WARPS
constexpr int TC_ROWS_PER_CTA = 8;              // tc::Api::kPerCta
constexpr int TC_SOLVE_ROWS_PER_CTA = 4;        // tc::Api::kSolveWarps
constexpr int LS128_FINISH_ROWS_PER_CTA = 6;    // FIN128_WARPS
constexpr int PAIR_WARPS_PER_SM = 12;           // als_solve_pair_kernel: __launch_bounds__(32 * WARPS, 12 / WARPS)

// The environment switches of the solve, read once when a handle is created
struct SolveSwitches {
  bool tc = false;             // PIO_ALS_TC=1 (KP 64 only): the wgmma kernel
  double tc_min_deg = 0.0;     // PIO_ALS_TC_MIN_DEG: ... only for sides whose rows average at least this many ratings
  bool tc_split = false;       // PIO_ALS_TC_SPLIT=1: the wgmma kernel only accumulates, a second kernel solves
  bool tc_timing = false;      // PIO_ALS_TC_TIMING: per-warp cycle counters of the wgmma kernel
  bool tc_debug = false;       // PIO_ALS_TC_DEBUG: A/b dump of the last wgmma half-step
  bool mma = true;             // PIO_ALS_MMA=0: the FP32 kernel instead of the mma.sync kernels at KP 64
  bool pair = true;            // PIO_ALS_MMA=1: the round-1 one-warp-per-row mma.sync kernel instead of the pair kernel
  int pair_seg_t = PAIR_SEG_T; // PIO_ALS_SEG_T (> 0)
  int pair_part = PAIR_PART;   // PIO_ALS_PART (>= 8, rounded up to a multiple of 8)
  int pair_warps = 4;          // PIO_ALS_PAIR_WARPS: 1, 2, 4, 6 or 12
  int n_pieces = 1;            // PIO_ALS_PIECES (1..8); default 4 when world_size > 1
};

// env: getenv, or anything shaped like it
template <class Env>
inline SolveSwitches read_solve_switches(Env env, int kp, int world_size) {
  SolveSwitches s;
  const char* v = env("PIO_ALS_TC");
  s.tc = kp == 64 && v && v[0] == '1';
  if ((v = env("PIO_ALS_TC_MIN_DEG"))) s.tc_min_deg = atof(v);
  if ((v = env("PIO_ALS_TC_SPLIT"))) s.tc_split = v[0] == '1';
  s.tc_timing = env("PIO_ALS_TC_TIMING") != nullptr;
  s.tc_debug = env("PIO_ALS_TC_DEBUG") != nullptr;
  if ((v = env("PIO_ALS_MMA"))) {
    s.mma = v[0] != '0';
    s.pair = v[0] != '1';
  }
  if ((v = env("PIO_ALS_SEG_T"))) s.pair_seg_t = atoi(v) > 0 ? atoi(v) : PAIR_SEG_T;
  if ((v = env("PIO_ALS_PART"))) s.pair_part = atoi(v) >= 8 ? (atoi(v) + 7) / 8 * 8 : PAIR_PART;
  if ((v = env("PIO_ALS_PAIR_WARPS"))) {
    const int w = atoi(v);
    if (w == 1 || w == 2 || w == 6 || w == 12) s.pair_warps = w;
  }
  s.n_pieces = world_size > 1 ? 4 : 1;
  if ((v = env("PIO_ALS_PIECES"))) {
    const int n = atoi(v);
    if (n >= 1 && n <= 8) s.n_pieces = n;
  }
  return s;
}

// Kernel of a side's rows at or below its heavy-row threshold.  The values are the labels of pio_als_get_phase_ms;
// LS128 reports itself as FP32 (phase_code).
enum SolveKernel { SOLVE_FP32 = 0, SOLVE_WGMMA = 1, SOLVE_MMA = 2, SOLVE_PAIR = 3, SOLVE_LS128 = 4 };
inline int phase_code(SolveKernel k) { return k == SOLVE_LS128 ? SOLVE_FP32 : k; }

struct SidePlan {
  SolveKernel kernel = SOLVE_FP32;
  int heavy_t = 0;    // rows with more ratings than this are cut into parts
  int part_len = 0;   // ratings per part
};

// One side: n_rows external rows, nnz_global ratings after dedup over all ranks.  Global numbers only, so that every
// rank of a sharded run and the single-GPU run take the same path for the same row.
inline SidePlan plan_side(const SolveSwitches& s, int kp, int n_rows, long long nnz_global) {
  SidePlan p;
  const bool tc = s.tc && kp == 64 && n_rows > 0 && (double)nnz_global / (double)n_rows >= s.tc_min_deg;
  const bool pair = !tc && kp == 64 && s.mma && s.pair;
  p.kernel = kp == 128 ? SOLVE_LS128 : tc ? SOLVE_WGMMA : pair ? SOLVE_PAIR : kp == 64 && s.mma ? SOLVE_MMA : SOLVE_FP32;
  p.heavy_t = kp == 128 ? 0 : pair ? s.pair_seg_t : (tc || (kp == 64 && s.mma)) ? HEAVY_T_TC : HEAVY_T;
  p.part_len = pair ? s.pair_part : PART;
  return p;
}

enum SolveStage {
  STAGE_PARTS,          // partial normal equations of the parts of the heavy rows (pair or FP32 kernel)
  STAGE_FINISH,         // sum the parts of every heavy row in fixed order, then solve (pair or FP32 finish kernel)
  STAGE_LS128_TILE,     // KP 128: partial normal equations of the parts of one tile of rows
  STAGE_LS128_FINISH,   // KP 128: sum and solve the rows of that tile
  STAGE_ROWS,           // rows solved whole (the side's kernel)
  STAGE_TC_SOLVE,       // wgmma split mode: solve the normal equations the wgmma launch before left behind
};

struct SolveLaunch {
  SolveStage stage;
  bool aux;             // on the auxiliary stream (pair path: heavy rows next to the whole rows)
  int row_begin, row_end;   // local rows this launch solves or finishes
  int wl_off, wl_count;     // parts [wl_off, wl_off + wl_count) it reads or writes (work-list stages)
  int grid;
};

struct SolvePlan {
  std::vector<SolveLaunch> launches;   // in launch order; the aux launches come first
  int n_aux = 0;                       // pair path: ev_heavy is recorded on aux after the first n_aux launches
  std::vector<int> piece_after;        // pair path: ev_piece[c] is recorded once piece_after[c] launches are issued
  long long partial_parts = 0;         // part slots of the partial buffer (times the kernel's PART_FLOATS)
};

// One half-step of a side with R local rows, the first n_active of them active and the first n_heavy of those cut into
// n_parts parts (row_part_ptr: host copy of the first part of each heavy row, n_heavy + 1 entries).
inline SolvePlan plan_half_step(const SolveSwitches& s, const SidePlan& sp, int kp, int sm_count, int R, int n_active,
                                int n_heavy, int n_parts, const std::vector<int>& row_part_ptr) {
  SolvePlan p;
  auto add = [&](SolveStage st, bool aux, int r0, int r1, int w0, int nw, int grid) {
    p.launches.push_back(SolveLaunch{st, aux, r0, r1, w0, nw, grid});
  };
  auto cap = [](long long g, long long most) { return (int)(g < most ? g : most); };
  if (sp.kernel == SOLVE_LS128) {
    // every active row is heavy (heavy_t = 0); tiles of rows, per tile one work-list launch over its parts and one
    // finish launch
    for (int r0 = 0; r0 < n_heavy; r0 += LS128_TILE_ROWS) {
      const int r1 = r0 + LS128_TILE_ROWS < n_heavy ? r0 + LS128_TILE_ROWS : n_heavy;
      const int part0 = row_part_ptr[r0], np = row_part_ptr[r1] - part0;
      const int ng = fp32_rows_per_cta(kp);
      add(STAGE_LS128_TILE, false, r0, r1, part0, np, (np + ng - 1) / ng);
      add(STAGE_LS128_FINISH, false, r0, r1, part0, np,
          cap((r1 - r0 + LS128_FINISH_ROWS_PER_CTA - 1) / LS128_FINISH_ROWS_PER_CTA, sm_count));
      if (np > p.partial_parts) p.partial_parts = np;
    }
    return p;
  }
  if (sp.kernel == SOLVE_PAIR) {
    // persistent CTAs of pair_warps warps, two rows (or parts) per warp, twelve warps per SM.  Long rows first, on the
    // auxiliary stream: the whole-row CTAs move in as the part CTAs retire and the finish overlaps the whole rows.
    const int w = s.pair_warps;
    const int max_ctas = (PAIR_WARPS_PER_SM / w) * sm_count;
    auto grid_for = [&](int items) { return cap(((items + 1) / 2 + w - 1) / w, max_ctas); };
    if (n_heavy > 0) {
      add(STAGE_PARTS, true, 0, n_heavy, 0, n_parts, grid_for(n_parts));
      add(STAGE_FINISH, true, 0, n_heavy, 0, n_parts, cap((n_heavy + 1) / 2, (long long)PAIR_WARPS_PER_SM * sm_count));
      p.partial_parts = n_parts;
    }
    p.n_aux = (int)p.launches.size();
    // whole rows, one launch per piece of the local row range
    const int C = s.n_pieces;
    for (int c = 0; c < C; ++c) {
      const long long plo = (long long)R * c / C, phi = (long long)R * (c + 1) / C;
      const int lo = plo > n_heavy ? (int)plo : n_heavy;
      const int hi = phi < n_active ? (int)phi : n_active;
      if (hi > lo) add(STAGE_ROWS, false, lo, hi, 0, 0, grid_for(hi - lo));
      p.piece_after.push_back((int)p.launches.size());
    }
    return p;
  }
  // FP32, MMA, WGMMA: very long rows as FP32 work-list items, then the finish kernel, then the rows solved whole
  const int ng = fp32_rows_per_cta(kp);
  if (n_heavy > 0) {
    add(STAGE_PARTS, false, 0, n_heavy, 0, n_parts, (n_parts + ng - 1) / ng);
    add(STAGE_FINISH, false, 0, n_heavy, 0, n_parts, (n_heavy + FINISH_ROWS_PER_CTA - 1) / FINISH_ROWS_PER_CTA);
    p.partial_parts = n_parts;
  }
  const int nlight = n_active - n_heavy;
  if (nlight <= 0) return p;
  if (sp.kernel == SOLVE_WGMMA) {
    // persistent, one CTA per SM; split mode: tiles of TC_TILE_ROWS rows, each followed by its solve
    const int tile = s.tc_split ? TC_TILE_ROWS : nlight;
    for (int t0 = n_heavy; t0 < n_active; t0 += tile) {
      const int t1 = t0 + tile < n_active ? t0 + tile : n_active;
      add(STAGE_ROWS, false, t0, t1, 0, 0, cap((t1 - t0 + TC_ROWS_PER_CTA - 1) / TC_ROWS_PER_CTA, sm_count));
      if (s.tc_split)
        add(STAGE_TC_SOLVE, false, t0, t1, 0, 0,
            cap((t1 - t0 + TC_SOLVE_ROWS_PER_CTA - 1) / TC_SOLVE_ROWS_PER_CTA, 4ll * sm_count));
    }
  } else {
    const int per = sp.kernel == SOLVE_MMA ? MMA_ROWS_PER_CTA : ng;
    add(STAGE_ROWS, false, n_heavy, n_active, 0, 0, (nlight + per - 1) / per);
  }
  return p;
}

}  // namespace pio
