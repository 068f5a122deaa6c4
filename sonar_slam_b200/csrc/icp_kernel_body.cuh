// The 2-D ICP kernel, icp_kernel (included by icp.cu only, after its helpers and IcpBatch).
//
// One instantiation per CTA size, THREADS with MINB CTAs per SM, so that the register budget follows the launch shape
// (a single __launch_bounds__(512) build capped the 128-thread class at 64 registers and spilled).  The flags are
// instantiations of their own so that the shipped point-to-point kernels keep their code and register allocation:
//   PLANE: errorMinimizer = PointToPlaneErrorMinimizer (sfe_icp_params.minimizer 1);
//   MAP:   the map class -- the target is a map grid in global memory, read through `mp` (map_build): no set-up per
//          problem, 32-bit target positions, and shared memory holds IcpShared and the source arrays only.  The in-CTA
//          class ignores `mp`; it comes after `b`, so `b` has the same parameter offsets in both classes;
//   FILT:  the batch runs sfe_icp_filters -- the MinDist / MedianDist outlier filters and the min_points gate on the
//          clouds before the data filters;
//   GSRC:  the global-source class (MAP only) -- sources too large for shared memory: the per-source-point arrays
//          (reading .. order) sit in the CTA's slice of global workspace (b.src_ws), with 32-bit entries in order[];
//          shared memory holds IcpShared and, PLANE, seq_sum9_warp's scratch;
//   ROBUST: (FILT only) the batch runs a RobustOutlierFilter (b.robust): the keep pass (3c) multiplies the 0 / 1 weights
//          by the robust weight and parks it in dist[], which is dead until the next search; the minimisers' sums
//          weight their terms by it.  PLANE: seq_sum9_warp's scratch then gets its own 2.5 KB;
//   GNRM:  (PLANE, FILT, in-CTA class only) the target's normals are given (b.given_nrm, laid out as the targets'
//          points: a SamplingSurfaceNormalDataPointsFilter's) and gathered to the sorted positions instead of computed.
//          The map classes need no instantiation of their own: map_build gathers them (MapArgs::nrm).
// The body is written in the kernel itself: behind a device-function wrapper the shipped instantiations compiled with
// larger stack frames.
template <int THREADS, int MINB, bool PLANE, bool MAP, bool FILT, bool GSRC, bool ROBUST = false, bool GNRM = false>
__global__ void __launch_bounds__(THREADS, MINB) icp_kernel(const IcpBatch b, const MapArgs mp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // layout: [IcpShared][sorted float2 nt_max][cells u32][reading float2 ns_max][dist f32 ns_max][match Pos ns_max]
  //         [prev Pos ns_max][qstate u8 ns_max][slack f32 ns_max][order Ord ns_max]   (MAP: no sorted, no cells)
  // GSRC: [IcpShared][seq_sum9_warp scratch] in shared memory, [reading .. order] at the start of the CTA's slice.
  // CTA sizes: the reference mean takes warps 0 and 1 (one per coordinate); the per-warp partials (wred, tot, red) and
  // block_total's final read (one lane per warp) hold at most 16 warps; the rest of the body loops over blockDim.x.
  static_assert(THREADS % 32 == 0 && THREADS >= 64 && THREADS <= 512, "icp_kernel: 2 to 16 warps per CTA");
  static_assert(MAP || !GSRC, "icp_kernel: the global-source class reads its targets as map grids");
  static_assert(FILT || !ROBUST, "icp_kernel: the robust filter runs in the FILT instantiations");
  static_assert(!GNRM || (PLANE && FILT && !MAP), "icp_kernel: given normals are point-to-plane, FILT and in-CTA only");
  using Pos = std::conditional_t<MAP, int, uint16_t>;   // a target point's sorted position
  using Ord = std::conditional_t<GSRC, int, uint16_t>;  // a source point's index
  constexpr int NONE = MAP ? -1 : 0xffff;                // "no match"
  IcpShared &sh = *reinterpret_cast<IcpShared *>(smem_raw);
  size_t off = (sizeof(IcpShared) + 15) & ~size_t(15);
  float2 *sorted = reinterpret_cast<float2 *>(smem_raw + off);  // MAP: set to the slot's points below
  if constexpr (!MAP) off += sizeof(float2) * (size_t)b.nt_max;
  uint32_t *cells = reinterpret_cast<uint32_t *>(smem_raw + off);
  if constexpr (!MAP) off += sizeof(uint32_t) * (size_t)((b.max_cells + 2) / 2 + 1);
  off = (off + 7) & ~size_t(7);
  unsigned char *src_base = smem_raw;  // where the per-source-point arrays start (GSRC: the CTA's slice, from 0)
  const size_t shared_end = off;
  if constexpr (GSRC) src_base = b.src_ws + (size_t)blockIdx.x * b.src_ws_stride, off = 0;
  float2 *reading = reinterpret_cast<float2 *>(src_base + off);
  off += sizeof(float2) * (size_t)b.ns_max;
  float *dist = reinterpret_cast<float *>(src_base + off);
  off += sizeof(float) * (size_t)b.ns_max;
  Pos *match = reinterpret_cast<Pos *>(src_base + off);
  off += sizeof(Pos) * (size_t)b.ns_max;
  Pos *prev = reinterpret_cast<Pos *>(src_base + off);  // NN of the previous iteration (search seed)
  off += sizeof(Pos) * (size_t)b.ns_max;
  uint8_t *qstate = reinterpret_cast<uint8_t *>(src_base + off);
  off += ((size_t)b.ns_max + 3) & ~size_t(3);
  // certified-match margin per source point (metres): every target point other than prev[i] is farther from the
  // point's current position than (distance to prev[i]) as long as that distance stays below slack[i]
  float *slack = reinterpret_cast<float *>(src_base + off);
  off += sizeof(float) * (size_t)b.ns_max;
  // processing order of the source points in the search passes: sorted by a coarse cell of the target grid, so that
  // the lanes of a warp look at neighbouring cells (similar amounts of work, the same shared-memory lines); results
  // are stored by point index and the sums run in point order, so the order is invisible in the results
  Ord *order = reinterpret_cast<Ord *>(src_base + off);
  if (b.use_order) off += sizeof(Ord) * (size_t)b.ns_max;
  off = (off + 15) & ~size_t(15);
  if constexpr (GSRC) off = (shared_end + 15) & ~size_t(15);  // (the scratch below stays in shared memory)
  (void)shared_end;
  // PLANE only: 640 floats for seq_sum9_warp.  dist[] is dead between the weights (3c) and the next iteration's
  // search, which rewrites all of it: launches with room for 640 source points (the front end's small class is
  // exactly that; 2 000 x 20 000 points leave nothing to spare at all) park the scratch there, smaller ones get
  // their own 2.5 KB.  GSRC: always its own, in shared memory.
  float *pl_scratch = !GSRC && !ROBUST && b.ns_max >= ICP_PLANE_SCRATCH ? dist : reinterpret_cast<float *>(smem_raw + off);
  (void)pl_scratch;

  const int tid = threadIdx.x, nthr = blockDim.x;
  ICP_PH_DECL
  int red_phase = 0, tot_phase = 0, sel_pass = 0;  // rotation counters of the one-barrier reductions (CTA-uniform)
  for (int h = threadIdx.x; h < 3 * 256; h += blockDim.x) (&sh.hist[0][0])[h] = 0;
  // Problems that allow one CTA per SM (config 3: ~200 KB of shared memory) are launched one CTA per problem, not
  // as persistent CTAs: problems of unequal length (checker mode: 4-40 iterations) balance themselves, and SMs
  // free up every few milliseconds so that concurrent NCCL send/recv kernels (the config-5 scatter) get scheduled.
  // The per-CTA global workspace is then indexed by the SM the CTA runs on.
  const unsigned slot = b.slot_by_smid ? icp_smid() : blockIdx.x;
  if (b.slot_by_smid && slot >= ICP_SM_SLOTS) __trap();
  uint16_t *orig = MAP ? nullptr : b.orig_ws + (size_t)slot * b.nt_max;
  const sfe_icp_params prm = b.prm;
  const float max_d2 = __fmul_rn(prm.matcher_max_dist, prm.matcher_max_dist);
  const float out_d2 = (prm.flags & 1) ? prm.outlier_max_dist : __fmul_rn(prm.outlier_max_dist, prm.outlier_max_dist);
  const int smooth = min(prm.smooth_length, ICP_HIST - 1);
  // Default: every sum over points is a sequential float32 sum in point order, as in oracle/icp_ref.c -- results
  // are bit-identical to the oracle.  flags bit 1: float32 terms accumulated in float64 (order-independent,
  // ~1e-4 closer to exact arithmetic; deviates from the oracle by up to ~2e-3 m on
  // ill-conditioned scans because the float32-sequential sums themselves are that noisy).
  const bool seq = (prm.flags & 2) == 0;

  // Persistent CTAs take problems from a work counter: problems differ in length (cloud sizes, early exits), and with
  // a static share the batch ends when the CTAs that drew the most work finish.  Problem p's results do not depend
  // on the CTA that solves it.  The index is broadcast through sh.status, which thread 0 rewrites only after the
  // next problem's first barrier.  With a class list (always from a counter) the work items are that list's entries.
  for (int p = icp_work_item(b, blockIdx.x); p < b.P;
       p = b.next ? icp_work_item(b, next_work_item(b.next, &sh.status)) : p + (int)gridDim.x) {
    const int si = b.src_id ? b.src_id[p] : p, ti = b.tgt_id ? b.tgt_id[p] : p;
    const float *src = b.src_pts + 2 * (size_t)b.src_off[si];
    const int ns = b.src_cnt ? b.src_cnt[si] : b.src_off[si + 1] - b.src_off[si];
    const float *tgt = b.tgt_pts + 2 * (size_t)b.tgt_off[ti];
    const int nt = b.tgt_cnt ? b.tgt_cnt[ti] : b.tgt_off[ti + 1] - b.tgt_off[ti];
    const float *guess = b.guess + 9 * (size_t)p;
    if (!icp_takes(b.box, ns, nt)) continue;  // another launch's
    __syncthreads();  // previous problem fully retired before shared state is reused

    // ---- admission checks (thread 0), failure leaves T = guess
    if (tid == 0) {
      int st = ICP_OK;
      if (ns > b.ns_max || nt > b.nt_max || (b.raw_cnt && b.raw_cnt[si] > b.raw_cap)) st = ICP_TOO_LARGE;
      else if (!FILT && (ns < b.min_points || nt < b.min_points)) st = ICP_SKIPPED;
      else if (FILT && ((b.gate_src_cnt ? b.gate_src_cnt[si] : ns) < b.min_points ||
                        (b.gate_tgt_cnt ? b.gate_tgt_cnt[ti] : nt) < b.min_points))
        st = ICP_SKIPPED;  // (the clouds before the data filters, as the SLAM node counts them before ICP)
      else if (nt <= 0) st = ICP_EMPTY_REF;
      const float det = __fsub_rn(__fmul_rn(guess[0], guess[4]), __fmul_rn(guess[1], guess[3]));
      if (st == ICP_OK && (!(fabsf(__fsub_rn(1.0f, det)) <= 0.001f))) st = ICP_NOT_RIGID;
      sh.status = st;
      sh.count = 0, sh.inliers = 0;
    }
    __syncthreads();
    if (sh.status != ICP_OK) {
      if (tid < 9) b.T_out[9 * (size_t)p + tid] = guess[tid];
      if (tid == 0) b.iters[p] = 0, b.inliers[p] = 0, b.status[p] = sh.status;
      continue;
    }

    ICP_PH_START();
    if constexpr (MAP) {  // ---- 1. (map class) mean and bounding box were computed once for the whole call
      const MapGrid &mg = mp.grid[mp.slot[p]];
      if (tid == 0) {
        sh.mean[0] = mg.mean[0], sh.mean[1] = mg.mean[1];
#pragma unroll
        for (int k = 0; k < 4; ++k) sh.bbox[k] = mg.bbox[k];
        sh.cnx = 0;  // no coarse occupancy map: pass B searches instead (DESIGN section 3)
      }
      __syncthreads();
    } else
    // ---- 1. mean of the reference, bounding box of the centred reference
    {
      float mx, my;
      if (seq) {
        if (tid < 64) {  // warps 0 and 1: x and y
          const float sum = seq_sum_warp_global(tgt + (tid >> 5), nt, 2);
          if ((tid & 31) == 0) sh.seq[tid >> 5] = __fdiv_rn(sum, (float)nt);
        }
        __syncthreads();
        mx = sh.seq[0], my = sh.seq[1];
      } else {
        double s[2] = {0.0, 0.0}, tot[2];
        for (int i = tid; i < nt; i += nthr) s[0] += (double)tgt[2 * i], s[1] += (double)tgt[2 * i + 1];
        block_sum<2>(s, sh.red, red_phase, tot);
        mx = (float)(tot[0] / (double)nt), my = (float)(tot[1] / (double)nt);
      }
      float mn_x = INFINITY, mn_y = INFINITY, mxx = -INFINITY, mxy = -INFINITY;
      for (int i = tid; i < nt; i += nthr) {
        const float x = tgt[2 * i] - mx, y = tgt[2 * i + 1] - my;
        mn_x = fminf(mn_x, x), mxx = fmaxf(mxx, x), mn_y = fminf(mn_y, y), mxy = fmaxf(mxy, y);
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        mn_x = fminf(mn_x, __shfl_xor_sync(0xffffffffu, mn_x, d));
        mn_y = fminf(mn_y, __shfl_xor_sync(0xffffffffu, mn_y, d));
        mxx = fmaxf(mxx, __shfl_xor_sync(0xffffffffu, mxx, d));
        mxy = fmaxf(mxy, __shfl_xor_sync(0xffffffffu, mxy, d));
      }
      float *fr = sh.wred;
      if ((tid & 31) == 0) {
        fr[(tid >> 5) * 4 + 0] = mn_x, fr[(tid >> 5) * 4 + 1] = mn_y;
        fr[(tid >> 5) * 4 + 2] = mxx, fr[(tid >> 5) * 4 + 3] = mxy;
      }
      __syncthreads();
      if (tid == 0) {
        float a = INFINITY, bb = INFINITY, c = -INFINITY, d = -INFINITY;
        for (int w = 0; w < (nthr >> 5); ++w) {
          a = fminf(a, fr[w * 4 + 0]), bb = fminf(bb, fr[w * 4 + 1]);
          c = fmaxf(c, fr[w * 4 + 2]), d = fmaxf(d, fr[w * 4 + 3]);
        }
        sh.bbox[0] = a, sh.bbox[1] = bb, sh.bbox[2] = c, sh.bbox[3] = d;
        sh.mean[0] = mx, sh.mean[1] = my;
      }
      __syncthreads();
    }
    const float mx = sh.mean[0], my = sh.mean[1];
    std::conditional_t<MAP, MapGridView, GridView> g;
    if constexpr (MAP) {  // the grid too (map_build)
      g = map_grid_view(mp, mp.slot[p]);
      sorted = const_cast<float2 *>(mp.pts);
    } else {
    grid_geometry(nt, sh.bbox[0], sh.bbox[1], sh.bbox[2], sh.bbox[3], 0.05f, g, b.max_cells, b.cell_scale);
    grid_build(tgt, 2, nt, mx, my, g, sorted, cells, orig, sh.scan);
    // coarse occupancy: which 8x8 blocks of cells hold any point (answers "is anything within maxDist?"
    // for far-away source points without walking the fine grid)
    {
      const int cnx = (g.nx + ICP_COARSE - 1) / ICP_COARSE, cny = (g.ny + ICP_COARSE - 1) / ICP_COARSE;
      if (tid == 0) sh.cnx = cnx, sh.cny = cny;
      for (int w = tid; w < ICP_COARSE_WORDS; w += nthr) sh.coarse[w] = 0;
      __syncthreads();
      if (cnx * cny <= ICP_COARSE_WORDS * 32) {
        for (int cc = tid; cc < cnx * cny; cc += nthr) {
          const int ccy = cc / cnx, ccx = cc - ccy * cnx;
          bool occ = false;
          for (int y = ccy * ICP_COARSE; y < min((ccy + 1) * ICP_COARSE, g.ny) && !occ; ++y) {
            const int xa = ccx * ICP_COARSE, xb = min((ccx + 1) * ICP_COARSE, g.nx);
            occ = g.cstart[y * g.nx + xb] > g.cstart[y * g.nx + xa];
          }
          if (occ) atomicOr(&sh.coarse[cc >> 5], 1u << (cc & 31));
        }
      } else if (tid == 0) {
        sh.cnx = 0;  // too many coarse cells: the test is skipped
      }
      __syncthreads();
    }
    }  // !MAP

    // ---- 1b. point-to-plane: normals of the (centred) target, one thread per sorted position, kept in global
    // memory (8 B per target point; the iterations gather them through L2)
    float2 *nrm = nullptr;
    if constexpr (PLANE && MAP) {
      nrm = const_cast<float2 *>(mp.nrm);  // computed once per target by map_build
    } else if constexpr (GNRM) {
      nrm = b.nrm_ws + (size_t)slot * b.nt_max;
      const float2 *given = b.given_nrm + b.tgt_off[ti];
      for (int j = tid; j < nt; j += nthr) nrm[j] = given[orig[j]];
    } else if constexpr (PLANE) {
      nrm = b.nrm_ws + (size_t)slot * b.nt_max;
      const int knn = min(max(prm.normals_knn, 1), GRID_KNN_MAX);
      // best-knn list per thread: the per-source arrays (reading .. slack) are idle until step 2
      unsigned char *scr = reinterpret_cast<unsigned char *>(reading);
      const size_t scr_bytes = (size_t)(reinterpret_cast<unsigned char *>(slack + b.ns_max) - scr);
      if (scr_bytes >= (size_t)nthr * knn * 6) {
        float *bd = reinterpret_cast<float *>(scr) + tid;
        uint16_t *bi = reinterpret_cast<uint16_t *>(scr + sizeof(float) * (size_t)nthr * knn) + tid;
        for (int j = tid; j < nt; j += nthr) nrm[j] = grid_surface_normal(g, j, knn, bd, bi, nthr);
      } else {
        float bd[GRID_KNN_MAX];
        uint16_t bi[GRID_KNN_MAX];
        for (int j = tid; j < nt; j += nthr) nrm[j] = grid_surface_normal(g, j, knn, bd, bi, 1);
      }
      // (published to the CTA, and the scratch released, by the barriers of step 2)
    }

    // ---- 2. reading into the centred frame; T_iter = I; checker history
    if (tid == 0) {
      const float Tinv[9] = {1.f, 0.f, -mx, 0.f, 1.f, -my, 0.f, 0.f, 1.f};
      float T0[9];
      mat3_mul_rn(Tinv, guess, T0);
#pragma unroll
      for (int i = 0; i < 9; ++i) sh.T0[i] = T0[i], sh.Ti[i] = sh.Tprev[i] = (i % 4 == 0) ? 1.f : 0.f;
      rot_to_quat(sh.Ti, sh.hq_w[0], sh.hq_z[0]);
      sh.ht_x[0] = 0.f, sh.ht_y[0] = 0.f;
      sh.hn = 1;
      sh.iterate = 1;
      sh.todo_n = 0;
    }
    __syncthreads();
    for (int i = tid; i < ns; i += nthr) {
      reading[i] = apply_T(sh.T0, src[2 * i], src[2 * i + 1]);
      prev[i] = NONE;
      slack[i] = 0.f;
    }
    __syncthreads();
    if (b.use_order) {  // counting sort of the point indices by a 16 x 16 bucket grid over the target's bounding box.  Counters: the
       // radix-select histogram that the next selection pass neither fills nor expects to be clear (pass p fills
       // hist[p % 3] and clears hist[(p + 1) % 3]; hist[(p + 2) % 3] is cleared by pass p + 1 before it is used)
      int *cnt = sh.hist[(sel_pass + 2) % 3];
      for (int h = tid; h < 256; h += nthr) cnt[h] = 0;
      __syncthreads();
      const float bw = fmaxf(sh.bbox[2] - sh.bbox[0], 1e-6f) * (1.f / 16.f), bh = fmaxf(sh.bbox[3] - sh.bbox[1], 1e-6f) * (1.f / 16.f);
      auto bucket = [&](int i) {
        const int bx = min(max((int)((reading[i].x - sh.bbox[0]) / bw), 0), 15);
        const int by = min(max((int)((reading[i].y - sh.bbox[1]) / bh), 0), 15);
        return by * 16 + bx;
      };
      for (int i = tid; i < ns; i += nthr) atomicAdd(&cnt[bucket(i)], 1);
      __syncthreads();
      if (tid < 32) {  // exclusive scan of the 256 counters by one warp (8 per lane)
        int c[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) c[j] = cnt[tid * 8 + j], sum += c[j];
        int incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, d);
          if (tid >= d) incl += t;
        }
        int run = incl - sum;
#pragma unroll
        for (int j = 0; j < 8; ++j) cnt[tid * 8 + j] = run, run += c[j];
      }
      __syncthreads();
      for (int i = tid; i < ns; i += nthr) order[atomicAdd(&cnt[bucket(i)], 1)] = (Ord)i;
      __syncthreads();
    }

    ICP_PH_MARK(0);
    // ---- 3. iterations
    while (true) {
      float Ti[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) Ti[i] = sh.Ti[i];
      // 3a. match.  Exact nearest neighbours are only needed for the pairs that can get a non-zero weight:
      //   pass A  every source point scans its 3x3 block of cells: that either settles its nearest neighbour
      //           or at least yields a candidate, i.e. an UPPER bound on its NN distance;
      //   pass B  points without a candidate inside maxDist learn whether ANY target point lies within
      //           maxDist (they then count as "finite" in the trimmed quantile) -- from the coarse
      //           occupancy grid when that is conclusive, else from a search that stops at the first hit;
      //   pass C  with n_finite known, kk = floor(n_finite * ratio).  The kk-th smallest of the upper bounds
      //           (maxDist^2 for a finite point without candidate) bounds the kk-th smallest true distance
      //           from above: call it U.  An unsettled point whose search proves "farther than U" has weight
      //           0 and needs no exact distance.  Results are identical to an exhaustive search (same
      //           quantile element, same kept pairs); the far outliers of a scan stop costing O(area).
      int n_fin = 0, total_fin = -1;
      const bool small = ns <= b.small_mult * nthr && nt <= 4096;  // few, cheap searches: one exact pass, no pruning
      // Certified matches.  A search that scans at least the 3x3 block also yields a lower bound L on the distance
      // from the point to every target point OTHER than its match (grid.cuh: nn_query_certified).  The point then
      // moves a little every iteration; by the triangle inequality every other target point stays farther than
      // L - (path length since).  slack[i] holds that margin, shrunk by safety terms far above float32 rounding:
      // while the distance to the old match is below it, the old match is the unique nearest neighbour -- the
      // answer an exhaustive search would give, ties impossible -- and costs one distance instead of a search.
      // Used for the small problems of the front end (window submaps thinned to 0.5 m: runner-ups are decimetres
      // away and a certificate lasts several iterations).
      float Tp[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) Tp[i] = sh.Tprev[i];
      auto certified = [&](int i, const float2 q, int seed, float &d2_out, float &step) -> bool {
        const float2 qo = apply_T(Tp, reading[i].x, reading[i].y);
        step = sqrtf(dist2_rn(q.x - qo.x, q.y - qo.y));
        const float sl = slack[i] - (step * 1.00001f + 2e-5f);
        slack[i] = sl;
        const float2 t = sorted[seed];
        const float d2 = dist2_rn(q.x - t.x, q.y - t.y);
        d2_out = d2;
        return d2 <= max_d2 && sqrtf(d2) * 1.00001f + 1e-4f < sl;
      };
      auto certify = [&](int i, float lb2) {  // margin after a certifying search
        slack[i] = lb2 < 3.0e38f ? sqrtf(lb2) * 0.99999f - 1e-4f : 3.0e38f;
      };
      // certificate size: a few of the point's steps (steps shrink as the scan converges), a fraction of a cell at most
      auto margin_for = [&](float step) { return fminf(fmaxf(b.margin_mult * step, 0.01f * g.cell), 0.35f * g.cell); };
      if (small) {
        if constexpr (THREADS <= 256) {
          // Two halves, so that the lanes of a warp stay on one code path.  First every point tests its certificate
          // (one distance; points without a seed search at once: that is the first iteration, all lanes together);
          // the points whose certificate failed are only LISTED -- in match[], which the weights (3c) rewrite from
          // prev[], with the counter in todo_n (zeroed by the single-thread step of the previous iteration).  Then the
          // list is searched densely.  In one loop the re-search ran with 2.4 of 32 lanes active and took 25 % of this
          // kernel's warp instructions on the front end's problems (tools/ncu_call_sites.py).
          uint16_t *todo = reinterpret_cast<uint16_t *>(match);
          for (int base = 0; base < ns; base += nthr) {
            const int ii = base + tid;
            bool later = false;
            int i = 0;
            if (ii < ns) {
              i = b.use_order ? order[ii] : ii;
              const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
              const int seed = prev[i];
              float d2s, step, lb2;
              if (seed == NONE) {
                const NNResult r = nn_query_certified(g, q.x, q.y, max_d2, &lb2);
                certify(i, lb2);
                dist[i] = r.d2;
                prev[i] = r.pos >= 0 ? (Pos)r.pos : (Pos)NONE;
                n_fin += r.pos >= 0;
              } else if (certified(i, q, seed, d2s, step)) {
                dist[i] = d2s;  // prev[i] stays
                n_fin += 1;
              } else {
                later = true;
              }
            }
            const unsigned m = __ballot_sync(0xffffffffu, later);
            if (m) {  // one shared-memory atomic per warp
              const int lane = tid & 31, lead = __ffs(m) - 1;
              int at = 0;
              if (lane == lead) at = atomicAdd(&sh.todo_n, __popc(m));
              at = __shfl_sync(0xffffffffu, at, lead);
              if (later) todo[at + __popc(m & ((1u << lane) - 1u))] = (uint16_t)i;
            }
          }
          __syncthreads();
          const int n_todo = sh.todo_n;
          for (int k = tid; k < n_todo; k += nthr) {
            const int i = todo[k];
            const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
            const float2 qo = apply_T(Tp, reading[i].x, reading[i].y);
            const float step = sqrtf(dist2_rn(q.x - qo.x, q.y - qo.y));
            float lb2;
            const NNResult r = nn_query_seeded_certified(g, q.x, q.y, max_d2, prev[i], margin_for(step), &lb2);
            certify(i, lb2);
            dist[i] = r.d2;
            prev[i] = r.pos >= 0 ? (Pos)r.pos : (Pos)NONE;
            n_fin += r.pos >= 0;
          }
          // the matches are prev[] now (3c reads them there); this barrier also publishes prev[] and dist[]
          total_fin = block_total(n_fin, &sh.tot[0][0], tot_phase);
        } else {
          // (512-thread CTAs rarely see a problem this small: the single loop is kept there, and with it the code of the
          //  config-3 instantiation)
          for (int ii = tid; ii < ns; ii += nthr) {
            const int i = b.use_order ? order[ii] : ii;
            const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
            const int seed = prev[i];
            NNResult r;
            float d2s, step, lb2;
            if (seed == NONE) {
              r = nn_query_certified(g, q.x, q.y, max_d2, &lb2);
              certify(i, lb2);
            } else if (certified(i, q, seed, d2s, step)) {
              r.d2 = d2s, r.pos = seed, r.tie = 0;
            } else {
              r = nn_query_seeded_certified(g, q.x, q.y, max_d2, seed, margin_for(step), &lb2);
              certify(i, lb2);
            }
            dist[i] = r.d2;
            match[i] = prev[i] = r.pos >= 0 ? (Pos)r.pos : (Pos)NONE;
            n_fin += r.pos >= 0;
          }
        }
      }
      const float stop_a = (0.999f * g.cell) * (0.999f * g.cell);
      for (int ii = tid; ii < ns && !small; ii += nthr) {
        const int i = b.use_order ? order[ii] : ii;
        const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
        NNResult r;
        r.d2 = INFINITY, r.pos = -1, r.tie = 0;
        int exact;
        const int seed = prev[i];
        // (no certificates here: a 20 000-point target puts the runner-up a centimetre from the match, so a
        // certificate rarely outlives an iteration, and checking it costs more than it saves)
        const float2 ts = sorted[seed != NONE ? seed : 0];
        if (seed != NONE && dist2_rn(q.x - ts.x, q.y - ts.y) <= stop_a) {
          r = nn_query_seeded(g, q.x, q.y, max_d2, seed);  // last iteration's match is still close: settle it now
          exact = 1;
        } else {
          exact = nn_search(g, q.x, q.y, max_d2, stop_a, -1, r);  // own cell, then at most the 3x3 block
        }
        if (exact) prev[i] = (r.pos >= 0 && r.d2 <= max_d2) ? (Pos)r.pos : (Pos)NONE;
        const bool fin = r.pos >= 0 && r.d2 <= max_d2;
        dist[i] = fin ? r.d2 : INFINITY;
        match[i] = fin ? (Pos)r.pos : (Pos)NONE;
        qstate[i] = (exact ? 1 : 0) | (fin ? 2 : 0) | ((fin || exact) ? 4 : 0);  // settled / finite / known
        n_fin += fin;
      }
      // pass B: finiteness of the points that have no candidate yet
      for (int ii = tid; ii < ns && !small; ii += nthr) {
        const int i = b.use_order ? order[ii] : ii;
        if (qstate[i] & 4) continue;
        const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
        int verdict = -1;  // 1 finite, 0 not, -1 unknown
        if (sh.cnx > 0) {
          const float C = g.cell * (float)ICP_COARSE, rad = prm.matcher_max_dist;
          // the window is clamped to [0, n] / [-1, n - 1] in float before the int conversion: a maxDist of inf or
          // 1e9 m would otherwise saturate and overflow it into an empty window ("nothing within maxDist")
          auto lo = [&](float v, int n) { return (int)fminf(fmaxf(floorf(v / C) - 1.f, 0.f), (float)n); };
          auto hi = [&](float v, int n) { return (int)fminf(fmaxf(floorf(v / C) + 1.f, -1.f), (float)(n - 1)); };
          const int xa = lo(q.x - rad - g.ox, sh.cnx), xb = hi(q.x + rad - g.ox, sh.cnx);
          const int ya = lo(q.y - rad - g.oy, sh.cny), yb = hi(q.y + rad - g.oy, sh.cny);
          if (xa > xb || ya > yb) {
            verdict = 0;
          } else if ((xb - xa + 1) * (yb - ya + 1) <= 256) {
            const float r_in = rad * (1.f - 1e-4f) - g.cell * 1e-3f, r_out = rad * (1.f + 1e-4f) + g.cell * 1e-3f;
            bool any_maybe = false;
            for (int cy2 = ya; cy2 <= yb && verdict != 1; ++cy2)
              for (int cx2 = xa; cx2 <= xb; ++cx2) {
                const int cc = cy2 * sh.cnx + cx2;
                if (!((sh.coarse[cc >> 5] >> (cc & 31)) & 1u)) continue;
                const float x0 = g.ox + (float)cx2 * C, x1 = x0 + C, y0 = g.oy + (float)cy2 * C, y1 = y0 + C;
                const float nx_ = fmaxf(fmaxf(x0 - q.x, q.x - x1), 0.f), ny_ = fmaxf(fmaxf(y0 - q.y, q.y - y1), 0.f);
                const float fx_ = fmaxf(fabsf(x0 - q.x), fabsf(x1 - q.x)), fy_ = fmaxf(fabsf(y0 - q.y), fabsf(y1 - q.y));
                if (fx_ * fx_ + fy_ * fy_ <= r_in * r_in) {
                  verdict = 1;  // an occupied block lies entirely inside the acceptance disc
                  break;
                }
                if (nx_ * nx_ + ny_ * ny_ <= r_out * r_out) any_maybe = true;
              }
            if (verdict != 1 && !any_maybe) verdict = 0;
          }
        }
        if (verdict < 0) {  // inconclusive: grow the block until the first point inside maxDist shows up
          NNResult r;
          r.d2 = INFINITY, r.pos = -1, r.tie = 0;
          const int cx = grid_cell_coord(q.x, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(q.y, g.oy, g.inv_cell, g.ny);
          const int kmax = max(g.nx, g.ny);
          verdict = 0;
          for (int k = 2;; k = min(2 * k, kmax)) {
            nn_scan_block(g, cx, cy, k, q.x, q.y, r);
            if (r.d2 <= max_d2) {
              verdict = 1;
              break;
            }
            const float b2 = nn_block_bound2(g, q.x, q.y, cx, cy, k);
            if (b2 == INFINITY || b2 > max_d2 || k >= kmax) break;
          }
        }
        qstate[i] |= 4 | (verdict ? 2 : 0) | (verdict ? 0 : 1);  // "nothing within maxDist" is a settled answer
        n_fin += verdict;
        // upper bound of a finite point without candidate; kept finite (maxDist = inf) so that pass C's selection
        // counts it among the total_fin finite entries
        dist[i] = verdict ? fminf(max_d2, ICP_PRUNED) : INFINITY;
      }
      if (total_fin < 0) total_fin = block_total(n_fin, &sh.tot[0][0], tot_phase);  // (its barrier also publishes dist[] / qstate[])
      // pass C: settle what still matters
      if (!small) {
        float stop_d2 = INFINITY;
        if constexpr (FILT) {
          // Several filters (sfe_icp_filters).  Every rank a selection needs must be exact, and so must every distance
          // the upper-limit filters together could keep.  U_k = the k-th smallest upper bound >= the k-th smallest
          // distance, so a search bounded by stop_d2 >= U_k leaves the k smallest distances exact: the selections of
          // 3b see the true elements.  A pair kept by the chain has d2 <= min(out_d2, trim limit, factor * median) <=
          // min(out_d2, U_ktrim, factor * U_kmed) (both limits are at most their upper bounds, the float32 product is
          // monotone), so with stop_d2 at least that minimum every keepable pair is exact, and a pruned point (stored
          // as ICP_PRUNED) fails the filter whose bound is the minimum.  Hence
          //   stop_d2 = max(U_k of each active selection, min(out_d2, U_ktrim, factor * U_kmed)).
          // MinDist keeps far pairs, so it bounds nothing: alone it allows no pruning.
          const bool q_trim = prm.trim_ratio >= 0.f, q_med = b.median_factor >= 0.f;
          if (!((q_trim || q_med) && total_fin == 0)) {
            float u_trim = INFINITY, u_med = INFINITY, sel = -INFINITY;
            if (q_trim && prm.trim_ratio < 1.0f) {
              int kk = (int)(size_t)__fmul_rn((float)total_fin, prm.trim_ratio);
              if (kk >= total_fin) kk = total_fin - 1;
              u_trim = block_select_kth(dist, ns, kk, sh, sel_pass);
            }
            if (q_trim) sel = u_trim;
            if (q_med) {
              int kk = (int)(size_t)__fmul_rn((float)total_fin, 0.5f);
              if (kk >= total_fin) kk = total_fin - 1;
              u_med = block_select_kth(dist, ns, kk, sh, sel_pass);
              sel = fmaxf(sel, u_med);
            }
            float upper = q_trim ? u_trim : INFINITY;
            if (prm.outlier_max_dist > 0.f) upper = fminf(upper, out_d2);
            if (q_med) upper = fminf(upper, __fmul_rn(b.median_factor, u_med));
            stop_d2 = fmaxf(sel, upper);
          }
        } else if (prm.trim_ratio >= 0.f) {
          if (prm.trim_ratio < 1.0f && total_fin > 0) {
            int kk = (int)(size_t)__fmul_rn((float)total_fin, prm.trim_ratio);
            if (kk >= total_fin) kk = total_fin - 1;
            stop_d2 = block_select_kth(dist, ns, kk, sh, sel_pass);  // kk-th smallest upper bound >= kk-th smallest distance
          }
        } else if (prm.outlier_max_dist > 0.f) {
          stop_d2 = out_d2;
        }
        // the unsettled points are few (the scan's outliers) and their searches long: every warp takes the
        // unsettled points of its 32 lanes one after the other and searches for each with all 32 lanes
        for (int i0 = tid & ~31; i0 < ns; i0 += nthr) {
          const int i = i0 + (tid & 31) < ns ? (b.use_order ? (int)order[i0 + (tid & 31)] : i0 + (tid & 31)) : ns;
          const bool mine = i < ns && !(qstate[i] & 1);
          float2 q = make_float2(0.f, 0.f);
          int cand = -1;
          float cand_d2 = INFINITY;
          if (mine) {
            q = apply_T(Ti, reading[i].x, reading[i].y);
            cand = match[i] == NONE ? -1 : (int)match[i];
            cand_d2 = cand >= 0 ? dist[i] : INFINITY;
          }
          unsigned todo = __ballot_sync(0xffffffffu, mine);
          while (todo) {
            const int L = __ffs(todo) - 1;
            todo &= todo - 1;
            const float qx = __shfl_sync(0xffffffffu, q.x, L), qy = __shfl_sync(0xffffffffu, q.y, L);
            NNResult r;
            r.pos = __shfl_sync(0xffffffffu, cand, L);
            r.d2 = __shfl_sync(0xffffffffu, cand_d2, L);
            r.tie = 1;  // pass A did not resolve ties; a block scan below replaces this flag with what it finds
            const int exact = nn_search_warp(g, qx, qy, max_d2, stop_d2, 1, r);
            if ((tid & 31) == L) {
              if (exact) {
                const bool fin = r.pos >= 0 && r.d2 <= max_d2;  // == the finiteness found in pass B
                dist[i] = fin ? r.d2 : INFINITY;
                match[i] = prev[i] = fin ? (Pos)r.pos : (Pos)NONE;
              } else {
                dist[i] = ICP_PRUNED;  // finite, farther than the quantile bound: weight 0
                match[i] = NONE;
              }
            }
          }
        }
        __syncthreads();
      }

      ICP_PH_MARK(1);
      // 3b. trimmed-distance limit = element floor(float(n)*ratio) of the ascending finite distances (FILT: and the
      // median-distance limit)
      float limit = INFINITY, med_limit = INFINITY;
      if (prm.trim_ratio >= 0.f || (FILT && b.median_factor >= 0.f)) {
        if (total_fin == 0) {
          if (tid == 0) sh.status = ICP_NO_OUTLIER;
          __syncthreads();
          break;
        }
        if constexpr (FILT) {  // MedianDistOutlierFilter: factor * getDistsQuantile(0.5), a float32 product
          if (b.median_factor >= 0.f) {
            int kk = (int)(size_t)__fmul_rn((float)total_fin, 0.5f);
            if (kk >= total_fin) kk = total_fin - 1;
            med_limit = __fmul_rn(b.median_factor, block_select_kth(dist, ns, kk, sh, sel_pass));
          }
        }
        if (FILT && prm.trim_ratio < 0.f) {  // (the median alone)
        } else if (prm.trim_ratio == 1.0f) {
          float m = 0.f;
          for (int i = tid; i < ns; i += nthr)
            if (dist[i] < INFINITY) m = fmaxf(m, dist[i]);
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
          float *fr = sh.wred;
          if ((tid & 31) == 0) fr[tid >> 5] = m;
          __syncthreads();
          m = 0.f;
          for (int w = 0; w < (nthr >> 5); ++w) m = fmaxf(m, fr[w]);
          limit = m;
          __syncthreads();
        } else {
          int kk = (int)(size_t)__fmul_rn((float)total_fin, prm.trim_ratio);
          if (kk >= total_fin) kk = total_fin - 1;
          limit = block_select_kth(dist, ns, kk, sh, sel_pass);
        }
      }
      (void)med_limit;

      ICP_PH_MARK(2);
      // 3c. kept pairs.  The candidate match of point i is prev[i] on the one-pass path (its re-search list took
      // match[] meanwhile) and match[i] after the pruning passes; match[i] becomes the candidate or NONE (dropped).
      const Pos *cand = small ? prev : match;
      // ROBUST: the pair's weight is the product of the 0 / 1 weights and the robust weight (oracle/robust_ref.c): the
      // robust weight where the others keep the pair, else 0 * w (NaN for w = inf); dist[i] becomes that weight, and
      // the pair is kept when it is not 0.  A point pruned by pass C (farther than stop_d2 >= 0, so e2 > 0 and w finite)
      // fails the 0 / 1 filter whose bound set stop_d2, so its weight is 0: the robust filter bounds nothing itself,
      // and pass C's argument for FILT holds unchanged.
      auto kept = [&](int i) -> int {
        const int m = cand[i];
        if constexpr (ROBUST) {
          if (m == NONE) return NONE;
          bool keep01 = true;
          if (prm.outlier_max_dist > 0.f) keep01 = keep01 && (dist[i] <= out_d2);
          if (prm.trim_ratio >= 0.f) keep01 = keep01 && (dist[i] <= limit);
          if (b.min_d2 >= 0.f) keep01 = keep01 && (dist[i] > b.min_d2);
          if (b.median_factor >= 0.f) keep01 = keep01 && (dist[i] <= med_limit);
          const float w = __fmul_rn(keep01 ? 1.f : 0.f, icp_robust_weight(b.robust, dist[i]));
          dist[i] = w;
          return w != 0.f ? m : NONE;
        }
        bool keep = m != NONE;
        if (prm.outlier_max_dist > 0.f) keep = keep && (dist[i] <= out_d2);
        if (prm.trim_ratio >= 0.f) keep = keep && (dist[i] <= limit);
        if constexpr (FILT) {
          if (b.min_d2 >= 0.f) keep = keep && (dist[i] > b.min_d2);
          if (b.median_factor >= 0.f) keep = keep && (dist[i] <= med_limit);
        }
        return keep ? m : NONE;
      };
      // Sequential mode: the sums are warp 0's alone, so warp 0 also forms the fit and, on the one-pass path, the
      // weights, with warp-level synchronisation only; the other warps go straight to the barrier that ends the
      // iteration.  (The pruned path's 2 000-point sources keep the weights parallel: measured slower on warp 0.)
      // Float64 mode: every thread takes part in the block_sum reductions.
      int n_keep = 0;
      float mrx = 0.f, mry = 0.f, mfx = 0.f, mfy = 0.f, sw = 0.f;  // (sw: ROBUST, the sum of the weights)
      double t4[4] = {0, 0, 0, 0};
      float pl[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // PLANE: A00 A01 A02 A11 A12 A22, sum F (q-r).n (thread 0)
      if (seq && !small) {  // big problems (long serial sums): every thread forms the weights of its points
        int cnt = 0;
        for (int i = tid; i < ns; i += nthr) {
          const int m = kept(i);
          match[i] = (Pos)m;
          cnt += m != NONE;
        }
        n_keep = block_total(cnt, &sh.tot[0][0], tot_phase);  // (its barrier publishes match[])
      }
      ICP_PH_MARK(3);
      if (!seq || tid < 32) {
        if (!seq) {
          double s5[5] = {0, 0, 0, 0, 0}, t5[5];
          for (int i = tid; i < ns; i += nthr) {
            const int m = kept(i);
            match[i] = (Pos)m;
            if (m == NONE) continue;
            const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
            const float2 r = sorted[m];
            s5[0] += 1.0, s5[1] += (double)q.x, s5[2] += (double)q.y, s5[3] += (double)r.x, s5[4] += (double)r.y;
          }
          block_sum<5>(s5, sh.red, red_phase, t5);
          n_keep = (int)t5[0];
          mrx = (float)t5[1], mry = (float)t5[2], mfx = (float)t5[3], mfy = (float)t5[4];
        } else if (PLANE) {
          if (small) {
            int cnt = 0;
            for (int i = tid; i < ns; i += 32) {
              const int m = kept(i);
              match[i] = (Pos)m;
              cnt += m != NONE;
            }
            n_keep = __reduce_add_sync(0xffffffffu, cnt);
            __syncwarp();  // (seq_sum9_warp's lanes read other lanes' match[] entries)
          }
        } else if constexpr (ROBUST) {
          // the five weighted sums (w, w * step x, w * step y, w * matched reference x, y); dropped pairs add +0
          int cnt = 0;
          const float sum = seq_sum_rows_warp<5>(ns, sh.seq_buf, [&](int i, float(&v)[5]) {
            const int m = small ? kept(i) : match[i];
            if (small) match[i] = (Pos)m;
            if (m == NONE) {
              v[0] = v[1] = v[2] = v[3] = v[4] = 0.f;
              return;
            }
            ++cnt;
            const float w = dist[i];
            const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
            const float2 r = sorted[m];
            v[0] = w, v[1] = __fmul_rn(w, q.x), v[2] = __fmul_rn(w, q.y), v[3] = __fmul_rn(w, r.x);
            v[4] = __fmul_rn(w, r.y);
          });
          if (small) n_keep = __reduce_add_sync(0xffffffffu, cnt);
          sw = __shfl_sync(0xffffffffu, sum, 0);
          mrx = __shfl_sync(0xffffffffu, sum, 1), mry = __shfl_sync(0xffffffffu, sum, 2);
          mfx = __shfl_sync(0xffffffffu, sum, 3), mfy = __shfl_sync(0xffffffffu, sum, 4);
        } else {
          // the four sums (step x, step y, matched reference x, y); dropped pairs add +0
          int cnt = 0;
          const float sum = seq_sum4_warp<(THREADS >= SFE_SEQ_PIPE_MIN)>(ns, sh.seq_buf, [&](int i) -> float4 {
            const int m = small ? kept(i) : match[i];
            if (small) match[i] = (Pos)m;
            if (m == NONE) return make_float4(0.f, 0.f, 0.f, 0.f);
            ++cnt;
            const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
            const float2 r = sorted[m];
            return make_float4(q.x, q.y, r.x, r.y);
          });
          if (small) n_keep = __reduce_add_sync(0xffffffffu, cnt);
          mrx = __shfl_sync(0xffffffffu, sum, 0), mry = __shfl_sync(0xffffffffu, sum, 1);
          mfx = __shfl_sync(0xffffffffu, sum, 2), mfy = __shfl_sync(0xffffffffu, sum, 3);
          __syncwarp();  // (seq_buf and match[] are read again by other lanes below)
        }
        ICP_PH_MARK(4);
        if (n_keep == 0) {
          if (tid == 0) sh.status = ICP_NO_POINT;
        } else {
          if constexpr (PLANE) {
            // 3c'/3d'. point-to-plane normal equations over the kept pairs (oracle/icp_ref.c, minimizer 1):
            //   c = q.x n.y - q.y n.x,  F = (c, n.x, n.y),  A = sum F F^T,  b = -sum F ((q - r).n)
            auto terms = [&](int i, int m, float2 n, float (&v)[9]) {
              const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
              const float2 r = sorted[m];
              const float cr = __fsub_rn(__fmul_rn(q.x, n.y), __fmul_rn(q.y, n.x));
              const float dp = __fadd_rn(__fmul_rn(__fsub_rn(q.x, r.x), n.x), __fmul_rn(__fsub_rn(q.y, r.y), n.y));
              if constexpr (ROBUST) {  // wF = w * F, then A = sum wF F^T, b = -sum wF ((q - r).n)
                const float w = dist[i];
                const float wc = __fmul_rn(w, cr), wx = __fmul_rn(w, n.x), wy = __fmul_rn(w, n.y);
                v[0] = __fmul_rn(wc, cr), v[1] = __fmul_rn(wc, n.x), v[2] = __fmul_rn(wc, n.y), v[3] = __fmul_rn(wx, n.x);
                v[4] = __fmul_rn(wx, n.y), v[5] = __fmul_rn(wy, n.y), v[6] = __fmul_rn(wc, dp), v[7] = __fmul_rn(wx, dp);
                v[8] = __fmul_rn(wy, dp);
                return;
              }
              v[0] = __fmul_rn(cr, cr), v[1] = __fmul_rn(cr, n.x), v[2] = __fmul_rn(cr, n.y), v[3] = __fmul_rn(n.x, n.x);
              v[4] = __fmul_rn(n.x, n.y), v[5] = __fmul_rn(n.y, n.y), v[6] = __fmul_rn(cr, dp), v[7] = __fmul_rn(n.x, dp);
              v[8] = __fmul_rn(n.y, dp);
            };
            if (seq) {  // nine sequential sums in one pass; dropped pairs add +0
              const float sum = seq_sum9_warp<NONE>(ns, pl_scratch, match, nrm, terms);
#pragma unroll
              for (int k = 0; k < 9; ++k) pl[k] = __shfl_sync(0xffffffffu, sum, k);
            } else {
              double s5[5] = {0, 0, 0, 0, 0}, s4[4] = {0, 0, 0, 0}, o5[5], o4[4];
              for (int i = tid; i < ns; i += nthr) {
                const int m = match[i];
                if (m == NONE) continue;
                float v[9];
                terms(i, m, nrm[m], v);
#pragma unroll
                for (int k = 0; k < 5; ++k) s5[k] += (double)v[k];
#pragma unroll
                for (int k = 0; k < 4; ++k) s4[k] += (double)v[5 + k];
              }
              block_sum<5>(s5, sh.red, red_phase, o5);
              block_sum<4>(s4, sh.red, red_phase, o4);
#pragma unroll
              for (int k = 0; k < 5; ++k) pl[k] = (float)o5[k];
#pragma unroll
              for (int k = 0; k < 4; ++k) pl[5 + k] = (float)o4[k];
            }
          } else {
            const float winv = __fdiv_rn(1.0f, ROBUST ? sw : (float)n_keep);
            mrx = __fmul_rn(mrx, winv), mry = __fmul_rn(mry, winv);
            mfx = __fmul_rn(mfx, winv), mfy = __fmul_rn(mfy, winv);

            // 3d. cross-covariance of the centred pairs
            if (seq) {  // m00 = qx*px, m01 = qx*py, m10 = qy*px, m11 = qy*py
              const float sum = seq_sum4_warp<(THREADS >= SFE_SEQ_PIPE_MIN)>(ns, sh.seq_buf, [&](int i) -> float4 {
                const int m = match[i];
                if (m == NONE) return make_float4(0.f, 0.f, 0.f, 0.f);
                const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
                const float2 r = sorted[m];
                const float px = __fsub_rn(q.x, mrx), py = __fsub_rn(q.y, mry);
                float qx = __fsub_rn(r.x, mfx), qy = __fsub_rn(r.y, mfy);
                if constexpr (ROBUST) qx = __fmul_rn(dist[i], qx), qy = __fmul_rn(dist[i], qy);  // (w r~) p~^T
                return make_float4(__fmul_rn(qx, px), __fmul_rn(qx, py), __fmul_rn(qy, px), __fmul_rn(qy, py));
              });
#pragma unroll
              for (int k = 0; k < 4; ++k) t4[k] = (double)__shfl_sync(0xffffffffu, sum, k);
            } else {
              double s4[4] = {0, 0, 0, 0};
              for (int i = tid; i < ns; i += nthr) {
                if (match[i] == NONE) continue;
                const float2 q = apply_T(Ti, reading[i].x, reading[i].y);
                const float2 r = sorted[match[i]];
                const float px = __fsub_rn(q.x, mrx), py = __fsub_rn(q.y, mry);
                const float qx = __fsub_rn(r.x, mfx), qy = __fsub_rn(r.y, mfy);
                s4[0] += (double)__fmul_rn(qx, px), s4[1] += (double)__fmul_rn(qx, py);
                s4[2] += (double)__fmul_rn(qy, px), s4[3] += (double)__fmul_rn(qy, py);
              }
              block_sum<4>(s4, sh.red, red_phase, t4);
            }
          }

          ICP_PH_MARK(5);
          // 3e. rigid fit, T_iter update, checkers (one thread)
          if (tid == 0) {
            float c = 1.f, s = 0.f, tx, ty;
            if constexpr (PLANE) {
              // A x = b by Cholesky (A.llt()); an unknown whose pivot is not positive stays 0
              const float a00 = pl[0], a01 = pl[1], a02 = pl[2], a11 = pl[3], a12 = pl[4], a22 = pl[5];
              const float b0 = -pl[6], b1 = -pl[7], b2 = -pl[8];
              float l00 = 0.f, l10 = 0.f, l20 = 0.f, l11 = 0.f, l21 = 0.f, l22 = 0.f;
              const bool p0 = a00 > 0.f;
              if (p0) l00 = __fsqrt_rn(a00), l10 = __fdiv_rn(a01, l00), l20 = __fdiv_rn(a02, l00);
              const float d1 = __fsub_rn(a11, __fmul_rn(l10, l10));
              const bool p1 = d1 > 0.f;
              if (p1) l11 = __fsqrt_rn(d1), l21 = __fdiv_rn(__fsub_rn(a12, __fmul_rn(l20, l10)), l11);
              const float d2 = __fsub_rn(__fsub_rn(a22, __fmul_rn(l20, l20)), __fmul_rn(l21, l21));
              const bool p2 = d2 > 0.f;
              if (p2) l22 = __fsqrt_rn(d2);
              const float y0 = p0 ? __fdiv_rn(b0, l00) : 0.f;
              const float y1 = p1 ? __fdiv_rn(__fsub_rn(b1, __fmul_rn(l10, y0)), l11) : 0.f;
              const float y2 = p2 ? __fdiv_rn(__fsub_rn(__fsub_rn(b2, __fmul_rn(l20, y0)), __fmul_rn(l21, y1)), l22) : 0.f;
              const float x2 = p2 ? __fdiv_rn(y2, l22) : 0.f;
              const float x1 = p1 ? __fdiv_rn(__fsub_rn(y1, __fmul_rn(l21, x2)), l11) : 0.f;
              const float x0 = p0 ? __fdiv_rn(__fsub_rn(__fsub_rn(y0, __fmul_rn(l10, x1)), __fmul_rn(l20, x2)), l00) : 0.f;
              c = (float)cos((double)x0), s = (float)sin((double)x0);  // Rotation2D(x0)
              tx = x1, ty = x2;
            } else {
              const float m00 = (float)t4[0], m01 = (float)t4[1], m10 = (float)t4[2], m11 = (float)t4[3];
              const float a = __fadd_rn(m00, m11), bq = __fsub_rn(m10, m01);
              const float h = sqrtf(__fadd_rn(__fmul_rn(a, a), __fmul_rn(bq, bq)));
              if (h > 0.f) c = __fdiv_rn(a, h), s = __fdiv_rn(bq, h);
              tx = __fsub_rn(mfx, __fadd_rn(__fmul_rn(c, mrx), __fmul_rn(-s, mry)));
              ty = __fsub_rn(mfy, __fadd_rn(__fmul_rn(s, mrx), __fmul_rn(c, mry)));
            }
            const float dT[9] = {c, -s, tx, s, c, ty, 0.f, 0.f, 1.f};
            float Tn[9];
            mat3_mul_rn(dT, Ti, Tn);
#pragma unroll
            for (int i = 0; i < 9; ++i) sh.Tprev[i] = Ti[i], sh.Ti[i] = Tn[i];
            sh.todo_n = 0;  // the next iteration's list counter (read before this iteration's n_fin total)
            sh.inliers = n_keep;
            const int count = ++sh.count;
            bool counter_stop = false;
            if (count >= prm.max_iterations) sh.iterate = 0, counter_stop = true;
            if (!counter_stop && smooth > 0) {
              int hn = sh.hn;
              if (hn == ICP_HIST) {
                for (int i = 0; i + 1 < ICP_HIST; ++i)
                  sh.hq_w[i] = sh.hq_w[i + 1], sh.hq_z[i] = sh.hq_z[i + 1], sh.ht_x[i] = sh.ht_x[i + 1],
                  sh.ht_y[i] = sh.ht_y[i + 1];
                hn = ICP_HIST - 1;
              }
              rot_to_quat(Tn, sh.hq_w[hn], sh.hq_z[hn]);
              sh.ht_x[hn] = Tn[2], sh.ht_y[hn] = Tn[5];
              ++hn;
              sh.hn = hn;
              float vr = 0.f, vt = 0.f;
              if (hn > smooth) {
                for (int i = hn - 1; i >= hn - smooth; --i) {
                  const float dw = __fadd_rn(__fmul_rn(sh.hq_w[i], sh.hq_w[i - 1]), __fmul_rn(sh.hq_z[i], sh.hq_z[i - 1]));
                  const float dz = __fsub_rn(__fmul_rn(sh.hq_z[i], sh.hq_w[i - 1]), __fmul_rn(sh.hq_w[i], sh.hq_z[i - 1]));
                  vr = __fadd_rn(vr, fabsf(__fmul_rn(2.0f, atan2f(fabsf(dz), fabsf(dw)))));
                  const float ex = __fsub_rn(sh.ht_x[i], sh.ht_x[i - 1]), ey = __fsub_rn(sh.ht_y[i], sh.ht_y[i - 1]);
                  vt = __fadd_rn(vt, fabsf(sqrtf(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)))));
                }
                vr = __fdiv_rn(vr, (float)smooth);
                vt = __fdiv_rn(vt, (float)smooth);
                if (vr < prm.min_diff_rot && vt < prm.min_diff_trans) sh.iterate = 0;
              }
              if (vr != vr)
                sh.status = ICP_NAN_ROT;
              else if (vt != vt)
                sh.status = ICP_NAN_TRANS;
            }
          }
        }
      }
      __syncthreads();
      ICP_PH_MARK(6);
      if (sh.status != ICP_OK || !sh.iterate) break;
    }

    // ---- 4. back to the caller's frame
    if (tid == 0) {
      if (sh.status == ICP_OK) {
        const float Tm[9] = {1.f, 0.f, mx, 0.f, 1.f, my, 0.f, 0.f, 1.f};
        float tmp[9], out[9], Ti[9], T0[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) Ti[i] = sh.Ti[i], T0[i] = sh.T0[i];
        mat3_mul_rn(Tm, Ti, tmp);
        mat3_mul_rn(tmp, T0, out);
#pragma unroll
        for (int i = 0; i < 9; ++i) b.T_out[9 * (size_t)p + i] = out[i];
      } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) b.T_out[9 * (size_t)p + i] = guess[i];
      }
      b.iters[p] = sh.count;
      b.inliers[p] = sh.inliers;
      b.status[p] = sh.status;
    }
  }
  ICP_PH_FLUSH();
}
