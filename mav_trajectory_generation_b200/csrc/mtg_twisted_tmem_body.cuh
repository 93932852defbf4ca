// mtg_twisted_tmem_body.cuh -- the body of v3 and of its cost-only forms, included as the body of
// twisted_tmem_kernel and of twisted_tmem_line_search_kernel (mtg_twisted_tmem_kernel.cuh).  Each kernel defines N, R,
// D, FUSED, COST and LSEARCH (with COST: the line-search time generator instead of the Mellinger one) and its
// parameters `prm` and `tmap`.  A textual body, not an inlined device function, keeps the code of the existing
// instantiations exactly what it was before the line-search form existed.
  constexpr int h = N / 2;
  constexpr int m = h - 1;
  using Lay = V3Layout<N, D>;
  // per eliminated vertex: L (strictly lower) + inverse pivots + y + the vertex position (so that the
  // outward sweep does not re-read it from global memory)
  constexpr int kSlots = Lay::kSlots;
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = kTmemThreads / 32;
  using G = H1Imm<N, R>;     // immediates: this kernel is register-bound (see mtg_device.cuh)
  using AI = A1InvImm<N>;
  using S = sweep::Sweep<N, D, G>;

  extern __shared__ __align__(128) unsigned char smem_raw[];  // TMA tensor stores need 128-byte aligned tiles
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int half = lane & 1;
  const int K = prm.K;
  const int nf = prm.n_fixed;
  const int M = (K + 1) >> 1;
  const int nh = half ? K - M - 1 : M - 1;
  const int nmax = M - 1;
  const sweep::Frame<N> fr{K, half};

  // ---- shared memory carve-up (V3Layout): [staging: kWarps tiles][prefetch ring][time history][sweep state]
  double2* stage = reinterpret_cast<double2*>(smem_raw) + size_t(warp) * 32 * (D * h);  // [half][16][D*h]
  // per-thread prefetch ring for the next step's inputs (segment time + D positions), filled by
  // cp.async: a register prefetch would share its scoreboard slot with the load being consumed and the
  // consumer would wait for the NEW loads as well (measured: 25 % of all stall samples).
  double* pf = reinterpret_cast<double*>(smem_raw + tmem_stage_bytes<N, D>()) + threadIdx.x;
  auto PF = [&](int buf, int slot) -> double* { return pf + (size_t(buf) * (1 + D) + slot) * kTmemThreads; };
  // per-thread history of the own-frame segment times seen by the inward sweep (nmax+1 doubles): the
  // outward sweep reads them back from shared memory (in FUSED mode this also saves the sqrt/exp)
  double* thist = pf + size_t(Lay::kHist) * kTmemThreads;
  auto HT = [&](int j) -> double& { return thist[size_t(j) * kTmemThreads]; };
  double* state = thist + size_t(Lay::hist_slots(nmax)) * kTmemThreads;
  auto SP = [&](int blk, int slot) -> double& { return state[(size_t(blk) * kSlots + slot) * kTmemThreads]; };

  const long long traj0 = ((long long)blockIdx.x * kWarps + warp) * 16;  // first trajectory of this warp
  long long traj = traj0 + (lane >> 1);
  const bool valid = traj < prm.B;
  if (!valid) traj = prm.B - 1;

  // cost-only mode with the Mellinger expansion generated on the fly: inputs come from the base trajectory
  long long src = traj;
  // each time generator reads its own of these
  [[maybe_unused]] int mel_n = -1;
  [[maybe_unused]] double mel_corr = 0.0;
  [[maybe_unused]] double ls_step = 0.0;
  if constexpr (COST && LSEARCH) {
    src = traj / kLineSearchSteps;
    ls_step = line_search_step(__ldg(prm.ls_alpha + src), int(traj - src * kLineSearchSteps));
  } else if constexpr (COST) {
    if (prm.mel_k1 > 0) {
      src = traj / prm.mel_k1;
      mel_n = int(traj - src * prm.mel_k1) - 1;
      mel_corr = prm.mel_inc / (K - 1.0);
    }
  }
  auto time_of = [&](double raw, int seg_index) -> double {  // seg_index: ORIGINAL segment index
    if constexpr (COST && LSEARCH) {
      return line_search_time(raw, __ldg(prm.ls_grad + src * K + seg_index), ls_step, prm.mel_lower);
    } else if constexpr (COST) {
      return mellinger_time(raw, seg_index, mel_n, prm.mel_inc, mel_corr, prm.mel_lower);
    }
    return raw;
  };
  const double* __restrict__ tt = FUSED ? nullptr : prm.times + src * K;
  const double* __restrict__ fx =
      FUSED ? prm.positions + src * (long long)(K + 1) * D : prm.dfix + src * (long long)D * nf;
  // address of coordinate d of own-frame vertex v
  auto xaddr = [&](int v, int d) -> const double* {
    if constexpr (FUSED) {
      return fx + fr.vert(v) * D + d;
    } else {
      return fx + d * nf + fr.pidx(v);
    }
  };
  // prefetch (time of own segment j, position of own vertex v) into ring buffer `buf`
  auto pf_issue = [&](int buf, int j, int v) {
    if constexpr (!FUSED) cp_async8(PF(buf, 0), tt + fr.seg(j));
#pragma unroll
    for (int d = 0; d < D; ++d) cp_async8(PF(buf, 1 + d), xaddr(v, d));
  };
  [[maybe_unused]] double* __restrict__ tout = (FUSED && prm.times_out != nullptr) ? prm.times_out + traj * K : nullptr;

  // ---- issue the first global loads NOW: their latency overlaps the index set-up below
  double T0e = 0.0, x0e[D], x1e[D], u0e[m][D];
  {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      x0e[d] = __ldg(xaddr(0, d));
      x1e[d] = __ldg(xaddr(1, d));
#pragma unroll
      for (int b = 0; b < m; ++b) u0e[b][d] = FUSED ? 0.0 : __ldg(fx + d * nf + fr.e0() + b);
    }
    if constexpr (!FUSED) T0e = __ldg(tt + fr.seg(0));
    pf_issue(1, 1, 2);  // inputs of sweep step v = 1 -> ring buffer (v & 1)
  }

  double2* my_row = stage + ((lane & 1) * 16 + (lane >> 1)) * (D * h);
  const int nhF = M - 1, nhB = K - M - 1;  // a half is active in sweep step v iff v <= its nh
  const TmaEmitter<N, D, AI> out{&tmap, stage, my_row, lane, K, nhF, nhB};

  double cost_acc = 0.0;
  auto emit_all = [&](int j, int v_step, double T, double iT, const double (&sd)[h][D], const double (&ed)[h][D]) {
    if constexpr (COST) {
      // 0.5 d^T H(T) d of this segment, d = [start derivatives; end derivatives] in the own frame (the cost is
      // invariant under the time reversal of the odd half): H = T^(1-2r) S G S / scale, S = diag(T^(s mod h)).
      (void)j;
      const int nh_own = half ? nhB : nhF;
      if (v_step <= nh_own) {
        double tp[h];
        tp[0] = 1.0;
#pragma unroll
        for (int k = 1; k < h; ++k) tp[k] = tp[k - 1] * T;
        double q = 0.0;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          double u[N];
#pragma unroll
          for (int k = 0; k < h; ++k) {
            u[k] = tp[k] * sd[k][d];
            u[h + k] = tp[k] * ed[k][d];
          }
#pragma unroll
          for (int s2 = 0; s2 < N; ++s2) {
            double row = 0.5 * G::at(s2, s2) * u[s2];
#pragma unroll
            for (int t2 = s2 + 1; t2 < N; ++t2) row = fma(G::at(s2, t2), u[t2], row);
            q = fma(row, u[s2], q);
          }
        }
        // T^(1-2r) = T * (1/T)^(2r)
        cost_acc = fma(q, T * pow_int<2 * R>(iT), cost_acc);
      }
      return;
    }
    out.emit(j, v_step, T, iT, sd, ed, traj0);
  };

  int stat = 0;
  double Wp[m][m], yp[m][D], Cee[m][m], cps[m], cpe[m], bcar[m][D], xm[D], xc[D];
  {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      xm[d] = x0e[d];
      xc[d] = x1e[d];
    }
    double T0;
    if constexpr (FUSED) {
      T0 = nfabian_time<D>(xm, xc, prm.v_max, prm.a_max, prm.magic);
    } else {
      T0 = time_of(T0e, fr.seg(0));
    }
    if (bad_segment_time(T0)) stat |= kStatusBadTime;
    HT(0) = T0;
    const double iT0 = fast_rcp(T0);
    double pw[N - 1];
    segment_powers<N, R>(T0, iT0, pw);
    S::end_blocks(pw, Cee, cps, cpe);
    S::carry_bcar(pw, [&](int b, int d) { return fr.sgn(b) * u0e[b][d]; }, Wp, yp, bcar);
  }

  // ---------------------------------------------------------------- sweep towards the middle
  for (int v = 1; v <= nmax; ++v) {
    double sv[kSlots];  // lanes with v > nh store whatever is here; they never read it back
    if (v <= nh) {
      cp_async_wait_all();
      double xn[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xn[d] = *PF(v & 1, 1 + d);
      double T;
      if constexpr (FUSED) {
        T = nfabian_time<D>(xc, xn, prm.v_max, prm.a_max, prm.magic);
      } else {
        T = time_of(*PF(v & 1, 0), fr.seg(v));
      }
      HT(v) = T;
      {  // prefetch the next step's inputs (clamped indices: never out of bounds)
        const int jn = v + 1 < K ? v + 1 : K - 1;
        const int vn = v + 2 <= K ? v + 2 : K;
        pf_issue((v + 1) & 1, jn, vn);
      }
      if (bad_segment_time(T)) stat |= kStatusBadTime;
      const double iT = fast_rcp(T);
      double pw[N - 1];
      segment_powers<N, R>(T, iT, pw);

      double Dp[m][m], E[m][m], bb[m][D], L[m][m], inv[m];
      S::assemble(pw, Cee, cps, cpe, bcar, Wp, yp, xm, xc, xn, Dp, E, bb);
      S::factor(Dp, E, bb, L, inv, Wp, yp, stat);
      S::pack(L, inv, yp, xc, sv);  // with the position of the vertex just eliminated
      S::end_blocks(pw, Cee, cps, cpe);
#pragma unroll
      for (int a = 0; a < m; ++a)
#pragma unroll
        for (int d = 0; d < D; ++d) bcar[a][d] = 0.0;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        xm[d] = xc[d];
        xc[d] = xn[d];
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kSlots; ++i) SP(v - 1, i) = sv[i];
  }
  __syncwarp();

  // ---------------------------------------------------------------- middle vertex
  double um[m][D];
  S::middle(Cee, cps, cpe, bcar, Wp, yp, xm, xc, um, stat);
  if (valid && half == 0 && prm.status != nullptr) prm.status[traj] = stat;

  // ---------------------------------------------------------------- outward back-substitution
  const sweep::FreeStore<N, D> store_free(prm.dfree, traj, valid, fr);

  double ed[h][D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ed[0][d] = xc[d];
#pragma unroll
    for (int j = 0; j < m; ++j) ed[1 + j][d] = um[j][d];
  }
  if (half == 0) store_free(nh + 1, ed);

  // outward steps take the vertex position from the sweep state; only the segment time is prefetched
  // (and the position of own vertex 0 for the final emission)
  auto pf_issue_out = [&](int j) {
    if (j == 0) pf_issue(0, 0, 0);  // position of own vertex 0 for the final emission (time comes from HT)
  };
  pf_issue_out(nh);

  for (int v = nmax; v >= 1; --v) {
    double sv[kSlots];
#pragma unroll
    for (int i = 0; i < kSlots; ++i) sv[i] = SP(v - 1, i);
    const bool act = v <= nh;
    double T = 1.0, iT = 1.0;
    double sd[h][D];  // inactive lanes (odd K only) emit garbage rows that are never stored
    if (act) {
      cp_async_wait_all();
      double xv[D];
#pragma unroll
      for (int d = 0; d < D; ++d) xv[d] = S::position(sv, d);
      T = HT(v);
      if constexpr (FUSED) {
        if (tout != nullptr && valid) tout[fr.seg(v)] = T;
      }
      pf_issue_out(v - 1);
      if constexpr (!FUSED) {
        if (v == 1) {  // the final emission re-reads the fixed end derivatives: pull their lines into L1 now
#pragma unroll
          for (int d = 0; d < D; ++d) asm volatile("prefetch.global.L1 [%0];" ::"l"(fx + d * nf + fr.e0()));
        }
      }
      iT = fast_rcp(T);
      double L[m][m], inv[m], rhs[m][D], pw[N - 1];
      S::unpack(sv, L, inv, rhs);
      segment_powers<N, R>(T, iT, pw);
      S::uncouple_from(pw, ed, L, inv, rhs);
      S::solve_back(L, inv, rhs, xv, sd);
      store_free(v, sd);
    }
    __syncwarp();
    emit_all(v, v, T, iT, sd, ed);
    if (act) {
#pragma unroll
      for (int d = 0; d < D; ++d)
#pragma unroll
        for (int k = 0; k < h; ++k) ed[k][d] = sd[k][d];
    }
  }
  {
    cp_async_wait_all();
    double sd[h][D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      sd[0][d] = *PF(0, 1 + d);
#pragma unroll
      for (int b = 0; b < m; ++b) sd[1 + b][d] = FUSED ? 0.0 : fr.sgn(b) * __ldg(fx + d * nf + fr.e0() + b);
    }
    const double T = HT(0);
    if constexpr (FUSED) {
      if (tout != nullptr && valid) tout[fr.seg(0)] = T;
    }
    const double iT = fast_rcp(T);
    __syncwarp();
    emit_all(0, 0, T, iT, sd, ed);
  }

  if constexpr (COST) {
    // q accumulated sum_{s<=t} (1 or 1/2) G u u = 0.5 u^T G u per segment: cost = sum over both halves / scale
    const double other = __shfl_xor_sync(kFull, cost_acc, 1);
    if (valid && half == 0 && prm.cost != nullptr) prm.cost[traj] = (cost_acc + other) * (1.0 / G::scale);
  }
  if (lane == 0) bulk_wait_all();  // every TMA store issued by this warp has completed
