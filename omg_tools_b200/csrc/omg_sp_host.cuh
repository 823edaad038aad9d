// omg_sp_host.cuh -- host side of the sparse kernel variant (included by omg_b200.cu after
// the definition of omg_problem): symbolic analysis of the condensed KKT matrix
//     K = [[H, Jc^T], [Jc, -dc I]]           (H = W + J^T Sigma J, Jc = equality rows)
// and construction of the thread streams.  Everything here runs once per problem structure
// (the counterpart of IPOPT's symbolic factorisation inside nlpsol, optilayer.py:49-60).
#pragma once
#include <queue>
#include <map>

namespace {

struct SpSym {
  int N = 0, n = 0, R0 = 0, nr = 0, n_lev = 0, Lsize = 0;
  std::vector<int> pos;                       // natural node (var j / n + eq k) -> permuted index
  std::vector<std::vector<int>> st;           // struct of each permuted column (ascending, < N)
  std::vector<int> colptr, lev, len;
  std::vector<std::vector<int>> st_true;      // struct without the explicit zeros of the supernode padding
  std::vector<int> sn_first, sn_w;            // first column / width of the supernode of a column (root: itself, 1)
  int n_pad = 0;                              // explicit zeros stored
  int max_sn_pad = 0;                         // ... by the supernode with the most
  int idx(int i, int j) const {               // L index of entry (row i, column j); i == N: rhs
    if (j >= R0) return colptr[j] + (i - j);
    if (i == j) return colptr[j];
    if (i == N) return colptr[j] + len[j] + 1;
    const std::vector<int>& s = st[j];
    const auto it = std::lower_bound(s.begin(), s.end(), i);
    if (it == s.end() || *it != i) return -1;
    return colptr[j] + 1 + (int)(it - s.begin());
  }
};

// constrained minimum-degree ordering (an equality row becomes eligible once every variable it
// couples is eliminated, so its pivot is a genuine Schur complement) + symbolic factorisation
static bool sp_symbolic(const omg_tables* tb, SpSym& Y, std::string* why) {
  const int n = tb->n, n_eq = tb->kkt_n_eq, N = n + n_eq;
  Y.N = N; Y.n = n;
  std::vector<std::vector<char>> A(N, std::vector<char>(N, 0));
  for (int q = 0; q < tb->nnz_h; ++q) {
    const int r = tb->hrow[q], c = tb->hcol[q];
    if (r != c) { A[r][c] = 1; A[c][r] = 1; }
  }
  std::vector<int> pending(n_eq, 0);          // uneliminated variables coupled to equality row k
  std::vector<std::vector<int>> eq_of_var(n);
  for (int k = 0; k < n_eq; ++k) {
    const int i = tb->kkt_eq_rows[k];
    for (int s = tb->jrow_ptr[i]; s < tb->jrow_ptr[i + 1]; ++s) {
      const int c = tb->jcol[s];
      if (!A[n + k][c]) { A[n + k][c] = 1; A[c][n + k] = 1; pending[k]++; eq_of_var[c].push_back(k); }
    }
  }
  std::vector<int> deg(N, 0);
  for (int a = 0; a < N; ++a) for (int b = 0; b < N; ++b) deg[a] += A[a][b];
  std::vector<char> gone(N, 0);
  std::vector<int> order; order.reserve(N);
  std::vector<std::vector<int>> st_nodes(N);
  for (int step = 0; step < N; ++step) {
    int v = -1;
    for (int a = 0; a < N; ++a) {
      if (gone[a]) continue;
      if (a >= n && pending[a - n] > 0) continue;
      if (v < 0 || deg[a] < deg[v]) v = a;
    }
    if (v < 0) { *why = "no eligible pivot in the ordering"; return false; }
    std::vector<int> nb;
    for (int b = 0; b < N; ++b) if (A[v][b] && !gone[b]) nb.push_back(b);
    for (size_t x = 0; x < nb.size(); ++x)
      for (size_t y = x + 1; y < nb.size(); ++y) {
        const int a = nb[x], b = nb[y];
        if (!A[a][b]) { A[a][b] = 1; A[b][a] = 1; deg[a]++; deg[b]++; }
      }
    for (int b : nb) deg[b]--;
    gone[v] = 1;
    if (v < n) for (int k : eq_of_var[v]) pending[k]--;
    st_nodes[step] = nb;
    order.push_back(v);
  }
  Y.pos.assign(N, 0);
  for (int s = 0; s < N; ++s) Y.pos[order[s]] = s;
  Y.st.assign(N, {});
  for (int j = 0; j < N; ++j) {
    for (int b : st_nodes[j]) Y.st[j].push_back(Y.pos[b]);
    std::sort(Y.st[j].begin(), Y.st[j].end());
  }
  // root = the final chain of the elimination tree while it stays dense enough
  std::vector<int> parent(N, -1);
  for (int j = 0; j < N; ++j) if (!Y.st[j].empty()) parent[j] = Y.st[j][0];
  // (a column joins only while it is alone on its level of the full tree: a chain that runs
  // beside other chains costs nothing as a level, but a barrier per pivot inside the root)
  std::vector<int> lev_all(N, 0), cnt(N + 1, 0);
  for (int j = 0; j < N; ++j) if (parent[j] >= 0) lev_all[parent[j]] = std::max(lev_all[parent[j]], lev_all[j] + 1);
  for (int j = 0; j < N; ++j) cnt[lev_all[j]]++;
  int R0 = N - 1;
  while (R0 > 0 && parent[R0 - 1] == R0 && cnt[lev_all[R0 - 1]] == 1 && (N - (R0 - 1)) <= SP_MAXROOT &&
         2 * (int)Y.st[R0 - 1].size() >= (N - R0)) --R0;
  if (N == 0) R0 = 0;
  Y.R0 = R0; Y.nr = N - R0;
  // ---- supernodes: paths of the elimination tree (column, parent, grandparent ...) of up to
  // SP_SNW columns.  Their columns get the structure of the LAST one (explicit zeros where a
  // column's own structure is smaller: all of it lies inside the last column's clique, so the
  // symbolic structure stays closed and the padded entries stay exactly zero), are numbered
  // consecutively and are scheduled as ONE level step: gather from outside, then a dense
  // (w + rows) x w panel finished without block-wide barriers (omg_sp.cuh, sp_factor).
  int snw_max = SP_SNW;                       // (tuning knob for experiments)
  { const char* e = getenv("OMG_B200_SNW"); if (e && atoi(e) >= 1 && atoi(e) <= SP_SNW) snw_max = atoi(e); }
  std::vector<int> sn_id(R0, -1);
  std::vector<std::vector<int>> paths;
  int total_z = 0;
  for (int j = 0; j < R0; ++j) {
    if (sn_id[j] >= 0) continue;
    const int id = (int)paths.size();
    std::vector<int> path(1, j);
    sn_id[j] = id;
    int zcur = 0;
    while ((int)path.size() < snw_max) {
      const int p = parent[path.back()];
      if (p < 0 || p >= R0 || sn_id[p] >= 0) break;
      const int L = (int)path.size() + 1;
      int newz = 0;
      for (int q = 0; q < L - 1; ++q) newz += (L - 1 - q) + (int)Y.st[p].size() - (int)Y.st[path[q]].size();
      if (newz > SP_SNZ || total_z + newz - zcur > SP_SNZ_TOTAL) break;
      path.push_back(p); sn_id[p] = id;
      total_z += newz - zcur; zcur = newz;
    }
    Y.max_sn_pad = std::max(Y.max_sn_pad, zcur);
    paths.push_back(path);
  }
  Y.n_pad = total_z;
  const int n_sn = (int)paths.size();
  std::vector<int> sn_lev(n_sn, 0), by_last(n_sn);
  for (int a = 0; a < n_sn; ++a) by_last[a] = a;
  std::sort(by_last.begin(), by_last.end(), [&](int a, int b) { return paths[a].back() < paths[b].back(); });
  for (int a : by_last) {                     // children (smaller last column) come first
    const int p = parent[paths[a].back()];
    if (p >= 0 && p < R0) sn_lev[sn_id[p]] = std::max(sn_lev[sn_id[p]], sn_lev[a] + 1);
  }
  std::vector<int> sn_order(n_sn);
  for (int a = 0; a < n_sn; ++a) sn_order[a] = a;
  std::stable_sort(sn_order.begin(), sn_order.end(), [&](int a, int b) {
    return sn_lev[a] != sn_lev[b] ? sn_lev[a] < sn_lev[b] : paths[a][0] < paths[b][0]; });
  std::vector<int> new_of(N);
  {
    int nxt = 0;
    for (int a : sn_order) for (int c : paths[a]) new_of[c] = nxt++;
    for (int j = R0; j < N; ++j) new_of[j] = j;
  }
  {
    std::vector<std::vector<int>> st2(N), tr2(N);
    Y.lev.assign(N, 0); Y.sn_first.assign(N, 0); Y.sn_w.assign(N, 1);
    for (int j = R0; j < N; ++j) { st2[j] = Y.st[j]; tr2[j] = Y.st[j]; Y.sn_first[j] = j; }
    int n_lev = 0;
    for (int a = 0; a < n_sn; ++a) {
      const std::vector<int>& path = paths[a];
      const int w = (int)path.size(), last = path.back();
      for (int q = 0; q < w; ++q) {
        const int c = path[q], cn = new_of[c];
        for (int b : Y.st[c]) tr2[cn].push_back(new_of[b]);
        for (int q2 = q + 1; q2 < w; ++q2) st2[cn].push_back(new_of[path[q2]]);
        for (int b : Y.st[last]) st2[cn].push_back(new_of[b]);
        std::sort(tr2[cn].begin(), tr2[cn].end());
        std::sort(st2[cn].begin(), st2[cn].end());
        Y.lev[cn] = sn_lev[a]; Y.sn_first[cn] = new_of[path[0]]; Y.sn_w[cn] = w;
      }
      n_lev = std::max(n_lev, sn_lev[a] + 1);
    }
    Y.st.swap(st2); Y.st_true.swap(tr2);
    Y.n_lev = n_lev;
    for (int v = 0; v < N; ++v) Y.pos[v] = new_of[Y.pos[v]];
  }
  Y.len.assign(N, 0); Y.colptr.assign(N + 1, 0);
  for (int j = 0; j < N; ++j) {
    Y.len[j] = (int)Y.st[j].size();
    if (j < R0 && Y.len[j] > SP_MAXCOL) { *why = "column structure too long for the packed pairs"; return false; }
    Y.colptr[j + 1] = Y.colptr[j] + ((j < R0) ? Y.len[j] + 2 : (N - j + 1));
  }
  Y.Lsize = Y.colptr[N];
  if (Y.Lsize + 1 > SP_MAXL || N > SP_MAXN) { *why = "factor too large for the packed pairs"; return false; }
  return true;
}

// thread-balanced stream: lists[o] = records of output o (the builder sets the end flag on the
// last one through `mark_end`; empty outputs get `dummy(o)`), laid out for nt threads
template <typename Rec, typename MarkEnd>
static void sp_build_stream(const std::vector<std::vector<Rec>>& lists, const std::vector<Rec>& dummies,
                            const Rec& pad, MarkEnd mark_end, int nt, std::vector<Rec>& out, int* n_chunk) {
  const int n_out = (int)lists.size();
  std::vector<int> ord(n_out);
  for (int o = 0; o < n_out; ++o) ord[o] = o;
  auto size_of = [&](int o) { return lists[o].empty() ? 1 : (int)lists[o].size(); };
  std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return size_of(a) > size_of(b); });
  typedef std::pair<int, int> LT;   // (load, thread)
  std::priority_queue<LT, std::vector<LT>, std::greater<LT>> heap;
  for (int t = 0; t < nt; ++t) heap.push(LT(0, t));
  std::vector<std::vector<Rec>> per(nt);
  for (int o : ord) {
    LT top = heap.top(); heap.pop();
    std::vector<Rec>& dst = per[top.second];
    if (lists[o].empty()) { Rec r = dummies[o]; mark_end(r); dst.push_back(r); }
    else {
      for (size_t k = 0; k < lists[o].size(); ++k) {
        Rec r = lists[o][k];
        if (k + 1 == lists[o].size()) mark_end(r);
        dst.push_back(r);
      }
    }
    heap.push(LT(top.first + size_of(o), top.second));
  }
  size_t mx = 0;
  for (int t = 0; t < nt; ++t) mx = std::max(mx, per[t].size());
  const int nc = (int)((mx + SP_R - 1) / SP_R);
  *n_chunk = nc;
  out.assign((size_t)std::max(nc, 1) * SP_R * nt, pad);
  for (int t = 0; t < nt; ++t)
    for (size_t k = 0; k < per[t].size(); ++k) out[k * nt + t] = per[t][k];
}

}  // namespace

// Build the sparse structure + streams; false (with a reason) when the problem is outside what
// the sparse kernel covers -- the caller then uses the envelope kernels.
static bool sp_setup(omg_problem* h, const omg_tables* tb, const cudaDeviceProp& prop, std::string* why) {
  const int n = tb->n, m = tb->m, n_eq = tb->kkt_n_eq, N = n + n_eq;
  if (tb->n_mid > 0) { *why = "intermediates"; return false; }
  if (tb->G.width > 2 || tb->J.width > 1 || tb->W.width > 1) { *why = "term degree > 2"; return false; }
  if (tb->n_v >= 32768 || tb->nnz_j >= 65535 || m + 2 >= 65535 || n + 2 >= 65535) { *why = "index range"; return false; }
  int nt = 128;
  // (the kernel is compiled for 128-thread blocks: __launch_bounds__(128, 3))
  SpSym Y;
  if (!sp_symbolic(tb, Y, why)) return false;
  const int R0 = Y.R0, nr = Y.nr;
  SpTab& P = h->P;
  memset(&P, 0, sizeof(P));
  bool ok = true;
  // counters of the structure line: which branches of sp_factor / sp_back_solve this structure
  // runs, and how close it comes to the packing limits (tests/test_sparse_structures.py)
  int eq_lev = 0, eq_panel = 0, eq_root = 0, n_snw[SP_SNW + 1] = {0}, max_col = 0, max_gather = 0,
      max_slices = 0, max_blk = 0, max_prounds = 0, max_nq = 0, max_brounds = 0;
  for (int j = 0; j < R0; ++j) max_col = std::max(max_col, Y.len[j]);
  P.nt = nt;
  P.zslot = Y.Lsize; P.Lsz = (Y.Lsize + 2) & ~1;
  P.R0 = R0; P.nr = nr; P.n_lev = Y.n_lev; P.root0 = Y.colptr[R0];
  P.n_rootent = Y.Lsize - Y.colptr[R0];
  {  // leading levels made of variables that no equality row touches (early inertia rejection)
    std::vector<char> touched(n, 0);
    for (int k = 0; k < n_eq; ++k) {
      const int i = tb->kkt_eq_rows[k];
      for (int s = tb->jrow_ptr[i]; s < tb->jrow_ptr[i + 1]; ++s) touched[tb->jcol[s]] = 1;
    }
    std::vector<int> node_of(N, 0);
    for (int v = 0; v < N; ++v) node_of[Y.pos[v]] = v;
    int nl = Y.n_lev;
    for (int j = 0; j < R0; ++j) {
      const int v = node_of[j];
      if (v >= n || touched[v]) nl = std::min(nl, Y.lev[j]);
    }
    P.neg_lev = nl;
    { const char* e = getenv("OMG_B200_EARLY_REJECT"); if (e && atoi(e) == 0) P.neg_lev = 0; }   // experiment knob
  }


  // ---- pair lists of the left-looking gather -----------------------------------------
  // One pair per (target entry, source SUPERNODE): with the rows i, j of the target among the
  // rows R below the supernode's block, the w columns contribute
  //     sum_t x_it x_jt / d_t        (padded entries are zero, so every column may be summed).
  // Pair = {byte offset of (i, first column) | of (j, first column) << 16, byte offset of the
  // supernode's table entry}; the table entry holds the byte distance from a row's entry in the
  // first column to its entry in column t, and where 1/d_t lives (a zero for t >= w).  The
  // segments below merge the pairs of neighbouring entries into the kernel's records.
  std::vector<std::vector<uint2>> plist(Y.Lsize);
  std::vector<uint4> sntab;
  for (int c0 = 0; c0 < R0; ++c0) {
    if (Y.sn_first[c0] != c0) continue;
    const int w = Y.sn_w[c0];
    n_snw[w]++;
    const unsigned snoff = (unsigned)sntab.size() * 16u;
    unsigned dl[4] = {0u, 0u, 0u, 0u}, rr[4];
    for (int t = 0; t < 4; ++t) {
      rr[t] = (unsigned)((t < w) ? (c0 + t) : N) * 8u;             // rd[N] = 0
      if (t > 0 && t < w) dl[t] = (unsigned)((Y.colptr[c0 + t] - t) - Y.colptr[c0]) * 8u;
    }
    sntab.push_back(make_uint4(dl[1] | (dl[2] << 16), dl[3] | (rr[0] << 16), rr[1] | (rr[2] << 16), rr[3]));
    const std::vector<int>& Rl = Y.st[c0 + w - 1];                 // rows below the block
    const int nR = (int)Rl.size();
    const int row0 = Y.colptr[c0] + w;                             // entry (Rl[0], c0)
    for (int bi = 0; bi < nR; ++bi) {
      const int j = Rl[bi];
      for (int ai = bi; ai <= nR; ++ai) {                          // ai == nR: the rhs row
        const int i = (ai < nR) ? Rl[ai] : N;
        const int tgt = Y.idx(i, j);
        if (tgt < 0) { *why = "symbolic structure is not closed"; return false; }
        plist[tgt].push_back(make_uint2(((unsigned)(row0 + ai) * 8u) | (((unsigned)(row0 + bi) * 8u) << 16), snoff));
      }
    }
  }
  for (const std::vector<uint2>& pl : plist) max_gather = std::max(max_gather, (int)pl.size());
  const unsigned sn_dummy = (unsigned)sntab.size() * 16u;           // pad records: 0 * rd[N] * 0
  sntab.push_back(make_uint4(0u, ((unsigned)N * 8u) << 16, ((unsigned)N * 8u) | (((unsigned)N * 8u) << 16), (unsigned)N * 8u));
  if (sntab.size() * 16u >= 65536u) { *why = "too many supernodes"; return false; }
  P.n_sn = (int)sntab.size();
  P.sntab = upload(h, sntab.data(), sntab.size(), &ok);
  std::vector<char> is_eq_pos(N, 0);          // permuted index -> pivot of an equality row
  for (int k = 0; k < n_eq; ++k) is_eq_pos[Y.pos[n + k]] = 1;
  // ---- segments of the gather ----------------------------------------------------------------
  // A segment is up to SP_GQ consecutive stored entries of one column: all of a level column's
  // entries, and on the root the runs of entries with a non-empty list.  Its entries share the row
  // j of every source, so ONE 16-byte record per (segment, source) serves all of them: {byte offset
  // of (j, first column) | table entry << 16, then the byte offsets of (i_q, first column) as 16-bit
  // halves, 0 where the source does not reach entry q}.  The kernel unpacks the table entry and
  // loads A_j. and rd once per record.  Records are the union of the entries' sources in ascending
  // supernode order, so every entry receives its contributions in the order of its pair list.
  static_assert(SP_GQ >= 1 && SP_GQ <= 6, "entry offsets: six 16-bit halves of a record");
  const uint4 padrec = make_uint4(((unsigned)P.zslot * 8u) | (sn_dummy << 16), 0u, 0u, 0u);
  std::vector<int> lev_ptr;
  std::vector<uint4> fdesc, fpair;
  size_t pair_slots = 0;                      // record slots of one record per (entry, source), 2 per uint4
  int n_seg = 0, max_seg_src = 0, seg_mismatch = 0;
  for (int lv = 0; lv <= Y.n_lev; ++lv) {
    std::vector<unsigned> words;              // segment words
    std::vector<std::vector<uint4>> recs;     // records of each segment
    std::vector<size_t> lens;                 // list length of each entry the level gathers
    const bool root = (lv == Y.n_lev);
    for (int j = root ? R0 : 0; j < (root ? N : R0); ++j) {
      if (!root && Y.lev[j] != lv) continue;
      for (int e0 = Y.colptr[j]; e0 < Y.colptr[j + 1];) {
        if (root && plist[e0].empty()) { ++e0; continue; }
        int cnt = 0;
        while (cnt < SP_GQ && e0 + cnt < Y.colptr[j + 1] && !(root && plist[e0 + cnt].empty())) ++cnt;
        std::map<unsigned, uint4> src;        // table entry -> record
        for (int q = 0; q < cnt; ++q) {
          lens.push_back(plist[e0 + q].size());
          for (const uint2& p : plist[e0 + q]) {
            uint4& r = src.emplace(p.y, make_uint4((p.x >> 16) | (p.y << 16), 0u, 0u, 0u)).first->second;
            (&r.y)[q / 2] |= (p.x & 0xffffu) << (16 * (q % 2));
          }
        }
        recs.emplace_back();
        for (const auto& kv : src) recs.back().push_back(kv.second);
        // what the kernel reads back: entry q's (i, j, table entry) in record order = its pair list
        for (int q = 0; q < cnt; ++q) {
          std::vector<uint2> back;
          for (const uint4& r : recs.back()) {
            const unsigned o = ((&r.y)[q / 2] >> (16 * (q % 2))) & 0xffffu;
            if (o) back.push_back(make_uint2(o | ((r.x & 0xffffu) << 16), r.x >> 16));
          }
          const std::vector<uint2>& pl = plist[e0 + q];
          bool same = back.size() == pl.size();
          for (size_t k = 0; same && k < pl.size(); ++k) same = back[k].x == pl[k].x && back[k].y == pl[k].y;
          if (!same) ++seg_mismatch;
        }
        const bool piv = !root && e0 == Y.colptr[j] && Y.sn_w[j] == 1;   // wider supernodes: pivots in the panel step
        if (piv && is_eq_pos[j]) ++eq_lev;
        words.push_back((unsigned)e0 | (root ? 0u : (unsigned)j << 13) | (piv ? (1u << 24) : 0u) |
                        ((piv && is_eq_pos[j]) ? (1u << 25) : 0u) | ((unsigned)(cnt - 1) << 26));
        e0 += cnt;
      }
    }
    // the per-entry layout (slices of 32 entries, lists in words of two pairs) that the structure
    // line's pairs= and max-slices= keep counting
    std::stable_sort(lens.begin(), lens.end(), std::greater<size_t>());
    for (size_t q0 = 0; q0 < lens.size(); q0 += 32) pair_slots += (lens[q0] + 1) / 2 * 64;
    max_slices = std::max(max_slices, (int)((lens.size() + 31) / 32));
    n_seg += (int)recs.size();
    std::vector<int> ord(recs.size());
    for (size_t q = 0; q < ord.size(); ++q) ord[q] = (int)q;
    std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return recs[a].size() > recs[b].size(); });
    lev_ptr.push_back((int)(fdesc.size() / 32));
    for (size_t q0 = 0; q0 < ord.size(); q0 += 32) {
      const unsigned nk = (unsigned)recs[ord[q0]].size();    // records per lane
      max_seg_src = std::max(max_seg_src, (int)nk);
      const unsigned pbase = (unsigned)fpair.size();
      fpair.resize(fpair.size() + (size_t)nk * 32, padrec);
      for (int l = 0; l < 32; ++l) {
        const size_t q = q0 + l;
        if (q >= ord.size()) { fdesc.push_back(make_uint4(0xffffffffu, pbase + l, nk, 0u)); continue; }
        fdesc.push_back(make_uint4(words[ord[q]], pbase + l, nk, 0u));
        for (size_t k = 0; k < recs[ord[q]].size(); ++k) fpair[pbase + k * 32 + l] = recs[ord[q]][k];
      }
    }
  }
  lev_ptr.push_back((int)(fdesc.size() / 32));
  P.lev_ptr = upload(h, lev_ptr.data(), lev_ptr.size(), &ok);
  P.fdesc = upload(h, fdesc.data(), fdesc.size(), &ok);
  P.fpair = upload(h, fpair.data(), fpair.size(), &ok);
  {  // panel tasks of the supernodes (w >= 2), per level in rounds of nt; the rows of the diagonal
     // block come last (their results are stored after the level's closing barrier)
    std::vector<int> tptr;
    std::vector<uint4> tasks;
    for (int lv = 0; lv < Y.n_lev; ++lv) {
      tptr.push_back((int)(tasks.size() / nt));
      std::vector<uint4> rows, blk;
      for (int c0 = 0; c0 < R0; ++c0) {
        if (Y.lev[c0] != lv || Y.sn_first[c0] != c0 || Y.sn_w[c0] < 2) continue;
        const int w = Y.sn_w[c0];
        unsigned eqb = 0, cb[4] = {0u, 0u, 0u, 0u};
        for (int t = 0; t < w; ++t) { cb[t] = (unsigned)Y.colptr[c0 + t] * 8u; if (is_eq_pos[c0 + t]) { eqb |= 1u << t; ++eq_panel; } }
        const int nR = Y.len[c0 + w - 1];                     // rows below the block (+ the rhs row)
        const unsigned head = (unsigned)c0 | ((unsigned)w << 11) | (eqb << 17) | 0x80000000u;
        for (int r = 0; r <= nR; ++r) rows.push_back(make_uint4(head, cb[0] | (cb[1] << 16), cb[2] | (cb[3] << 16), (unsigned)r));
        for (int q = 1; q < w; ++q) blk.push_back(make_uint4(head | ((unsigned)q << 14), cb[0] | (cb[1] << 16), cb[2] | (cb[3] << 16), 0u));
      }
      if ((int)blk.size() > nt) { *why = "too many supernodes on one level"; return false; }
      max_blk = std::max(max_blk, (int)blk.size());
      if (!rows.empty() || !blk.empty()) {
        const size_t tot = rows.size() + blk.size();
        const size_t padded = (tot + nt - 1) / nt * nt;
        std::vector<uint4> lvl(padded, make_uint4(0u, 0u, 0u, 0u));
        for (size_t q = 0; q < rows.size(); ++q) lvl[q] = rows[q];
        for (size_t q = 0; q < blk.size(); ++q) lvl[padded - blk.size() + q] = blk[q];    // last round
        // (rows that would share the last round with the block rows stay where they are: a
        //  thread has at most one task per round)
        if (rows.size() > padded - blk.size()) { *why = "panel round overflow"; return false; }
        max_prounds = std::max(max_prounds, (int)(padded / nt));
        tasks.insert(tasks.end(), lvl.begin(), lvl.end());
      }
    }
    tptr.push_back((int)(tasks.size() / nt));
    if (tasks.empty()) tasks.push_back(make_uint4(0u, 0u, 0u, 0u));
    h->sp_info_extra = " panel-rounds=" + std::to_string(tptr.back());
    P.ptask_ptr = upload(h, tptr.data(), tptr.size(), &ok);
    P.ptask = upload(h, tasks.data(), tasks.size(), &ok);
  }
  {  // root: row chunks, dealt round-robin to the threads (long rows first)
    std::vector<unsigned> chunks;
    for (int i = nr; i >= 0; --i) {
      const int kmax = std::min(i, nr - 1);
      for (int k0 = 0; k0 <= kmax; k0 += SP_RCW) {
        const int cnt = std::min(SP_RCW, kmax - k0 + 1);
        const bool has_diag = (i < nr && k0 <= i && i < k0 + cnt);
        if (has_diag && is_eq_pos[R0 + i]) ++eq_root;
        chunks.push_back((unsigned)i | ((unsigned)k0 << 6) | ((unsigned)cnt << 12) |
                         ((has_diag && is_eq_pos[R0 + i]) ? 0x10000u : 0u));
      }
    }
    if ((int)chunks.size() > SP_RCH * nt) { *why = "root block too large"; return false; }
    std::vector<unsigned> rc((size_t)SP_RCH * nt, 0u);
    for (size_t c = 0; c < chunks.size(); ++c) rc[(c / nt) * nt + (c % nt)] = chunks[c];
    P.root_ch = upload(h, rc.data(), rc.size(), &ok);
  }
  // ---- backward sweep descriptors ---------------------------------------------------------
  // Per level, rounds of nt/8 columns (8 lanes each).  The columns of a supernode sit in
  // consecutive lane groups of ONE warp, first column first: the lanes gather the part of
  // column c that lies outside the supernode (ancestors: already solved), then the warp solves
  // the supernode's own triangle from its last column down with shuffles.
  {
    std::vector<int> brnd;
    std::vector<uint4> bdesc;
    int rounds = 0;
    const int wpr = nt / 32;                                   // warps per round
    for (int lv = 0; lv < Y.n_lev; ++lv) {
      brnd.push_back(rounds);
      std::vector<int> firsts;
      for (int j = 0; j < R0; ++j) if (Y.lev[j] == lv && Y.sn_first[j] == j) firsts.push_back(j);
      std::stable_sort(firsts.begin(), firsts.end(), [&](int a, int b) { return Y.sn_w[a] > Y.sn_w[b]; });
      std::vector<std::vector<int>> bins;                      // warp bins: columns (or -1) of its 4 groups
      for (int c0 : firsts) {
        const int w = Y.sn_w[c0];
        size_t b = 0;
        for (; b < bins.size(); ++b) if ((int)bins[b].size() + w <= 4) break;
        if (b == bins.size()) bins.push_back({});
        for (int t = 0; t < w; ++t) bins[b].push_back(c0 + t);
      }
      int maxlen = 0;
      for (int j = 0; j < R0; ++j) if (Y.lev[j] == lv) {
        int cntj = 0;
        for (int i : Y.st_true[j]) if (!(i < R0 && Y.sn_first[i] == Y.sn_first[j])) ++cntj;
        maxlen = std::max(maxlen, cntj);
      }
      const unsigned nq = (unsigned)std::max(1, (maxlen + 7) / 8);
      max_nq = std::max(max_nq, (int)nq);
      max_brounds = std::max(max_brounds, (int)((bins.size() + wpr - 1) / wpr));
      for (size_t b0 = 0; b0 < bins.size(); b0 += wpr) {
        for (int t = 0; t < nt; ++t) {
          const size_t b = b0 + (size_t)(t >> 5);
          const int grp = (t >> 3) & 3, sub = t & 7;
          const unsigned none = (unsigned)P.zslot * 8u;          // LK[zslot] = 0
          // absent entries: 0 * u[N] -- a slot of u that the sweep sets to zero and never writes again
          // (u[0] would do numerically, but reading it races with the round that solves column 0)
          const unsigned none_ent = none | (((unsigned)N * 8u) << 16);
          unsigned ent[8];
          for (int q = 0; q < 8; ++q) ent[q] = none_ent;
          unsigned h0 = nq << 17, h1 = none, cb8 = none, snw = 0u;
          if (b < bins.size() && grp < (int)bins[b].size()) {
            const int j = bins[b][grp];
            std::vector<int> outs;                               // rows outside the supernode (true non-zeros)
            for (int i : Y.st_true[j]) if (!(i < R0 && Y.sn_first[i] == Y.sn_first[j])) outs.push_back(i);
            for (int q = 0; q < 8; ++q) if (sub + 8 * q < (int)outs.size()) {
              const int i = outs[sub + 8 * q];
              ent[q] = ((unsigned)Y.idx(i, j) * 8u) | (((unsigned)i * 8u) << 16);
            }
            const int w = Y.sn_w[j], q = j - Y.sn_first[j];
            h0 = ((unsigned)j * 8u) | (1u << 16) | (nq << 17) | ((w > 1) ? (1u << 21) : 0u);
            h1 = (unsigned)Y.idx(N, j) * 8u;
            cb8 = (unsigned)Y.colptr[j] * 8u;
            snw = (unsigned)q | ((unsigned)w << 3);
          }
          bdesc.push_back(make_uint4(h0, h1, ent[0], ent[1]));
          bdesc.push_back(make_uint4(ent[2], ent[3], ent[4], ent[5]));
          bdesc.push_back(make_uint4(ent[6], ent[7], cb8, snw));
        }
        ++rounds;
      }
    }
    brnd.push_back(rounds);
    h->sp_info_extra += " back-rounds=" + std::to_string(rounds);
    P.brnd_ptr = upload(h, brnd.data(), brnd.size(), &ok);
    P.bdesc = upload(h, bdesc.data(), bdesc.size(), &ok);
  }
  // ---- index maps ---------------------------------------------------------------------------
  std::vector<int> pos_var(n), pos_eq(std::max(n_eq, 1)), ksign(N, 1), diagidx(N), rhsidx(N);
  for (int j = 0; j < n; ++j) pos_var[j] = Y.pos[j];
  for (int k = 0; k < n_eq; ++k) { pos_eq[k] = Y.pos[n + k]; ksign[Y.pos[n + k]] = -1; }
  for (int j = 0; j < N; ++j) { diagidx[j] = Y.idx(j, j); rhsidx[j] = Y.idx(N, j); }
  P.pos_var = upload(h, pos_var.data(), pos_var.size(), &ok);
  P.pos_eq = upload(h, pos_eq.data(), pos_eq.size(), &ok);
  P.ksign = upload(h, ksign.data(), ksign.size(), &ok);
  P.diagidx = upload(h, diagidx.data(), diagidx.size(), &ok);
  P.rhsidx = upload(h, rhsidx.data(), rhsidx.size(), &ok);
  auto lidx_of = [&](int pa, int pb) { return (pa >= pb) ? Y.idx(pa, pb) : Y.idx(pb, pa); };
  std::vector<char> is_eq(m, 0);
  {
    std::vector<int> jdst(std::max(tb->nnz_j, 1), -1);
    for (int k = 0; k < n_eq; ++k) {
      const int i = tb->kkt_eq_rows[k];
      is_eq[i] = 1;
      for (int s = tb->jrow_ptr[i]; s < tb->jrow_ptr[i + 1]; ++s) {
        jdst[s] = lidx_of(Y.pos[n + k], Y.pos[tb->jcol[s]]);
        if (jdst[s] < 0) { *why = "border entry outside the structure"; return false; }
      }
    }
    P.jdst = upload(h, jdst.data(), jdst.size(), &ok);
    std::vector<uint2> border;
    for (int k = 0; k < n_eq; ++k) {
      const int i = tb->kkt_eq_rows[k];
      for (int s = tb->jrow_ptr[i]; s < tb->jrow_ptr[i + 1]; ++s)
        border.push_back(make_uint2((unsigned)s | ((unsigned)i << 16), (unsigned)jdst[s]));
      border.push_back(make_uint2(0xffffu | ((unsigned)i << 16), (unsigned)rhsidx[Y.pos[n + k]]));
    }
    P.n_border = (int)border.size();
    P.border = upload(h, border.data(), border.size(), &ok);
    std::vector<unsigned short> vd(N);
    for (int j = 0; j < N; ++j) vd[j] = (unsigned short)((unsigned)diagidx[j] | (is_eq_pos[j] ? 0x8000u : 0u));
    P.vdiag = upload(h, vd.data(), vd.size(), &ok);
  }
  std::vector<int> hdst(std::max(tb->nnz_h, 1));
  for (int q = 0; q < tb->nnz_h; ++q) {
    hdst[q] = lidx_of(Y.pos[tb->hrow[q]], Y.pos[tb->hcol[q]]);
    if (hdst[q] < 0) { *why = "H position outside the structure"; return false; }
  }
  // ---- thread streams -------------------------------------------------------------------------
  auto xi_of = [&](const omg_termlist& L, int t, int w) { return (w < L.width) ? L.xi[(size_t)t * L.width + w] : n; };
  auto end16 = [](PT16& r) { r.cidx |= 0x8000u; };
  PT16 pad16; pad16.coef = 0.0; pad16.cidx = 0; pad16.a = (unsigned short)n; pad16.b = (unsigned short)n; pad16.c = 0;
  {  // J: a = n (x[n] = 1.0), b = x0, c = slot
    std::vector<std::vector<PT16>> lists(tb->nnz_j);
    std::vector<PT16> dum(tb->nnz_j);
    for (int s = 0; s < tb->nnz_j; ++s) {
      PT16 d = pad16; d.c = (unsigned short)s; dum[s] = d;
      for (int t = tb->J.ptr[s]; t < tb->J.ptr[s + 1]; ++t) {
        PT16 r; r.coef = tb->J.coef[t]; r.cidx = (unsigned short)tb->J.cidx[t];
        r.a = (unsigned short)n; r.b = (unsigned short)xi_of(tb->J, t, 0); r.c = (unsigned short)s;
        lists[s].push_back(r);
      }
    }
    std::vector<PT16> out;
    sp_build_stream(lists, dum, pad16, end16, nt, out, &P.J.n_chunk);
    P.J.rec = upload(h, out.data(), out.size(), &ok);
  }
  {  // G: a, b = x0, x1, c = row
    std::vector<std::vector<PT16>> lists(m);
    std::vector<PT16> dum(m);
    for (int i = 0; i < m; ++i) {
      PT16 d = pad16; d.c = (unsigned short)i; dum[i] = d;
      for (int t = tb->G.ptr[i]; t < tb->G.ptr[i + 1]; ++t) {
        PT16 r; r.coef = tb->G.coef[t]; r.cidx = (unsigned short)tb->G.cidx[t];
        r.a = (unsigned short)xi_of(tb->G, t, 0); r.b = (unsigned short)xi_of(tb->G, t, 1); r.c = (unsigned short)i;
        lists[i].push_back(r);
      }
    }
    std::vector<PT16> out;
    sp_build_stream(lists, dum, pad16, end16, nt, out, &P.G.n_chunk);
    P.G.rec = upload(h, out.data(), out.size(), &ok);
  }
  {  // W: a = lambda row (m: padding, y[m] = 0; m + 1: the objective, y[m+1] = its factor), b = x0, c = L index
    PT16 padw = pad16; padw.a = (unsigned short)m; padw.c = (unsigned short)P.zslot;
    std::vector<std::vector<PT16>> lists(tb->nnz_w);
    std::vector<PT16> dum(tb->nnz_w, padw);
    for (int q = 0; q < tb->nnz_w; ++q) {
      const int dst = hdst[tb->w2h[q]];
      dum[q].c = (unsigned short)dst;
      for (int t = tb->W.ptr[q]; t < tb->W.ptr[q + 1]; ++t) {
        PT16 r; r.coef = tb->W.coef[t]; r.cidx = (unsigned short)tb->W.cidx[t];
        const int lr = tb->W.lrow ? tb->W.lrow[t] : m;
        r.a = (unsigned short)((lr == m) ? m + 1 : lr); r.b = (unsigned short)xi_of(tb->W, t, 0);
        r.c = (unsigned short)dst;
        lists[q].push_back(r);
      }
    }
    std::vector<PT16> out;
    sp_build_stream(lists, dum, padw, end16, nt, out, &P.W.n_chunk);
    P.W.rec = upload(h, out.data(), out.size(), &ok);
  }
  {  // H: x = s1 | s2<<16, y = row | (dst | diag<<13 | end<<14)<<16
    std::vector<std::vector<uint2>> lists(tb->nnz_h);
    std::vector<uint2> dum(tb->nnz_h);
    for (int q = 0; q < tb->nnz_h; ++q) {
      const unsigned tag = ((unsigned)hdst[q] | ((tb->hrow[q] == tb->hcol[q]) ? (1u << 13) : 0u)) << 16;
      dum[q] = make_uint2(0u, (unsigned)m | tag);
      for (int e = tb->hp_ptr[q]; e < tb->hp_ptr[q + 1]; ++e) {
        const int row = tb->hp_row[e];
        if (is_eq[row]) continue;                 // equality rows sit in the border, Sigma = 0
        lists[q].push_back(make_uint2((unsigned)tb->hp_s1[e] | ((unsigned)tb->hp_s2[e] << 16), (unsigned)row | tag));
      }
    }
    std::vector<uint2> out;
    sp_build_stream(lists, dum, make_uint2(0u, (unsigned)m | ((unsigned)P.zslot << 16)),
                    [](uint2& r) { r.y |= 0x40000000u; }, nt, out, &P.H.n_chunk);
    P.H.rec = upload(h, out.data(), out.size(), &ok);
  }
  {  // C (columns: J^T v): x = slot | row<<16, y = column | rhs L index<<16 | end<<30
    std::vector<std::vector<uint2>> cl(n);
    std::vector<uint2> cd(n);
    auto ctag = [&](int j) { return (unsigned)j | ((unsigned)rhsidx[Y.pos[j]] << 16); };
    for (int j = 0; j < n; ++j) cd[j] = make_uint2((unsigned)m << 16, ctag(j));
    for (int s = 0; s < tb->nnz_j; ++s)
      cl[tb->jcol[s]].push_back(make_uint2((unsigned)s | ((unsigned)tb->jrow[s] << 16), ctag(tb->jcol[s])));
    auto end8 = [](uint2& r) { r.y |= 0x40000000u; };
    std::vector<uint2> out;
    sp_build_stream(cl, cd, make_uint2((unsigned)m << 16, 0u), end8, nt, out, &P.C.n_chunk);
    P.C.rec = upload(h, out.data(), out.size(), &ok);
  }
  {  // R (rows: J dx from the terms): a = x0, b = column, c = row
    std::vector<std::vector<PT16>> lists(m);
    std::vector<PT16> dum(m);
    PT16 padr = pad16; padr.b = (unsigned short)N;
    for (int i = 0; i < m; ++i) {
      PT16 d = padr; d.c = (unsigned short)i; dum[i] = d;
      for (int s = tb->jrow_ptr[i]; s < tb->jrow_ptr[i + 1]; ++s)
        for (int t = tb->J.ptr[s]; t < tb->J.ptr[s + 1]; ++t) {
          PT16 r; r.coef = tb->J.coef[t]; r.cidx = (unsigned short)tb->J.cidx[t];
          r.a = (unsigned short)xi_of(tb->J, t, 0); r.b = (unsigned short)tb->jcol[s]; r.c = (unsigned short)i;
          lists[i].push_back(r);
        }
    }
    std::vector<PT16> out;
    sp_build_stream(lists, dum, padr, end16, nt, out, &P.R.n_chunk);
    P.R.rec = upload(h, out.data(), out.size(), &ok);
  }
  if (!ok) { *why = "device allocation/upload failed"; return false; }

  // ---- shared-memory / scratch layout ---------------------------------------------------------
  SpSmem& S = h->SS;
  int off = 0;
  auto take = [&](int cnt) { int o = off; off += (cnt + 1) & ~1; return o; };
  S.LK = take(std::max(P.Lsz, tb->nnz_j + 2)); S.jval = S.LK;   // the factor is staged over the Jacobian values
  S.xe = take(n + 2); S.xt = take(N + 2); S.dx = take(N + 2); S.gf = take(n + 2);
  S.rd = take(N + 2); S.diag0 = S.rd; S.V = take(tb->n_v);   // rd holds |K_jj| until column j is pivoted
  S.sig = take(m + 2); S.y = take(m + 2);
  S.red = take((nt / 32) * NRED); S.filt = take(2 * MAXF);
  S.rt8 = take((m + 7) / 8); S.rki = 0;
  S.lptr = take((3 * Y.n_lev + 6 + 1) / 2 + 1);
  S.sntab = take(2 * P.n_sn);
  S.total = off;
  int goff = 0;
  auto gtake = [&](int cnt) { int o = goff; goff += (cnt + 1) & ~1; return o; };
  S.Kc = gtake(P.Lsz);
  S.g = gtake(m + 2); S.s = gtake(m + 2); S.zU = gtake(m + 2); S.dsc = gtake(m + 2);
  S.ds = gtake(m + 2); S.gt = gtake(m + 2); S.wv = gtake(m + 2); S.zL = gtake(m + 2); S.yg = gtake(m + 2);
  // what an iteration touches: everything but the trial Jacobian of soft restoration
  const size_t touched = (size_t)goff * sizeof(double);
  S.jt = gtake(tb->nnz_j + 2);
  S.gtotal = goff;
  h->sp_smem_bytes = (size_t)off * sizeof(double);
  const void* kfn = (const void*)omg_ipm_kernel_sp;
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, kfn) != cudaSuccess) { *why = "cudaFuncGetAttributes failed"; return false; }
  if (h->sp_smem_bytes + fa.sharedSizeBytes > (size_t)prop.sharedMemPerBlockOptin) { *why = "does not fit shared memory"; return false; }
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)((size_t)prop.sharedMemPerBlockOptin - fa.sharedSizeBytes)) != cudaSuccess) {
    *why = "cudaFuncSetAttribute failed"; return false; }
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, nt, h->sp_smem_bytes);
  if (occ < 1) { *why = "zero occupancy"; return false; }
  h->sp_ctas = occ;
  h->sp_dscr_stride = goff + 8;
  h->sp_info = "sparse LDL^T: N=" + std::to_string(N) + " nnz(L)=" + std::to_string(Y.Lsize) +
               h->sp_info_extra + " levels=" + std::to_string(Y.n_lev) + " (early-reject " + std::to_string(P.neg_lev) + ")" + " root=" + std::to_string(nr) +
               " pairs=" + std::to_string(pair_slots) + " nt=" + std::to_string(nt) +
               " ctas/SM=" + std::to_string(occ) + " smem=" + std::to_string(h->sp_smem_bytes) +
               " scratch/iter=" + std::to_string(touched);
  auto kv = [&](const char* k, int v) { h->sp_info += std::string(" ") + k + "=" + std::to_string(v); };
  h->sp_info += " |";
  kv("eqpiv-level", eq_lev); kv("eqpiv-panel", eq_panel); kv("eqpiv-root", eq_root);
  for (int w = 1; w <= SP_SNW; ++w) kv(("sn" + std::to_string(w)).c_str(), n_snw[w]);
  kv("zeros", Y.n_pad); kv("max-sn-zeros", Y.max_sn_pad); kv("max-col", max_col);
  kv("max-gather", max_gather); kv("max-nq", max_nq); kv("max-slices", max_slices);
  kv("max-block-rows", max_blk); kv("max-panel-rounds", max_prounds); kv("max-back-rounds", max_brounds);
  kv("root-mod4", nr % 4);
  kv("segments", n_seg); kv("seg-records", (int)fpair.size()); kv("max-seg-sources", max_seg_src);
  kv("seg-mismatch", seg_mismatch);
  return true;
}
