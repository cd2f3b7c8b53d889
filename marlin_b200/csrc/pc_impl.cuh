// The polynomial-commitment layer of MarlinKZG10 and SonicKZG10 over polynomials resident in HBM: `PC::commit` and
// `PC::open_combinations` [U ark-poly-commit 0.3 marlin_pc / sonic_pc].  `Marlin::index`, `Marlin::prove` and the Level-1
// C ABI all commit and open through here.
#pragma once
#include <algorithm>
#include <vector>

#include "capi_types.cuh"
#include "hostutil.hpp"
#include "poly_impl.cuh"

namespace b2m {

// ---- small host-side polynomials (the KZG10 blinding polynomials) -------------------------------
template <class Fr>
void hp_axpy(std::vector<Fr>& acc, const Fr& k, const std::vector<Fr>& p) {
  if (acc.size() < p.size()) acc.resize(p.size(), Fr::zero());
  for (size_t i = 0; i < p.size(); i++) acc[i] = acc[i] + k * p[i];
}
template <class Fr>
Fr hp_eval(const std::vector<Fr>& p, const Fr& z) {
  Fr acc = Fr::zero();
  for (size_t i = p.size(); i-- > 0;) acc = acc * z + p[i];
  return acc;
}
template <class Fr>
std::vector<Fr> hp_div_linear(const std::vector<Fr>& p, const Fr& z) {  // quotient of p / (X - z)
  if (p.size() <= 1) return std::vector<Fr>();
  std::vector<Fr> q(p.size() - 1);
  Fr acc = Fr::zero();
  for (size_t i = p.size() - 1; i >= 1; i--) {
    acc = p[i] + acc * z;
    q[i - 1] = acc;
  }
  return q;
}
template <class Fr>
bool hp_is_zero(const std::vector<Fr>& p) {
  for (auto& c : p)
    if (!c.is_zero()) return false;
  return true;
}

template <class Fr>
struct LcTerms {  // out[i] = sum_t coef[t] * (off[t] <= i < off[t] + len[t] ? src[t][i - off[t]] : 0)
  static constexpr int MAX = 8;
  const Fr* src[MAX];
  size_t off[MAX], len[MAX];
  Fr coef[MAX];
  int n = 0;
  void add(const Fr* p, size_t l, const Fr& c, size_t o = 0) {
    src[n] = p; off[n] = o; len[n] = l; coef[n] = c; n++;
  }
};
// `out` may be one of the sources if its offset is 0: every thread reads its element before it writes it
template <class Fr>
__global__ void lincomb_kernel(LcTerms<Fr> t, size_t n, Fr* out) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr acc = Fr::zero();
  for (int k = 0; k < t.n; k++)
    if (i >= t.off[k] && i - t.off[k] < t.len[k]) acc = acc + t.coef[k] * ld_fr(t.src[k] + (i - t.off[k]));
  st_fr(out + i, acc);
}
template <class Fr>
void launch_lincomb(Ctx& cx, const LcTerms<Fr>& lt, size_t n_out, Fr* dst) {
  lincomb_kernel<Fr><<<div_up(n_out, 256), 256, 0, cx.stream>>>(lt, n_out, dst);
  B2M_CHECK_LAUNCH();
  cx.launches++;
}

// The witness MSMs of one or more opening points [U marlin_pc open].  A point's witness is its plain witness scalars against
// powers_of_g[0 ..), its hiding witness against the gamma powers and, for MarlinKZG10, one shifted witness per degree-bounded
// polynomial against powers_of_g[D - bound ..].  Each shifted witness is only ever added to its point's witness and an MSM is
// linear in its scalars, so a shifted witness whose slice overlaps the plain slice, or starts at most MERGE_GAP powers past
// its end, is summed into the plain scalars: one MSM over the union of the slices.  A shifted witness farther away stays an
// MSM of its own in an earlier batch, and its result enters the point's MSM as an `extra` term: merging it would widen the
// plain MSM by up to D zero scalars for a small bounded polynomial under a large key.
template <class Fr, class Fq>
struct WitnessMsms {
  struct Shifted {  // coef * src[i] pairs with powers_of_g[off + i], i < n
    const Fr* src;
    Fr coef;
    size_t n, off;
  };
  // A zero scalar has no digits: it costs the counting sort a few bytes and the bucket pass nothing.  A separate MSM costs its
  // own sort and bucket reduction, and a whole batch (with its host round trip) when no other separate MSM shares it.
  static constexpr size_t MERGE_GAP = 1024;

  Ctx& cx;
  std::vector<MsmJob<Fr, Fq>> pre, fin;  // the separate shifted witnesses; one MSM per point
  std::vector<DBuf<Fr>> keep_sc;
  std::vector<DBuf<XYZZ<Fq>>> keep_pt;
  explicit WitnessMsms(Ctx& c) : cx(c) {}

  // plain[0 .. n) may be overwritten; hw against the gamma powers from slot gslot; the affine witness goes to out (device)
  void add_point(Fr* plain, size_t n, std::vector<Shifted> shifted, const std::vector<Fr>& hw, size_t gslot, Affine<Fq>* out) {
    std::sort(shifted.begin(), shifted.end(), [](const Shifted& a, const Shifted& b) { return a.off < b.off; });
    std::vector<Shifted> merged, apart;
    size_t end = n;
    for (const Shifted& s : shifted) {
      if (s.n == 0) continue;
      if (s.off <= end + MERGE_GAP) {
        merged.push_back(s);
        end = std::max(end, s.off + s.n);
      } else {
        apart.push_back(s);
      }
    }
    Fr* sc = plain;
    if (end > n) {
      keep_sc.emplace_back(cx, end);
      sc = keep_sc.back().p;
    }
    constexpr size_t per_pass = LcTerms<Fr>::MAX - 1;
    for (size_t at = 0; at < merged.size(); at += per_pass) {
      LcTerms<Fr> lt;
      if (at == 0) lt.add(plain, n, Fr::one());
      else lt.add(sc, end, Fr::one());
      for (size_t k = at; k < std::min(merged.size(), at + per_pass); k++) lt.add(merged[k].src, merged[k].n, merged[k].coef, merged[k].off);
      launch_lincomb(cx, lt, end, sc);
    }
    DBuf<XYZZ<Fq>> ex(cx, std::max<size_t>(apart.size(), 1));
    for (size_t k = 0; k < apart.size(); k++) {
      keep_sc.emplace_back(cx, apart[k].n);
      LcTerms<Fr> lt;
      lt.add(apart[k].src, apart[k].n, apart[k].coef);
      launch_lincomb(cx, lt, apart[k].n, keep_sc.back().p);
      pre.push_back(MsmJob<Fr, Fq>{keep_sc.back().p, true, apart[k].n, apart[k].off, nullptr, 0, 0, nullptr, 0, ex.p + k, nullptr});
    }
    const Fr* hw_dev = nullptr;
    if (!hw.empty()) {
      keep_sc.emplace_back(cx, hw.size());
      keep_sc.back().upload(hw.data(), hw.size());
      hw_dev = keep_sc.back().p;
    }
    fin.push_back(MsmJob<Fr, Fq>{sc, true, end, 0, hw_dev, hw.size(), gslot, ex.p, (int)apart.size(), nullptr, out});
    keep_pt.push_back(std::move(ex));
  }
  // the separate shifted witnesses first: their results are `extra` terms of the points' MSMs
  void run(Msm<Fr, Fq>& msm) {
    for (size_t at = 0; at < pre.size(); at += MSM_MAX_BATCH) msm.run_batch(pre.data() + at, (int)std::min<size_t>(MSM_MAX_BATCH, pre.size() - at));
    for (size_t at = 0; at < fin.size(); at += MSM_MAX_BATCH) msm.run_batch(fin.data() + at, (int)std::min<size_t>(MSM_MAX_BATCH, fin.size() - at));
  }
};

// A labelled polynomial living in HBM, with its commitment and its kzg10::Randomness (host blinding polynomials; empty when
// it is not hiding).  A host-resident index's polynomials live in pinned host memory instead (`host`): pc_open streams them.
template <class Fr, class Fq>
struct LabeledPoly {
  const Fr* p = nullptr;
  size_t len = 0;
  bool host = false;    // p is pinned host memory (an index polynomial of a host-resident index; never bounded or hiding)
  int64_t bound = -1;   // degree bound, or -1
  int64_t hiding = -1;  // hiding bound, or -1
  std::vector<Fr> rand, shifted_rand;
  Affine<Fq> comm, shifted_comm;  // shifted_comm: MarlinKZG10, bounded polynomials only (the identity otherwise)
};

// Streams vectors held in pinned host memory to the device in chunks of INDEX_STREAM_CHUNK elements, double-buffered: chunk
// j of every vector is copied into slot j % 2 on the index's own copy stream (not cx.side, which the MSM's counting sort
// uses) while the consumer of chunk j - 1 reads the other slot on cx.stream.  Events order each slot's copy before its
// consumer and the consumer before the slot's next copy.  Each vector crosses PCIe once per call.
template <class Fr>
struct HostStager {
  Ctx& cx;
  cudaStream_t copy;
  size_t bytes = 0;                                          // streamed by this stager
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> copies;   // first to last copy of each call, on the copy stream
  HostStager(Ctx& c, cudaStream_t s) : cx(c), copy(s) {}
  HostStager(const HostStager&) = delete;
  ~HostStager() {
    for (auto& e : copies) {
      cudaEventDestroy(e.first);
      cudaEventDestroy(e.second);
    }
  }
  // milliseconds the copy engine spent on the calls so far (waits for them)
  double copy_ms() {
    double ms = 0;
    for (auto& e : copies) {
      float t = 0;
      B2M_CUDA(cudaEventSynchronize(e.second));
      B2M_CUDA(cudaEventElapsedTime(&t, e.first, e.second));
      ms += t;
    }
    return ms;
  }
  // consume(slot, stride, at, m) launches on cx.stream a kernel reading elements [at, at + m) of vector v at slot + v * stride
  template <class F>
  void stream(const char* span, const Fr* const* src, int nv, size_t n, F&& consume) {
    if (n == 0 || nv == 0) return;
    B2M_REQUIRE(nv <= INDEX_STREAM_VECS, B2M_ERR_INVALID_ARG, "%d streamed vectors, at most %d", nv, INDEX_STREAM_VECS);
    const size_t chunk = std::min(n, INDEX_STREAM_CHUNK);
    DBuf<Fr> slot[2] = {DBuf<Fr>(cx, nv * chunk), DBuf<Fr>(cx, nv * chunk)};
    cudaEvent_t ready, copied[2], consumed[2], t0, t1;
    B2M_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    for (int s = 0; s < 2; s++) {
      B2M_CUDA(cudaEventCreateWithFlags(&copied[s], cudaEventDisableTiming));
      B2M_CUDA(cudaEventCreateWithFlags(&consumed[s], cudaEventDisableTiming));
    }
    B2M_CUDA(cudaEventCreate(&t0));
    B2M_CUDA(cudaEventCreate(&t1));
    B2M_CUDA(cudaEventRecord(ready, cx.stream));  // the slots' stream-ordered allocation, and whatever came before
    B2M_CUDA(cudaStreamWaitEvent(copy, ready, 0));
    B2M_CUDA(cudaEventRecord(t0, copy));
    Ctx::Span prof{"index_h2d", 0.0, nullptr, nullptr};  // b2m_ctx_profile: the copies as a span of their own, on the copy stream
    if (cx.profiling) {
      B2M_CUDA(cudaEventCreate(&prof.a));
      B2M_CUDA(cudaEventCreate(&prof.b));
      B2M_CUDA(cudaEventRecord(prof.a, copy));
    }
    for (size_t at = 0, j = 0; at < n; at += chunk, j++) {
      const int s = (int)(j & 1);
      const size_t m = std::min(chunk, n - at);
      if (j >= 2) B2M_CUDA(cudaStreamWaitEvent(copy, consumed[s], 0));
      for (int v = 0; v < nv; v++)
        B2M_CUDA(cudaMemcpyAsync(slot[s].p + v * chunk, src[v] + at, m * sizeof(Fr), cudaMemcpyHostToDevice, copy));
      if (at + m == n) {  // the last copy: timed before the event cx.stream waits on, so a sync of cx.stream covers them
        B2M_CUDA(cudaEventRecord(t1, copy));
        if (cx.profiling) B2M_CUDA(cudaEventRecord(prof.b, copy));
      }
      B2M_CUDA(cudaEventRecord(copied[s], copy));
      B2M_CUDA(cudaStreamWaitEvent(cx.stream, copied[s], 0));
      const size_t sp = cx.span_begin(span, (double)m);
      consume((const Fr*)slot[s].p, chunk, at, m);
      cx.span_end(sp);
      B2M_CUDA(cudaEventRecord(consumed[s], cx.stream));
    }
    const size_t moved = (size_t)nv * n * sizeof(Fr);
    bytes += moved;
    copies.push_back({t0, t1});
    if (cx.profiling) {
      prof.units = (double)moved;
      cx.spans.push_back(prof);
    }
    // (destroying an event still pending in a stream releases it once it completes)
    cudaEventDestroy(ready);
    for (int s = 0; s < 2; s++) {
      cudaEventDestroy(copied[s]);
      cudaEventDestroy(consumed[s]);
    }
  }
};

// out[at + i] += sum_t c[t] * slot[t * stride + i], i < m: host terms of a combination, one streamed chunk at a time
template <class Fr>
struct StreamTerms {
  Fr c[INDEX_STREAM_VECS];
  int n;
};
template <class Fr>
__global__ void index_stream_lincomb_kernel(StreamTerms<Fr> t, const Fr* __restrict__ slot, size_t stride, size_t m, Fr* out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  Fr acc = ld_fr(out + i);
  for (int k = 0; k < t.n; k++) acc = acc + t.c[k] * ld_fr(slot + k * stride + i);
  st_fr(out + i, acc);
}

// `PC::commit`: draws the blinding polynomials from zk in the reference's order (per polynomial: its randomness, then, for a
// bounded polynomial under MarlinKZG10, its shifted randomness) and runs the KZG10 commitments in batches of MSM_MAX_BATCH.
// MarlinKZG10 commits a bounded polynomial twice, against powers_of_g[0 ..] and against its shifted powers powers_of_g[D -
// bound ..], blinded by gamma powers 0, 1, ..; SonicKZG10 commits it once, against the shifted powers, blinded by the gamma
// powers D - bound, D - bound + 1, .. (shifted_powers_of_gamma_g[bound]).
template <class Fr, class Fq>
void pc_commit(b2m_srs* srs, Msm<Fr, Fq>& msm, int pc, const std::vector<LabeledPoly<Fr, Fq>*>& polys, ZkSource<b2m_rng>& zk) {
  using Pt = Affine<Fq>;
  Ctx& cx = srs->ctx->cx;
  const size_t D = srs->n_g - 1;
  std::vector<DBuf<Fr>> blind;
  std::vector<MsmJob<Fr, Fq>> jobs;
  DBuf<Pt> out(cx, 2 * polys.size());
  out.zero();  // the shifted slot of an unbounded polynomial is never written
  // one KZG10::commit: the coefficients against powers_of_g[off ..], the blinding polynomial (drawn here, degree hiding + 1)
  // against the gamma powers gpow, gpow + 1, .., which must sit in consecutive slots
  auto kzg_commit = [&](const LabeledPoly<Fr, Fq>& q, size_t off, size_t gpow, std::vector<Fr>& r, Pt* dst) {
    r.clear();
    size_t gslot = 0;
    const Fr* s2 = nullptr;
    if (q.hiding >= 0) {
      for (int64_t k = 0; k < q.hiding + 2; k++) r.push_back(field_rand<Fr>(zk));
      gslot = srs->gamma_slot(gpow);
      for (size_t k = 1; k < r.size(); k++)
        B2M_REQUIRE(srs->gamma_slot(gpow + k) == gslot + k, B2M_ERR_INVALID_ARG, "gamma powers are not consecutive");
      blind.emplace_back(cx, r.size());
      blind.back().upload(r.data(), r.size());
      s2 = blind.back().p;
    }
    jobs.push_back(MsmJob<Fr, Fq>{q.p, true, q.len, off, s2, r.size(), gslot, nullptr, 0, nullptr, dst});
  };
  for (size_t i = 0; i < polys.size(); i++) {
    LabeledPoly<Fr, Fq>& q = *polys[i];
    const size_t shift = q.bound >= 0 ? D - (size_t)q.bound : 0;
    if (pc == B2M_PC_MARLIN_KZG10) {
      kzg_commit(q, 0, 0, q.rand, out.p + 2 * i);
      if (q.bound >= 0) kzg_commit(q, shift, 0, q.shifted_rand, out.p + 2 * i + 1);
    } else {
      kzg_commit(q, shift, shift, q.rand, out.p + 2 * i);
    }
  }
  for (size_t at = 0; at < jobs.size(); at += MSM_MAX_BATCH)
    msm.run_batch(jobs.data() + at, (int)std::min<size_t>(MSM_MAX_BATCH, jobs.size() - at));
  std::vector<Pt> h(2 * polys.size());
  out.download(h.data(), h.size());
  for (size_t i = 0; i < polys.size(); i++) {
    polys[i]->comm = h[2 * i];
    polys[i]->shifted_comm = h[2 * i + 1];
  }
}

// A linear combination queried at a point.  LCTerm::One terms affect the evaluation only and are left out.  A degree-bounded
// polynomial appears alone with coefficient one; its quotient by (X - z) is given in `quot` (len - 1 coefficients) when the
// caller already has it, and computed here otherwise.
template <class Fr, class Fq>
struct OpenLc {
  struct Term {
    const LabeledPoly<Fr, Fq>* poly;
    Fr coef;
  };
  std::vector<Term> terms;
  const Fr* quot = nullptr;
};
template <class Fr, class Fq>
struct OpenPoint {
  Fr z;
  std::vector<OpenLc<Fr, Fq>> lcs;  // in label order
};
template <class Fr, class Fq>
struct Opening {
  Affine<Fq> w;
  bool hiding;  // random_v is Some
  Fr random_v;
};

// `PC::open_combinations` [U marlin_pc / sonic_pc open_combinations_individual_opening_challenges] at every point at once.  At
// each point the opening challenges xi^0, xi^1, .. go to its combinations in order, and under MarlinKZG10 one more to the
// shifted part of each bounded one.  A point's combination sum_k ch_k * lc_k is formed by as few lincomb_kernel launches as
// hold its terms; the witness MSMs of all points share one WitnessMsms and all witnesses come back in one download.  Terms in
// pinned host memory (LabeledPoly::host, which needs a stager) are added to the combination afterwards, streamed chunk by
// chunk, INDEX_STREAM_VECS at a time.
template <class Fr, class Fq>
std::vector<Opening<Fr, Fq>> pc_open(b2m_srs* srs, Msm<Fr, Fq>& msm, int pc, const Fr& xi, const std::vector<OpenPoint<Fr, Fq>>& points,
                                     HostStager<Fr>* stager = nullptr) {
  typedef typename WitnessMsms<Fr, Fq>::Shifted Shifted;
  Ctx& cx = srs->ctx->cx;
  const size_t D = srs->n_g - 1;
  const bool marlin = pc == B2M_PC_MARLIN_KZG10;
  const Fr one = Fr::one();
  DBuf<Affine<Fq>> w(cx, points.size());
  WitnessMsms<Fr, Fq> wit(cx);
  std::vector<Opening<Fr, Fq>> res(points.size());
  for (size_t p = 0; p < points.size(); p++) {
    const Fr& z = points[p].z;
    struct Weighted {
      const Fr* src;
      size_t len;
      Fr c;
    };
    std::vector<Weighted> flat, host;
    std::vector<Shifted> shifted;
    std::vector<Fr> r, sr, srw;  // combined randomness, shifted randomness, shifted randomness / (X - z)
    size_t n = 1;
    Fr ch = one;
    for (const auto& lc : points[p].lcs) {
      std::vector<Fr> lr;
      for (const auto& t : lc.terms) {
        (t.poly->host ? host : flat).push_back(Weighted{t.poly->p, t.poly->len, ch * t.coef});
        n = std::max(n, t.poly->len);
        hp_axpy(lr, t.coef, t.poly->rand);
      }
      hp_axpy(r, ch, lr);
      ch = ch * xi;
      const LabeledPoly<Fr, Fq>* b = lc.terms.size() == 1 && lc.terms[0].poly->bound >= 0 ? lc.terms[0].poly : nullptr;
      if (!marlin || !b) continue;
      if (b->len > 1) {  // shifted witness ch * (p / (X - z)) against shifted_powers: powers_of_g[D - bound ..]
        const Fr* quot = lc.quot;
        if (!quot) {
          wit.keep_sc.emplace_back(cx, b->len);
          rec_suffix<Fr>(cx, b->p, wit.keep_sc.back().p, b->len, 1, z, true);
          quot = wit.keep_sc.back().p + 1;
        }
        shifted.push_back(Shifted{quot, ch, b->len - 1, D - (size_t)b->bound});
      }
      hp_axpy(sr, ch, b->shifted_rand);
      if (!hp_is_zero(b->shifted_rand)) hp_axpy(srw, ch, hp_div_linear(b->shifted_rand, z));
      ch = ch * xi;
    }
    DBuf<Fr> comb(cx, n), sfx(cx, n);
    if (flat.empty()) comb.zero();
    for (size_t at = 0; at < flat.size();) {  // the first launch takes MAX terms, later ones MAX - 1 and the running sum
      LcTerms<Fr> lt;
      if (at > 0) lt.add(comb.p, n, one);
      for (; lt.n < LcTerms<Fr>::MAX && at < flat.size(); at++) lt.add(flat[at].src, flat[at].len, flat[at].c);
      launch_lincomb(cx, lt, n, comb.p);
    }
    if (!host.empty()) {
      B2M_REQUIRE(stager != nullptr, B2M_ERR_INVALID_ARG, "a host-resident polynomial needs a stager");
      for (size_t at = 0; at < host.size(); at += INDEX_STREAM_VECS) {
        const Fr* src[INDEX_STREAM_VECS];
        StreamTerms<Fr> st;
        st.n = (int)std::min<size_t>(INDEX_STREAM_VECS, host.size() - at);
        size_t len = 0;
        for (int k = 0; k < st.n; k++) {
          src[k] = host[at + k].src;
          st.c[k] = host[at + k].c;
          len = std::max(len, host[at + k].len);
        }
        for (int k = 0; k < st.n; k++)
          B2M_REQUIRE(host[at + k].len == len, B2M_ERR_INVALID_ARG, "streamed terms of one pass differ in length");
        Fr* out = comb.p;
        stager->stream("index_open_lincomb", src, st.n, len, [&](const Fr* slot, size_t stride, size_t off, size_t m) {
          index_stream_lincomb_kernel<Fr><<<div_up(m, 256), 256, 0, cx.stream>>>(st, slot, stride, m, out + off);
          B2M_CHECK_LAUNCH();
          cx.launches++;
        });
      }
    }
    // S[0] = comb(z), S[1 ..] = comb / (X - z): the plain witness; r / (X - z) plus the shifted part: the hiding witness
    rec_suffix<Fr>(cx, comb.p, sfx.p, n, 1, z, true);
    res[p].hiding = !hp_is_zero(r);
    std::vector<Fr> hw = res[p].hiding ? hp_div_linear(r, z) : std::vector<Fr>();
    hp_axpy(hw, one, srw);
    wit.add_point(sfx.p + 1, n - 1, shifted, hw, hw.empty() ? 0 : srs->gamma_slot(0), w.p + p);
    // Both buffers live until the MSMs have run: released here, they left the stream-ordered pool in a state where later
    // allocations of the prover's opening intermittently blocked in cudaMallocAsync for up to 0.3 s (H100, 2^20).
    wit.keep_sc.push_back(std::move(sfx));
    wit.keep_sc.push_back(std::move(comb));
    res[p].random_v = res[p].hiding ? hp_eval(r, z) + hp_eval(sr, z) : Fr::zero();
  }
  wit.run(msm);
  std::vector<Affine<Fq>> h(points.size());
  w.download(h.data(), h.size());
  for (size_t p = 0; p < points.size(); p++) res[p].w = h[p];
  return res;
}

}  // namespace b2m
