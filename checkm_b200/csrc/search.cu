// search.cu -- the search driver: launches the filter cascade and the domain-definition stages on the engine's
// stream and assembles the hit table.  Replaces the body of `hmmsearch` behind checkm/hmmer.py:61-74.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>
#include "engine.hpp"
#include "stages.hpp"
#include "pool.hpp"

using namespace ckm;

namespace ckm {

std::atomic<int> g_live_engines{0};     // engines alive in this process: they share the envelope-scratch budget
thread_local ckm_engine *g_pool_engine = nullptr;
thread_local int g_pool_next = 0;
// the trace ensemble of the multi-domain regions (kernels_ensemble.cu)
constexpr int X_NX_HOST = 6;
struct EnsembleJob;
int ensembles_launch(ckm_engine *e, const ckm_models *m, DomdefParams &p, const std::vector<PairWork> &pairs,
                     const std::vector<Region> &regs, const std::vector<int> &multi_idx, const std::vector<EnsembleCaps> &caps,
                     cudaStream_t st, EnsembleJob **job_out);
int ensembles_collect(EnsembleJob *job, cudaStream_t st, std::vector<std::vector<Envelope>> &out, std::vector<EnsembleCaps> &grow, int *n_over);
void ensembles_abandon(EnsembleJob *job, cudaStream_t st);
enum { CTR_UNIT4 = 0, CTR_UNIT8, CTR_UNIT16, CTR_UNIT32, CTR_CAND, CTR_MSV, CTR_BIAS, CTR_VIT, CTR_FWD, CTR_ENV, CTR_DOM, CTR_VREDO, CTR_SSVRES, CTR_VWORK = 16 /* .. 25: cursors of the packed-Viterbi class kernels */, CTR_N = 32 };
// timing events of a search (e->ev): the start of each cascade stage and its end, the domain stage, the whole call
enum { EV_SSV = 0, EV_MSV, EV_BIAS, EV_VIT, EV_FWD, EV_CASCADE_END, EV_DOMDEF, EV_END, EV_CALL };

static int64_t env_scratch_budget() {
  // CKM_ENV_SCRATCH_MB (a positive number of MiB, read on every search) replaces the rule below for each engine: a small
  // budget splits the envelopes of any batch into many waves, a large one keeps them in one.  The waves change no result.
  if (const char *v = std::getenv("CKM_ENV_SCRATCH_MB")) {
    char *end = nullptr;
    const long long mb = std::strtoll(v, &end, 10);
    if (end != v && *end == '\0' && mb > 0) return (int64_t)std::min<long long>(mb, (long long)1 << 30) * ((int64_t)1 << 20) / (int64_t)sizeof(float);
  }
  // fixed scratch budget (the cached pool is reused by every later search): 40% of the device shared by the live engines,
  // at most 56 GiB each.  The rest holds each engine's other workspace (for a batch of 32 bins x 5,000 models ~10 GB of
  // Forward/Backward special-state columns and lists), the sequence and model databases, and the caller's own buffers --
  // on an 80 GB H100 running two engines, 2 x 16 GB of scratch leave ~48 GB for them.
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  const size_t neng = (size_t)std::max(1, g_live_engines.load());
  return (int64_t)std::min<size_t>(total_b * 4 / 10 / neng, (size_t)56 << 30) / (int64_t)sizeof(float);
}
// The runtime knobs (INTEGRATION.md §5), read once at the start of every call: CKM_BLK, CKM_VITP (only with blk),
// CKM_SSV_RESOLVE, CKM_TRACE, CKM_ENS_FIRST (-1 unset: automatic order), the envelope scratch budget in floats (only for the
// calls that rescore envelopes; after cudaSetDevice: it depends on the device).
struct SearchKnobs { bool blk, vitp, ssv_resolve, trace; int ens_first; int64_t env_budget; };
static SearchKnobs read_knobs(bool envelopes) {
  auto starts = [](const char *name, char c) { const char *v = std::getenv(name); return v != nullptr && v[0] == c; };
  SearchKnobs k;
  k.blk = !starts("CKM_BLK", '0');
  k.vitp = k.blk && !starts("CKM_VITP", '0');
  k.ssv_resolve = !starts("CKM_SSV_RESOLVE", '0');
  k.trace = starts("CKM_TRACE", '1');
  const char *ens = std::getenv("CKM_ENS_FIRST");
  k.ens_first = ens == nullptr ? -1 : (ens[0] == '0' ? 0 : 1);
  k.env_budget = envelopes ? env_scratch_budget() : 0;
  return k;
}
// CKM_TRACE=1: host-side wall-clock marks of one search on stderr (where the time between the CUDA events goes)
struct Trace {
  bool on; std::chrono::steady_clock::time_point t0, last;
  explicit Trace(bool on_) : on(on_) { t0 = last = std::chrono::steady_clock::now(); }
  void mark(const char *what) {
    if (!on) return;
    const auto now = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[ckm trace] %-28s +%8.3f ms  (%9.3f)\n", what, std::chrono::duration<double, std::milli>(now - last).count(),
                 std::chrono::duration<double, std::milli>(now - t0).count());
    last = now;
  }
};

static int cls_of(int M, bool use_blk) { return use_blk ? blk_class(vq_of(M)) : N_BLK_CLASSES; }

// the per-class launches of one stage go to the engine's class streams: fork after the main stream, join back into it
static int fan_out(ckm_engine *e) {
  CKM_CUDA(cudaEventRecord(e->fan_ev, e->stream));
  for (auto &s : e->cls) CKM_CUDA(cudaStreamWaitEvent(s, e->fan_ev, 0));
  return CKM_OK;
}
static int fan_in(ckm_engine *e) {
  for (int c = 0; c < ckm_engine::NCLS; ++c) {
    CKM_CUDA(cudaEventRecord(e->cls_ev[c], e->cls[c]));
    CKM_CUDA(cudaStreamWaitEvent(e->stream, e->cls_ev[c], 0));
  }
  return CKM_OK;
}

// One stage, one launch per class on that class's stream: `blocked` for the lane-block classes (with p.use_blk), `unblocked`
// (if any) for the models beyond them; grids of blk_per_sm / per_sm CTAs per SM.
template <class P> static int per_class(ckm_engine *e, const P &p, int (*blocked)(const P &, int, int, cudaStream_t), int blk_per_sm,
                                        int (*unblocked)(const P &, int, cudaStream_t), int per_sm, bool widest_first = false) {
  const int nsm = e->prop.multiProcessorCount;
  int rc;
  if ((rc = fan_out(e))) return rc;
  for (int i = 0; i < ckm_engine::NCLS; ++i) {
    const int c = widest_first ? ckm_engine::NCLS - 1 - i : i;
    if (c == N_BLK_CLASSES) rc = unblocked ? unblocked(p, nsm * per_sm, e->cls[c]) : CKM_OK;
    else rc = p.use_blk ? blocked(p, c, nsm * blk_per_sm, e->cls[c]) : CKM_OK;
    if (rc) return rc;
  }
  return fan_in(e);
}
// order[b0, b1) is sorted by class: one launch per run of equal class, on that class's stream (forked here, joined by the
// caller).  launch(c, begin, end, grid, stream) takes the run [begin, end) of `order`.
template <class Launch> static int launch_class_runs(ckm_engine *e, const std::vector<int32_t> &order, const std::vector<int8_t> &cls, size_t b0, size_t b1, Launch launch) {
  const int nsm = e->prop.multiProcessorCount;
  int rc;
  if ((rc = fan_out(e))) return rc;
  while (b0 < b1) {
    size_t r1 = b0; const int c = cls[order[b0]];
    while (r1 < b1 && cls[order[r1]] == c) ++r1;
    const int cnt = (int)(r1 - b0);
    const int grid = c < N_BLK_CLASSES ? std::min(nsm * 8, (cnt + 3) / 4) : std::min(nsm * 4, (cnt + FWD_WARPS - 1) / FWD_WARPS);
    if ((rc = launch(c, (int32_t)b0, (int32_t)r1, grid, e->cls[c]))) return rc;
    e->stats.kernel_launches++;
    b0 = r1;
  }
  return CKM_OK;
}

struct ActiveMasks { DevBuf tile_active, model_active, model_slot; bool all_active = true; };
static FilterParams filter_params(const ckm_models *m, const ckm_seqdb *db, ActiveMasks &am) {
  FilterParams p{};
  p.res = db->d_res; p.off = db->d_off; p.len = db->d_len; p.lenA = db->d_lenA; p.lenB = db->d_lenB; p.tmove_w = db->d_tmove_w;
  p.ms = m->d_scalars; p.bias_eo = m->d_bias_eo; p.rwv = m->d_rwv; p.twv = m->d_twv; p.rfv = m->d_rfv; p.tfv = m->d_tfv;
  p.twb = m->d_twb; p.rwb = m->d_rwb; p.tfb = m->d_tfb; p.rfb = m->d_rfb; p.twp = m->d_twp; p.rwp = m->d_rwp;
  p.row_elems = ((m->maxM + 31) / 32) * 32 + 64;
  p.F1 = 0.02; p.F2 = 1e-3; p.F3 = 1e-5;
  p.model_slot = am.model_slot.as<int32_t>(); p.nseq = db->nseq;
  return p;
}

static DomdefParams domdef_params(const ckm_models *m, const ckm_seqdb *db, const SearchKnobs &k) {
  DomdefParams p{};
  p.res = db->d_res; p.off = db->d_off; p.nullsc = db->d_nullsc; p.ms = m->d_scalars; p.rfv = m->d_rfv; p.tfv = m->d_tfv;
  p.row_elems = ((m->maxM + 31) / 32) * 32 + 64;
  p.tfb = m->d_tfb; p.rfb = m->d_rfb; p.use_blk = k.blk ? 1 : 0;
  return p;
}
// counters and stage times of the cascade; `stages` of its stages ran (2: SSV and MSV, 5: all)
static void fill_filter_stats(ckm_engine *e, int64_t n_pairs, const int32_t *ctr, unsigned long long cells, int stages) {
  ckm_stats &s = e->stats;
  s.n_pairs = n_pairs; s.n_cells = (int64_t)cells;
  s.n_ssv_cand = (int64_t)ctr[CTR_CAND] + ctr[CTR_SSVRES]; s.n_msv_exact = ctr[CTR_CAND]; s.n_past_msv = ctr[CTR_MSV]; s.n_past_bias = ctr[CTR_BIAS];
  s.n_past_vit = ctr[CTR_VIT]; s.n_past_fwd = ctr[CTR_FWD]; s.n_vit_redo = ctr[CTR_VREDO];
  float *ms[] = {&s.ms_ssv, &s.ms_msv, &s.ms_bias, &s.ms_vit, &s.ms_fwd};
  for (int i = 0; i < stages; ++i) ev_elapsed(e, ms[i], EV_SSV + i, EV_SSV + i + 1);
}
static std::vector<float> &logsum_table() {
  static std::vector<float> t = [] {
    std::vector<float> v(16000);
    for (int i = 0; i < 16000; ++i) v[i] = (float)std::log(1.0 + std::exp((double)-i / 1000.0));
    return v;
  }();
  return t;
}

// Builds the per-bin activity masks for a query subset.  bin_model_offsets == nullptr: the same nmodels queries for all bins.
static int build_masks(const ckm_models *m, const ckm_seqdb *db, const int32_t *model_idx, int32_t nmodels,
                       const int64_t *bin_model_offsets, ActiveMasks &am, std::vector<int32_t> &slot_of_model, cudaStream_t st) {
  const int ndb = (int)m->models.size(), nbins = db->nbins, ntiles = (int)m->tiles.size();
  slot_of_model.assign(ndb, -1);
  bool all = (bin_model_offsets == nullptr) && (model_idx == nullptr || nmodels == ndb);
  if (model_idx == nullptr) { for (int i = 0; i < ndb; ++i) slot_of_model[i] = i; }
  else if (bin_model_offsets == nullptr) {
    for (int i = 0; i < nmodels; ++i) {
      if (model_idx[i] < 0 || model_idx[i] >= ndb) { set_error("model index out of range"); return CKM_EINVAL; }
      if (slot_of_model[model_idx[i]] >= 0) { set_error("duplicate model index in query list"); return CKM_EINVAL; }
      slot_of_model[model_idx[i]] = i;
    }
    if (all) for (int i = 0; i < ndb; ++i) if (slot_of_model[i] < 0) all = false;
  }
  am.all_active = all;
  CKM_TRY(am.model_slot.put(slot_of_model.data(), (size_t)ndb, st));
  if (all) return CKM_OK;
  std::vector<uint8_t> ma((size_t)nbins * ndb, 0), ta((size_t)nbins * ntiles, 0);
  for (int b = 0; b < nbins; ++b) {
    if (bin_model_offsets == nullptr) {
      for (int i = 0; i < nmodels; ++i) ma[(size_t)b * ndb + model_idx[i]] = 1;
    } else {
      for (int64_t i = bin_model_offsets[b]; i < bin_model_offsets[b + 1]; ++i) {
        if (model_idx[i] < 0 || model_idx[i] >= ndb) { set_error("model index out of range"); return CKM_EINVAL; }
        // a model listed twice would be searched once but counted twice in the bin's pairs: refused, as in a shared list
        if (ma[(size_t)b * ndb + model_idx[i]]) { set_error("duplicate model index in the query list of bin " + std::to_string(b)); return CKM_EINVAL; }
        ma[(size_t)b * ndb + model_idx[i]] = 1;
      }
    }
    for (int t = 0; t < ntiles; ++t) {
      const TileDesc &td = m->tiles[t];
      uint8_t any = 0;
      for (int j = 0; j < td.nmodels; ++j) any |= ma[(size_t)b * ndb + m->tile_models[td.first_model + j].model];
      ta[(size_t)b * ntiles + t] = any;
    }
    // a chained model is addressed through its first tile
  }
  CKM_TRY(am.model_active.put(ma.data(), ma.size(), st));
  CKM_TRY(am.tile_active.put(ta.data(), ta.size(), st));
  return stream_sync(st);     // host vectors go out of scope
}
// Stage 1: SSV pre-filter over all pairs -> candidate list; exact MSV on the candidates -> pass list.
struct Stage1 {
  DevBuf cand, pass, bnd, glist, cells;
  int32_t cand_cap = 0, pass_cap = 0;
};
// Queue capacities: a fraction of the pairs (SSV forwards ~3%, exact MSV keeps ~2%; 1/6 and 1/12 leave a wide margin), all in
// 64-bit arithmetic, never beyond QUEUE_MAX entries.  `attempt` > 0 is a retry after an overflow: the fractions grow 8-fold
// each time, so the third attempt holds every pair (or QUEUE_MAX of them).
constexpr int64_t QUEUE_MAX = (int64_t)1 << 30;
constexpr int QUEUE_ATTEMPTS = 3;
static int32_t queue_cap(int64_t n_pairs, int64_t divisor, int attempt) {
  int64_t want = n_pairs / divisor + 65536;
  for (int a = 0; a < attempt && want < n_pairs; ++a) want *= 8;
  return (int32_t)std::min<int64_t>(std::min<int64_t>(n_pairs, QUEUE_MAX), std::max<int64_t>((int64_t)1 << 16, want));
}

static int run_stage1(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const ckm_seqdb *db, ActiveMasks &am, int64_t n_pairs,
                      Stage1 &s1, int32_t *xj_dense, int attempt = 0) {
  cudaStream_t st = e->stream;
  int rc;
  s1.cand_cap = queue_cap(n_pairs, 6, attempt);
  const int64_t n_bypass = (int64_t)m->ssv_bypass.size() * db->nseq;          // models without SSV tiles: every pair is a candidate
  s1.cand_cap = (int32_t)std::min<int64_t>(QUEUE_MAX, (int64_t)s1.cand_cap + n_bypass);
  s1.pass_cap = queue_cap(n_pairs, 12, attempt);
  CKM_TRY(s1.cand.alloc(sizeof(int2) * (size_t)s1.cand_cap));
  CKM_TRY(s1.pass.alloc(sizeof(Candidate) * (size_t)s1.pass_cap));
  CKM_TRY(set_bytes(e->d_counters, 0, CTR_N * sizeof(int32_t), st));
  CKM_TRY(s1.cells.fill(sizeof(unsigned long long), 0, st));
  const int nsm = e->prop.multiProcessorCount;
  bool need_bnd = false;
  for (int nt : m->chain_ntiles) need_bnd |= (nt > 1);
  const int64_t bnd_stride = ((int64_t)db->maxL + 31) / 16 * 16;
  if (need_bnd) CKM_TRY(s1.bnd.alloc((size_t)nsm * SSV_WARPS_HOST * 2 * bnd_stride * sizeof(int16_t)));
  // group lists per J
  std::vector<int32_t> gl[4];
  for (size_t g = 0; g < m->groups.size(); ++g) gl[m->groups[g].J == 4 ? 0 : (m->groups[g].J == 8 ? 1 : (m->groups[g].J == 16 ? 2 : 3))].push_back((int32_t)g);
  std::vector<int32_t> flat;
  size_t goff[4];
  for (int c = 0; c < 4; ++c) { goff[c] = flat.size(); flat.insert(flat.end(), gl[c].begin(), gl[c].end()); }
  CKM_TRY(s1.glist.put(flat.data(), flat.size(), st));
  CKM_TRY(stream_sync(st));     // `flat` is read by the copy above

  CKM_TRY(ev_record(e, EV_SSV));
  SsvParams sp{};
  sp.res = db->d_res; sp.off = db->d_off; sp.len = db->d_len; sp.bin = db->d_bin;
  sp.msvB = db->d_msvB; sp.tjb = db->d_tjb; sp.order = db->d_order;
  sp.nseq = db->nseq; sp.seq_chunk = 128; sp.nchunks = (db->nseq + sp.seq_chunk - 1) / sp.seq_chunk;
  sp.groups = m->d_groups; sp.tiles = m->d_tiles; sp.tile_models = m->d_tile_models; sp.tile_blob = m->d_tile_blob;
  sp.chain_first_tile = m->d_chain_first_tile; sp.chain_ntiles = m->d_chain_ntiles;
  sp.tile_active = am.all_active ? nullptr : am.tile_active.as<uint8_t>();
  sp.model_active = am.all_active ? nullptr : am.model_active.as<uint8_t>();
  sp.ntiles = (int32_t)m->tiles.size(); sp.nmodels = (int32_t)m->models.size();
  sp.cand = s1.cand.as<int2>(); sp.cand_count = e->d_counters + CTR_CAND; sp.cand_cap = s1.cand_cap;
  sp.bnd = need_bnd ? s1.bnd.as<int16_t>() : nullptr; sp.bnd_stride = bnd_stride;
  sp.cells = s1.cells.as<unsigned long long>();
  sp.resolve = k.ssv_resolve ? 1 : 0;
  sp.ms = m->d_scalars; sp.nullsc = db->d_nullsc;
  sp.pass = s1.pass.as<Candidate>(); sp.pass_count = e->d_counters + CTR_MSV; sp.pass_cap = s1.pass_cap;
  sp.resolved_count = e->d_counters + CTR_SSVRES;
  sp.xj_dense = xj_dense; sp.model_slot = am.model_slot.as<int32_t>();
  sp.F1 = 0.02;
  const int Js[4] = {4, 8, 16, 32};
  for (int c = 0; c < 4; ++c) {
    if (gl[c].empty() || db->nseq == 0) continue;
    sp.group_list = s1.glist.as<int32_t>() + goff[c]; sp.ngroups = (int32_t)gl[c].size();
    sp.unit_counter = e->d_counters + CTR_UNIT4 + c;
    int64_t maxbytes = 0;
    for (int g : gl[c]) maxbytes = std::max<int64_t>(maxbytes, m->groups[g].table_bytes);
    const int64_t units = (int64_t)sp.ngroups * sp.nchunks;
    const int grid = (int)std::min<int64_t>(nsm, units);
    if ((rc = launch_ssv(Js[c], sp, grid, (size_t)maxbytes, st))) return rc;
    e->stats.kernel_launches++;
  }
  if (!m->ssv_bypass.empty()) {
    if ((rc = launch_ssv_bypass(m->d_ssv_bypass, (int32_t)m->ssv_bypass.size(), db->nseq, db->d_len, db->d_bin,
                                am.all_active ? nullptr : am.model_active.as<uint8_t>(), (int32_t)m->models.size(),
                                s1.cand.as<int2>(), e->d_counters + CTR_CAND, s1.cand_cap, st))) return rc;
    e->stats.kernel_launches++;
  }
  CKM_TRY(ev_record(e, EV_MSV));
  // exact MSV on the candidates
  MsvParams p{};
  p.res = db->d_res; p.off = db->d_off; p.len = db->d_len; p.nullsc = db->d_nullsc; p.tjb = db->d_tjb;
  p.ms = m->d_scalars; p.rbv = m->d_rbv; p.rmb = m->d_rmb;
  p.cand = s1.cand.as<int2>(); p.cand_count = e->d_counters + CTR_CAND; p.cand_cap = s1.cand_cap;
  p.out = s1.pass.as<Candidate>(); p.out_count = e->d_counters + CTR_MSV; p.out_cap = s1.pass_cap;
  p.xj_dense = xj_dense; p.model_slot = am.model_slot.as<int32_t>(); p.nseq = db->nseq;
  p.row_bytes = (m->maxM + 2 + 15) / 16 * 16;
  p.F1 = 0.02;
  p.use_blk = k.blk ? 1 : 0;
  if ((rc = per_class(e, p, launch_msv2, 16, launch_msv_exact, 4))) return rc;
  e->stats.kernel_launches += 1 + (p.use_blk ? N_BLK_CLASSES : 0);
  CKM_TRY(ev_record(e, EV_BIAS));
  return CKM_OK;
}

// ViterbiFilter from p.in to p.out.  packed: the int16x2 kernels, one per class, score first, from an index list grouped
// by (class, model) in `grp`; what they cannot score exactly (strong hits near the int16 ceiling, models without a class,
// pairs outside the safety conditions of kernels_vitp.cu) lands in the redo list, which the int32 kernels then take as their
// input.  No stage depends on the order of its input list: every kernel appends through atomics, and sorted_pairs orders the
// Forward survivors on the host.
static int run_viterbi(ckm_engine *e, const ckm_models *m, FilterParams &p, bool packed, DevBuf &grp) {
  int rc;
  if (packed) {
    const int nm = (int)m->models.size();
    const size_t nchunks = (size_t)p.in_cap / VITP_CHUNK + nm + 1;           // every model's last chunk may be partial
    const size_t words = 4 * (size_t)nm + 16 + ((size_t)p.in_cap + 1) / 2 * 2;
    CKM_TRY(grp.alloc(sizeof(int32_t) * words + sizeof(int2) * nchunks));
    int32_t *ws = grp.as<int32_t>();
    p.vit_cls_chunks = ws + 4 * (size_t)nm;
    p.vit_idx = p.vit_cls_chunks + 16;
    p.vit_chunks = reinterpret_cast<int2 *>(ws + words);
    p.vit_work = e->d_counters + CTR_VWORK;      // zeroed with the other counters at the start of the call
    if ((rc = launch_vit_group(p, nm, ws, e->prop.multiProcessorCount * 8, e->stream))) return rc;
    if ((rc = per_class<FilterParams>(e, p, launch_vitp, 8, nullptr, 0))) return rc;
    e->stats.kernel_launches += 3;
    p.in = p.redo; p.in_count = p.redo_count; p.in_cap = p.redo_cap;
  }
  // lane-blocked register kernels, one per class; models beyond the classes (all models without use_blk): shared-memory rows
  return per_class(e, p, launch_vit2, 8, launch_vit, 4);
}
// Stages 2-4 on the MSV survivors: bias filter -> ViterbiFilter -> ForwardParser.  Lists ping-pong between two buffers.
struct Stage2 {
  DevBuf a, b, redo, vgrp;      // the survivors of the Forward filter end in a; vgrp: the packed Viterbi work list
  int32_t cap = 0;
};
static int run_stage2(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const ckm_seqdb *db, ActiveMasks &am, Stage1 &s1, Stage2 &s2,
                      float *d_filtersc, float *d_vit, float *d_fwd, uint8_t *d_passed) {
  cudaStream_t st = e->stream;
  int rc;
  s2.cap = s1.pass_cap;
  CKM_TRY(s2.a.alloc(sizeof(Candidate) * (size_t)s2.cap));
  CKM_TRY(s2.b.alloc(sizeof(Candidate) * (size_t)s2.cap));
  CKM_TRY(s2.redo.alloc(sizeof(Candidate) * (size_t)s2.cap));
  const int nsm = e->prop.multiProcessorCount;
  FilterParams p = filter_params(m, db, am);
  p.redo = s2.redo.as<Candidate>(); p.redo_count = e->d_counters + CTR_VREDO; p.redo_cap = s2.cap;
  p.use_blk = k.blk ? 1 : 0;
  p.dense_filtersc = d_filtersc; p.dense_vit = d_vit; p.dense_fwd = d_fwd; p.dense_passed = d_passed;
  // bias: pass list (stage 1) -> a
  p.in = s1.pass.as<Candidate>(); p.in_count = e->d_counters + CTR_MSV; p.in_cap = s1.pass_cap;
  p.out = s2.a.as<Candidate>(); p.out_count = e->d_counters + CTR_BIAS; p.out_cap = s2.cap;
  if ((rc = launch_bias(p, nsm * 8, st))) return rc;
  CKM_TRY(ev_record(e, EV_VIT));
  // viterbi: a -> b
  p.in = s2.a.as<Candidate>(); p.in_count = e->d_counters + CTR_BIAS; p.in_cap = s2.cap;
  p.out = s2.b.as<Candidate>(); p.out_count = e->d_counters + CTR_VIT; p.out_cap = s2.cap;
  if ((rc = run_viterbi(e, m, p, k.vitp, s2.vgrp))) return rc;
  CKM_TRY(ev_record(e, EV_FWD));
  // forward: b -> a
  p.in = s2.b.as<Candidate>(); p.in_count = e->d_counters + CTR_VIT; p.in_cap = s2.cap;
  p.out = s2.a.as<Candidate>(); p.out_count = e->d_counters + CTR_FWD; p.out_cap = s2.cap;
  // widest classes first: their one-warp-per-pair kernels are the long pole of the stage, the narrow ones fill in around them
  if ((rc = per_class(e, p, launch_fwd2, 8, launch_fwd, 4, /*widest_first=*/true))) return rc;
  CKM_TRY(ev_record(e, EV_CASCADE_END));
  e->stats.kernel_launches += 3 + (k.vitp ? N_BLK_CLASSES : 0) + (p.use_blk ? 2 * N_BLK_CLASSES : 0);
  return CKM_OK;
}

// floats of scratch one envelope needs (blocked kernels: one matrix, the OA fill overwrites F.B row by row; chunked kernels: two)
static int64_t envelope_need(const ckm_models *m, const PairWork &pw, const Envelope &en, bool use_blk) {
  const int64_t Ld = en.j - en.i + 1, Mpad = ((m->models[pw.model].M + 1) + 31) / 32 * 32 + 32;
  const int64_t vq = use_blk ? vq_of(m->models[pw.model].M) : 0;
  const int64_t width = vq ? 32 * vq : Mpad;
  return (vq ? 1 : 2) * (Ld + 1) * 3 * width + (Ld + 1) * 15 + 64;
}
// Envelope rescoring in waves: each envelope's matrix and specials in `scratch`, under `budget` floats per wave (never less
// than one envelope), every class on its own stream.  leave_last: the last wave is left running on the class streams (the
// caller joins them with fan_in).
static int run_envelope_waves(ckm_engine *e, const ckm_models *m, const std::vector<PairWork> &pairs, DomdefParams &p, int64_t budget,
                              DevBuf &scratch, std::vector<Envelope> &ev, DevBuf &d_ev, DevBuf &d_ord, bool leave_last) {
  if (ev.empty()) return CKM_OK;
  cudaStream_t st = e->stream;
  int rc;
  std::vector<int64_t> need(ev.size());
  std::vector<int8_t> ecls(ev.size());
  for (size_t i = 0; i < ev.size(); ++i) {
    const PairWork &pw = pairs[ev[i].pair];
    need[i] = envelope_need(m, pw, ev[i], p.use_blk != 0);
    ecls[i] = (int8_t)cls_of(m->models[pw.model].M, p.use_blk != 0);
  }
  budget = std::max<int64_t>(budget, *std::max_element(need.begin(), need.end()));
  CKM_TRY(d_ev.alloc(sizeof(Envelope) * ev.size()));
  CKM_TRY(d_ord.alloc(sizeof(int32_t) * ev.size()));
  std::vector<int32_t> eorder(ev.size());
  for (size_t w0 = 0, w1; w0 < ev.size(); w0 = w1) {
    int64_t tot = 0;
    for (w1 = w0; w1 < ev.size() && (w1 == w0 || tot + need[w1] <= budget); ++w1) { ev[w1].scratch_off = tot; tot += need[w1]; }
    if (sizeof(float) * (size_t)tot > scratch.bytes && (rc = scratch.alloc(sizeof(float) * (size_t)tot))) return rc;
    // this wave's envelopes grouped by class, largest first; one stream per class
    for (size_t i = w0; i < w1; ++i) eorder[i] = (int32_t)i;
    std::stable_sort(eorder.begin() + w0, eorder.begin() + w1, [&](int32_t a, int32_t b) { return ecls[a] != ecls[b] ? ecls[a] > ecls[b] : need[a] > need[b]; });
    CKM_TRY(copy_in(d_ev.as<Envelope>() + w0, ev.data() + w0, w1 - w0, st));
    CKM_TRY(copy_in(d_ord.as<int32_t>() + w0, eorder.data() + w0, w1 - w0, st));
    p.envs = d_ev.as<Envelope>(); p.env_order = d_ord.as<int32_t>(); p.scratch = scratch.as<float>();
    if ((rc = launch_class_runs(e, eorder, ecls, w0, w1, [&](int c, int32_t b0, int32_t b1, int grid, cudaStream_t s) -> int {
          p.env_begin = b0; p.env_end = b1; return c < N_BLK_CLASSES ? launch_envelopes2(p, c, grid, s) : launch_envelopes(p, grid, s); }))) return rc;
    CKM_TRY(stream_sync(st));          // the two copies above have read the host vectors
    if (w1 < ev.size() || !leave_last) { CKM_TRY(fan_in(e)); CKM_TRY(stream_sync(st)); }
  }
  return CKM_OK;
}

// The queries of one search: activity masks, each model's position in each bin's query list (the order of the bin's rows;
// one shared list: qorder[0]) and the number of pairs.
struct QueryPlan { ActiveMasks am; bool per_bin = false; std::vector<std::vector<int32_t>> qorder; int64_t n_pairs = 0; };
static int plan_queries(const ckm_models *m, const ckm_seqdb *db, const int32_t *model_idx, int32_t nmodels, const int64_t *bin_model_offsets, QueryPlan &q, cudaStream_t st) {
  const int ndb = (int)m->models.size();
  if (model_idx == nullptr && bin_model_offsets == nullptr) nmodels = ndb;
  std::vector<int32_t> slot;
  int rc = build_masks(m, db, model_idx, nmodels, bin_model_offsets, q.am, slot, st);
  if (rc) return rc;
  q.per_bin = bin_model_offsets != nullptr;
  if (q.per_bin) {
    q.qorder.assign(db->nbins, std::vector<int32_t>(ndb, -1));
    for (int b = 0; b < db->nbins; ++b) {
      for (int64_t i = bin_model_offsets[b]; i < bin_model_offsets[b + 1]; ++i) q.qorder[b][model_idx[i]] = (int32_t)(i - bin_model_offsets[b]);
      q.n_pairs += (int64_t)db->bin_nseq[b] * (bin_model_offsets[b + 1] - bin_model_offsets[b]);
    }
  } else {
    q.qorder.emplace_back(std::move(slot));     // moved, not copied: with every model active, build_masks' upload of it is still in flight
    q.n_pairs = (int64_t)db->nseq * nmodels;
  }
  return CKM_OK;
}

// The filter cascade over all pairs.  A candidate-dense input (many pairs past SSV) overflows the default queues: the cascade
// is re-run with larger ones.
static int run_cascade(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const ckm_seqdb *db, ActiveMasks &am, int64_t n_pairs, Stage1 &s1, Stage2 &s2, int32_t *ctr) {
  cudaStream_t st = e->stream;
  unsigned long long cells = 0;
  int rc;
  for (int attempt = 0; attempt < QUEUE_ATTEMPTS; ++attempt) {
    if (attempt > 0) e->stats.n_queue_retries++;
    if ((rc = run_stage1(e, k, m, db, am, std::max<int64_t>(n_pairs, 1), s1, nullptr, attempt))) return rc;
    if ((rc = run_stage2(e, k, m, db, am, s1, s2, nullptr, nullptr, nullptr, nullptr))) return rc;
    CKM_TRY(copy_out(ctr, e->d_counters, CTR_N, st));
    CKM_TRY(s1.cells.get(&cells, 1, st));
    CKM_TRY(stream_sync(st));
    const bool over = ctr[CTR_CAND] > s1.cand_cap || ctr[CTR_MSV] > s1.pass_cap || ctr[CTR_BIAS] > s2.cap || ctr[CTR_VIT] > s2.cap || ctr[CTR_FWD] > s2.cap ||
                      ctr[CTR_VREDO] > s2.cap;
    if (!over) { fill_filter_stats(e, n_pairs, ctr, cells, 5); return CKM_OK; }
    if (s1.cand_cap >= std::min<int64_t>(n_pairs, QUEUE_MAX) && s1.pass_cap >= std::min<int64_t>(n_pairs, QUEUE_MAX)) break;
  }
  set_error("candidate queue overflow in the filter cascade: more than 2^30 candidate pairs in one batch; search fewer bins per call");
  return CKM_ECAPACITY;
}

// The Forward survivors sorted by (sequence, model), each with the offset of its per-residue rows; rows: their total.
static int sorted_pairs(const ckm_seqdb *db, const Candidate *d_fwd_list, int npairs, std::vector<PairWork> &pairs, int64_t &rows) {
  std::vector<Candidate> fl((size_t)npairs);
  if (npairs) CKM_CUDA(cudaMemcpy(fl.data(), d_fwd_list, sizeof(Candidate) * fl.size(), cudaMemcpyDeviceToHost));
  std::sort(fl.begin(), fl.end(), [](const Candidate &a, const Candidate &b) { return a.seq != b.seq ? a.seq < b.seq : a.model < b.model; });
  pairs.assign((size_t)npairs, PairWork{});
  rows = 0;
  for (int i = 0; i < npairs; ++i) {
    PairWork &pw = pairs[i];
    pw.seq = fl[i].seq; pw.model = fl[i].model; pw.L = db->len[pw.seq];
    pw.first_dom = 0; pw.ndom_slots = 0; pw.fwdsc = fl[i].fwdsc; pw.filtersc = fl[i].filtersc; pw.usc = fl[i].usc;
    pw.row_off = rows; rows += pw.L + 1;
  }
  return CKM_OK;
}
// The domain stage of one search: its parameters, workspaces and host results.  The workspaces of the domain passes live as
// long as the stage, so a repeated pass reuses the cache slots of the first.
struct DomainStage {
  DomdefParams p{};
  DevBuf dpairs, dxf, dxb, dvec, dtbl, dregions, dporder, ddoms, dhits, dscratch, denvs, deorder, denvs2, deorder2;
  std::vector<Region> regs;          // sorted by (pair, start)
  std::vector<DomainOut> doms; std::vector<HitOut> hout;
};
// Forward/Backward of every pair and its regions (the pairs' candidate domains), sorted.
static int run_regions(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const ckm_seqdb *db, const std::vector<PairWork> &pairs, int64_t rows, DomainStage &D, Trace &tr) {
  cudaStream_t st = e->stream;
  const int npairs = (int)pairs.size();
  const size_t rws = (size_t)rows;
  CKM_TRY(D.dpairs.put(pairs.data(), pairs.size(), st));
  CKM_TRY(D.dxf.alloc(sizeof(float) * rws * X_NX_HOST));
  CKM_TRY(D.dxb.alloc(sizeof(float) * rws * X_NX_HOST));
  CKM_TRY(D.dvec.alloc(sizeof(float) * rws * 4));
  CKM_TRY(D.dtbl.put(logsum_table().data(), 16000, st));
  const int region_cap = npairs * 8 + 1024;
  CKM_TRY(D.dregions.alloc(sizeof(Region) * (size_t)region_cap));
  CKM_TRY(set_bytes(e->d_counters + CTR_ENV, 0, sizeof(int32_t), st));
  DomdefParams &p = D.p = domdef_params(m, db, k);
  p.pairs = D.dpairs.as<PairWork>(); p.npairs = npairs;
  p.xf = D.dxf.as<float>(); p.xb = D.dxb.as<float>();
  p.btot = D.dvec.as<float>(); p.etot = p.btot + rws; p.mocc = p.etot + rws; p.n2sc = p.mocc + rws;
  p.regions = D.dregions.as<Region>(); p.region_count = e->d_counters + CTR_ENV; p.region_cap = region_cap;
  p.logsum_tbl = D.dtbl.as<float>();
  // pairs grouped by class (widest class first: it is the long pole), longest target first inside a class; every class runs on its own stream
  std::vector<int32_t> order((size_t)npairs);
  std::vector<int8_t> pcls((size_t)npairs);
  for (int i = 0; i < npairs; ++i) { order[i] = i; pcls[i] = (int8_t)cls_of(m->models[pairs[i].model].M, p.use_blk != 0); }
  std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return pcls[a] != pcls[b] ? pcls[a] > pcls[b] : pairs[a].L > pairs[b].L; });
  CKM_TRY(D.dporder.put(order.data(), order.size(), st));
  p.pair_order = D.dporder.as<int32_t>();
  CKM_TRY(launch_class_runs(e, order, pcls, 0, (size_t)npairs, [&](int c, int32_t b0, int32_t b1, int grid, cudaStream_t s) -> int {
        p.pair_begin = b0; p.pair_end = b1; return c < N_BLK_CLASSES ? launch_regions2(p, c, grid, s) : launch_regions(p, grid, s); }));
  CKM_TRY(fan_in(e));
  int32_t nreg = 0;
  CKM_TRY(copy_out(&nreg, e->d_counters + CTR_ENV, 1, st));
  CKM_TRY(stream_sync(st));     // also the end of the copy that reads `order`
  tr.mark("regions kernels");
  if (nreg > region_cap) { set_error("region queue overflow"); return CKM_ECAPACITY; }
  D.regs.resize((size_t)nreg);
  if (nreg) CKM_CUDA(cudaMemcpy(D.regs.data(), D.dregions.p, sizeof(Region) * D.regs.size(), cudaMemcpyDeviceToHost));
  std::sort(D.regs.begin(), D.regs.end(), [](const Region &a, const Region &b) { return a.pair != b.pair ? a.pair < b.pair : a.i < b.i; });
  tr.mark("regions sorted");
  return CKM_OK;
}

// owner of the trace-ensemble job in flight: unless ensembles_collect takes it (release), it is abandoned (its stream drained)
struct AbandonJob { cudaStream_t st; void operator()(EnsembleJob *job) const { ensembles_abandon(job, st); } };
// One pass of the domain phase.  Domain slots: regions are sorted by (pair, start), so a pair's slots are contiguous and in
// sequence order: one slot per single-domain region, caps[].envelopes (ENS_MAXENV at first) per multi-domain region (the
// ensemble decides how many it fills; unused slots keep ok = 0 and are skipped by every consumer).  Fixing the slots before
// the ensemble has run lets the envelopes of the single-domain regions be rescored WHILE the trace ensemble of the
// multi-domain ones is still sampling.  A region that turns out to hold more domains than its slots (or more sampled segments
// than its clustering buffers) reports what it needs: caps takes it, *grown is set and the pass has to be repeated.
static int domain_pass(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, std::vector<PairWork> &pairs, DomainStage &D,
                       const std::vector<int> &multi_idx, std::vector<EnsembleCaps> &caps, Trace &tr, bool *grown) {
  cudaStream_t st = e->stream;
  DomdefParams &p = D.p;
  const std::vector<Region> &regs = D.regs; const int nreg = (int)regs.size();
  int rc;
  *grown = false;
  std::vector<int32_t> reg_slot((size_t)nreg);
  std::vector<Envelope> envs1, envs2;
  int32_t nslots = 0;
  for (auto &pw : pairs) { pw.ndom_slots = 0; pw.first_dom = 0; }
  for (int r = 0, mi = 0; r < nreg; ++r) {
    PairWork &pw = pairs[regs[r].pair];
    if (pw.ndom_slots == 0) pw.first_dom = nslots;
    reg_slot[r] = nslots;
    if (!regs[r].multi) { Envelope en{}; en.pair = regs[r].pair; en.i = regs[r].i; en.j = regs[r].j; en.slot = nslots; envs1.push_back(en); }
    const int n = regs[r].multi ? caps[mi++].envelopes : 1;
    nslots += n; pw.ndom_slots += n;
  }
  D.doms.assign((size_t)nslots, DomainOut{});
  if (nslots == 0) return CKM_OK;
  CKM_TRY(D.ddoms.fill(sizeof(DomainOut) * (size_t)nslots, 0, st));
  CKM_TRY(D.dhits.alloc(sizeof(HitOut) * pairs.size()));
  CKM_TRY(copy_in(D.dpairs.as<PairWork>(), pairs.data(), pairs.size(), st));
  p.doms = D.ddoms.as<DomainOut>();
  // The trace ensemble of the multi-domain regions (one warp per region, latency-bound, its own stream) runs next to the
  // envelope kernels of the single-domain regions (class streams).  Next to them its dependent loads take 2-3x longer than
  // alone.  When the envelopes need more than one wave of scratch (large batches) it is queued FIRST and has all the waves to
  // hide under (32-bin batch: domain stage 501 -> 485 ms); with a single wave it is queued after the envelope kernels and takes
  // the SMs as they drain.  CKM_ENS_FIRST=1 / 0 forces one order.
  const bool multi = !multi_idx.empty();
  bool ens_first = (k.ens_first == 1);
  if (k.ens_first < 0 && multi) {
    int64_t tot = 0;
    for (const Envelope &en : envs1) tot += envelope_need(m, pairs[en.pair], en, p.use_blk != 0);
    ens_first = tot > k.env_budget;
  }
  std::unique_ptr<EnsembleJob, AbandonJob> ens(nullptr, AbandonJob{e->aux});
  auto launch_ensemble = [&]() -> int {
    CKM_CUDA(cudaEventRecord(e->fan_ev, st));
    CKM_CUDA(cudaStreamWaitEvent(e->aux, e->fan_ev, 0));
    EnsembleJob *job = nullptr;
    const int r = ensembles_launch(e, m, p, pairs, regs, multi_idx, caps, e->aux, &job);
    ens.reset(job);       // a job that failed to launch is abandoned too
    return r;
  };
  if (multi && ens_first && (rc = launch_ensemble())) return rc;
  if ((rc = run_envelope_waves(e, m, pairs, p, k.env_budget, D.dscratch, envs1, D.denvs, D.deorder, multi))) return rc;
  tr.mark("envelope batch 1 launched");
  if (multi) {
    if (!ens_first && (rc = launch_ensemble())) return rc;
    if (!envs1.empty()) { CKM_TRY(fan_in(e)); CKM_TRY(stream_sync(st)); }
    std::vector<std::vector<Envelope>> multi_envs; std::vector<EnsembleCaps> grow;
    int n_over = 0;
    if ((rc = ensembles_collect(ens.release(), e->aux, multi_envs, grow, &n_over))) return rc;
    tr.mark("batch 1 + ensemble done");
    if (n_over > 0) {
      for (size_t mi = 0; mi < caps.size(); ++mi) if (grow[mi].segments) caps[mi] = grow[mi];
      *grown = true;
      return CKM_OK;
    }
    for (size_t mi = 0; mi < multi_idx.size(); ++mi) {
      int c = 0;
      for (Envelope en : multi_envs[mi]) { en.slot = reg_slot[multi_idx[mi]] + c++; envs2.push_back(en); }     // no more than the region's slots (ensembles_collect)
    }
    if ((rc = run_envelope_waves(e, m, pairs, p, k.env_budget, D.dscratch, envs2, D.denvs2, D.deorder2, false))) return rc;
    tr.mark("envelope batch 2 done");
  }
  p.hits = D.dhits.as<HitOut>();
  if ((rc = launch_scores(p, ((int)pairs.size() + 127) / 128, st))) return rc;
  e->stats.kernel_launches++;
  CKM_TRY(D.ddoms.get(D.doms.data(), D.doms.size(), st));
  CKM_TRY(D.dhits.get(D.hout.data(), D.hout.size(), st));
  return stream_sync(st);
}
// The domain phase: envelopes, domains and scores of every pair, repeated while a multi-domain region outgrows its capacities.
constexpr int DOMAIN_PASSES = 4;
static int run_domain_phase(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, std::vector<PairWork> &pairs, DomainStage &D, Trace &tr) {
  std::vector<int> multi_idx;
  for (int r = 0; r < (int)D.regs.size(); ++r) if (D.regs[r].multi) multi_idx.push_back(r);
  std::vector<EnsembleCaps> caps(multi_idx.size(), ENS_DEFAULT_CAPS);
  D.hout.assign(pairs.size(), HitOut{});
  for (int pass = 0; pass < DOMAIN_PASSES; ++pass) {
    if (pass > 0) e->stats.n_queue_retries++;
    bool grown = false;
    int rc = domain_pass(e, k, m, pairs, D, multi_idx, caps, tr, &grown);
    if (rc || !grown) return rc;
  }
  set_error("a multi-domain region keeps outgrowing the capacities it asked for");
  return CKM_ECAPACITY;
}

// Thresholds, ordering and rows: hmmsearch's output phase on the hit list.  Per bin and query, in query order, the targets
// by P-value; the domain E-values use the number of targets that pass the sequence threshold.
static std::vector<ckm_hit> assemble_rows(ckm_engine *e, const ckm_models *m, const ckm_seqdb *db, const QueryPlan &q, const std::vector<PairWork> &pairs,
                                          const std::vector<HitOut> &hout, const std::vector<DomainOut> &doms, double Ecut, double domEcut) {
  struct Key { int bin, q, pair; double lnP; int seq; };
  std::vector<Key> keys;
  for (int i = 0; i < (int)pairs.size(); ++i) {
    if (!hout[i].valid) continue;
    const int b = db->bin_of_seq[pairs[i].seq];
    keys.push_back(Key{b, (q.per_bin ? q.qorder[b] : q.qorder[0])[pairs[i].model], i, hout[i].lnP, pairs[i].seq});
  }
  std::sort(keys.begin(), keys.end(), [](const Key &a, const Key &b) {
    if (a.bin != b.bin) return a.bin < b.bin;
    if (a.q != b.q) return a.q < b.q;
    if (a.lnP != b.lnP) return a.lnP < b.lnP;
    return a.seq < b.seq;
  });
  std::vector<ckm_hit> rows_out;
  size_t g0 = 0;
  int64_t n_dom = 0;
  for (size_t i = 0; i < doms.size(); ++i) if (doms[i].ok) n_dom++;
  while (g0 < keys.size()) {
    size_t g1 = g0;
    while (g1 < keys.size() && keys[g1].bin == keys[g0].bin && keys[g1].q == keys[g0].q) ++g1;
    const double Z = (double)db->bin_nseq[keys[g0].bin];
    double domZ = 0.0;
    for (size_t k = g0; k < g1; ++k) if (std::exp(keys[k].lnP) * Z <= Ecut) domZ += 1.0;
    for (size_t k = g0; k < g1; ++k) {
      if (!(std::exp(keys[k].lnP) * Z <= Ecut)) continue;
      const PairWork &pw = pairs[keys[k].pair];
      const HitOut &h = hout[keys[k].pair];
      int nrep = 0;
      for (int d = pw.first_dom; d < pw.first_dom + pw.ndom_slots; ++d)
        if (doms[d].ok && std::exp(doms[d].lnP) * domZ <= domEcut) nrep++;
      int nd = 0;
      for (int d = pw.first_dom; d < pw.first_dom + pw.ndom_slots; ++d) {
        const DomainOut &dm = doms[d];
        if (!dm.ok || !(std::exp(dm.lnP) * domZ <= domEcut)) continue;
        ckm_hit r;
        std::memset(&r, 0, sizeof(r));
        r.bin = keys[k].bin; r.seq = pw.seq; r.model = pw.model; r.tlen = pw.L; r.qlen = m->models[pw.model].M;
        r.dom = ++nd; r.ndom = nrep;
        r.hmm_from = dm.hmmfrom; r.hmm_to = dm.hmmto; r.ali_from = dm.sqfrom; r.ali_to = dm.sqto; r.env_from = dm.ienv; r.env_to = dm.jenv;
        r.full_score = h.score; r.full_bias = h.pre_score - h.score;
        r.dom_score = dm.bitscore; r.dom_bias = (float)((double)dm.dombias * 1.44269504088896341);
        r.acc = (float)(dm.oasc / (1.0 + std::fabs((float)(dm.jenv - dm.ienv))));
        r.full_evalue = std::exp(h.lnP) * Z; r.c_evalue = std::exp(dm.lnP) * domZ; r.i_evalue = std::exp(dm.lnP) * Z;
        r.full_lnP = h.lnP; r.dom_lnP = dm.lnP;
        rows_out.push_back(r);
      }
    }
    g0 = g1;
  }
  e->stats.n_hits_seq = (int64_t)keys.size(); e->stats.n_domains = n_dom; e->stats.n_reported = (int64_t)rows_out.size();
  return rows_out;
}

static int do_search(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const int32_t *model_idx, int32_t nmodels,
                     const int64_t *bin_model_offsets, const ckm_seqdb *db, double Ecut, double domEcut, ckm_hit **hits_out, int64_t *nhits_out) {
  *hits_out = nullptr; *nhits_out = 0;
  const DeviceScope ws(e);
  QueryPlan q;
  int rc = plan_queries(m, db, model_idx, nmodels, bin_model_offsets, q, ws.st);
  if (rc) return rc;
  std::memset(&e->stats, 0, sizeof(e->stats));
  if (q.n_pairs > ((int64_t)1 << 40)) { set_error("ckm_search: more than 2^40 (ORF x HMM) pairs in one call; search fewer bins per call"); return CKM_ECAPACITY; }
  CKM_TRY(ev_record(e, EV_CALL));
  Trace tr(k.trace);
  Stage1 s1; Stage2 s2; int32_t ctr[CTR_N];
  if ((rc = run_cascade(e, k, m, db, q.am, q.n_pairs, s1, s2, ctr))) return rc;
  tr.mark("filters done");
  std::vector<PairWork> pairs; int64_t rows = 0;
  if ((rc = sorted_pairs(db, s2.a.as<Candidate>(), ctr[CTR_FWD], pairs, rows))) return rc;
  CKM_TRY(ev_record(e, EV_DOMDEF));
  tr.mark("pair list sorted");
  DomainStage D;
  if (!pairs.empty()) {
    if ((rc = run_regions(e, k, m, db, pairs, rows, D, tr))) return rc;
    if ((rc = run_domain_phase(e, k, m, pairs, D, tr))) return rc;
  }
  CKM_TRY(ev_record(e, EV_END));
  CKM_CUDA(cudaEventSynchronize(e->ev[EV_END]));
  tr.mark("scores + downloads");
  const std::vector<ckm_hit> rows_out = assemble_rows(e, m, db, q, pairs, D.hout, D.doms, Ecut, domEcut);
  tr.mark("rows assembled");
  ev_elapsed(e, &e->stats.ms_domdef, EV_DOMDEF, EV_END);
  ev_elapsed(e, &e->stats.ms_total, EV_CALL, EV_END);
  if (!rows_out.empty()) {
    ckm_hit *out = (ckm_hit *)std::malloc(sizeof(ckm_hit) * rows_out.size());
    if (!out) { set_error("out of host memory"); return CKM_ENOMEM; }
    std::memcpy(out, rows_out.data(), sizeof(ckm_hit) * rows_out.size());
    *hits_out = out;
  }
  *nhits_out = (int64_t)rows_out.size();
  return CKM_OK;
}

// hmmalign: every sequence against one model, as one full-length envelope in unihit local mode (what `hmmalign` configures:
// Forward, Backward, posterior decoding, optimal-accuracy fill and traceback); the traceback's state per residue is the output.
// A sequence that carries a second strong copy of the domain cannot be scored as ONE unihit envelope in scaled fp32 (the
// Backward pass overflows where the Forward pass has underflowed); such a sequence is aligned over the envelope of its
// best-scoring domain as the search pipeline defines it, the rest of it being flank.
static int align_pass(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const ckm_seqdb *db, std::vector<PairWork> &pairs,
                      std::vector<Envelope> &envs, int64_t rows, std::vector<int32_t> &trace, std::vector<DomainOut> &doms) {
  const DeviceScope ws(e);
  DevBuf dpairs, dn2, dtrace, ddoms, dscratch, denvs, deorder;
  const size_t rws = (size_t)rows;
  CKM_TRY(dpairs.put(pairs.data(), pairs.size(), ws.st));
  CKM_TRY(dn2.fill(sizeof(float) * rws, 0, ws.st));
  CKM_TRY(dtrace.fill(sizeof(int32_t) * rws, 0, ws.st));
  CKM_TRY(ddoms.fill(sizeof(DomainOut) * pairs.size(), 0, ws.st));
  DomdefParams p = domdef_params(m, db, k);
  p.pairs = dpairs.as<PairWork>(); p.npairs = (int32_t)pairs.size();
  p.n2sc = dn2.as<float>(); p.trace = dtrace.as<int32_t>();
  p.doms = ddoms.as<DomainOut>();
  CKM_TRY(run_envelope_waves(e, m, pairs, p, k.env_budget, dscratch, envs, denvs, deorder, false));
  trace.resize(rws);
  doms.resize(pairs.size());
  CKM_TRY(dtrace.get(trace.data(), rws, ws.st));
  CKM_TRY(ddoms.get(doms.data(), doms.size(), ws.st));
  return stream_sync(ws.st);
}

// The group driver behind ckm_align and ckm_align_groups: the sequences of group g against model group_model[g], every group
// in one align_pass (the envelope kernels take pairs of mixed models, as the search feeds them).  The groups' ranges of
// sequences are disjoint (checked by the caller), so a sequence has one model.  The fallback searches the models of the
// groups that have failed sequences in one call over `db`; a pair's domains do not depend on the other pairs of a search.
static int do_align_groups(ckm_engine *e, const SearchKnobs &k, const ckm_models *m, const int32_t *group_model, const int64_t *group_seq_off,
                           int32_t ngroups, const ckm_seqdb *db, int32_t *state_out, float *oasc_out) {
  std::memset(&e->stats, 0, sizeof(e->stats));
  const int nseq = db->nseq;
  for (int64_t i = 0; i < db->nres; ++i) state_out[i] = 0;
  if (oasc_out) for (int s = 0; s < nseq; ++s) oasc_out[s] = 0.0f;
  std::vector<PairWork> pairs;
  std::vector<Envelope> envs;
  int64_t rows = 0;
  auto add = [&](int s, int model, int i, int j) {
    PairWork pw{};
    pw.seq = s; pw.model = model; pw.L = db->len[s]; pw.first_dom = (int32_t)pairs.size(); pw.ndom_slots = 1; pw.row_off = rows;
    rows += pw.L + 1;
    Envelope en{};
    en.pair = (int32_t)pairs.size(); en.i = i; en.j = j; en.null2_done = 1; en.slot = (int32_t)pairs.size();
    pairs.push_back(pw); envs.push_back(en);
  };
  for (int g = 0; g < ngroups; ++g)
    for (int64_t s = group_seq_off[g]; s < group_seq_off[g + 1]; ++s) if (db->len[s] > 0) add((int)s, group_model[g], 1, db->len[s]);
  if (pairs.empty()) return CKM_OK;
  std::vector<int32_t> trace; std::vector<DomainOut> doms;
  int rc;
  if ((rc = align_pass(e, k, m, db, pairs, envs, rows, trace, doms))) return rc;
  auto emit = [&](const std::vector<PairWork> &pp, const std::vector<DomainOut> &dd, const std::vector<int32_t> &tr, std::vector<PairWork> *failed) {
    for (size_t pi = 0; pi < pp.size(); ++pi) {
      const PairWork &pw = pp[pi];
      if (!dd[pi].ok) { if (failed) failed->push_back(pw); continue; }
      if (oasc_out) oasc_out[pw.seq] = dd[pi].oasc;
      int32_t *dst = state_out + (db->offsets[pw.seq] - db->offsets[0]);
      for (int i = 1; i <= pw.L; ++i) dst[i - 1] = tr[pw.row_off + i];
    }
  };
  std::vector<PairWork> failed;
  emit(pairs, doms, trace, &failed);
  if (failed.empty()) return CKM_OK;
  // the rare sequences one unihit envelope cannot hold: the envelope of the best domain the search pipeline defines
  std::vector<int32_t> fmodels;
  for (const PairWork &pw : failed) fmodels.push_back(pw.model);
  std::sort(fmodels.begin(), fmodels.end());
  fmodels.erase(std::unique(fmodels.begin(), fmodels.end()), fmodels.end());
  ckm_hit *hits = nullptr; int64_t nhits = 0;
  if ((rc = do_search(e, k, m, fmodels.data(), (int32_t)fmodels.size(), nullptr, db, 1e300, 1e300, &hits, &nhits))) return rc;
  std::vector<int> model_of(nseq, -1), best(nseq, -1);
  for (const PairWork &pw : failed) model_of[pw.seq] = pw.model;
  for (int64_t h = 0; h < nhits; ++h) {
    const int s = hits[h].seq;
    if (hits[h].model != model_of[s]) continue;
    if (best[s] < 0 || hits[h].dom_score > hits[best[s]].dom_score) best[s] = (int)h;
  }
  pairs.clear(); envs.clear(); rows = 0;
  for (const PairWork &pw : failed) if (best[pw.seq] >= 0) add(pw.seq, pw.model, hits[best[pw.seq]].env_from, hits[best[pw.seq]].env_to);
  std::free(hits);
  if (pairs.empty()) return CKM_OK;
  if ((rc = align_pass(e, k, m, db, pairs, envs, rows, trace, doms))) return rc;
  emit(pairs, doms, trace, nullptr);
  return CKM_OK;
}

static int checked_align(ckm_engine *e, const ckm_models *m, const int32_t *group_model, const int64_t *group_seq_off, int32_t ngroups,
                         const ckm_seqdb *db, int32_t *state_out, float *oasc_out) {
  cudaSetDevice(e->device);
  return do_align_groups(e, read_knobs(true), m, group_model, group_seq_off, ngroups, db, state_out, oasc_out);
}

static int checked_search(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, int32_t nmodels, const int64_t *bin_model_offsets,
                          const ckm_seqdb *db, double E, double domE, ckm_hit **hits_out, int64_t *nhits_out) {
  if (!e || !m || !db || !hits_out || !nhits_out) { set_error("ckm_search: bad argument"); return CKM_EINVAL; }
  cudaSetDevice(e->device);
  return do_search(e, read_knobs(true), m, model_idx, nmodels, bin_model_offsets, db, E, domE, hits_out, nhits_out);
}

}  // namespace ckm

extern "C" {

int ckm_search(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, int32_t nmodels,
               const ckm_seqdb *db, double E, double domE, ckm_hit **hits_out, int64_t *nhits_out) {
  return checked_search(e, m, model_idx, nmodels, nullptr, db, E, domE, hits_out, nhits_out);
}
int ckm_search_per_bin(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, const int64_t *bin_model_offsets,
                       const ckm_seqdb *db, double E, double domE, ckm_hit **hits_out, int64_t *nhits_out) {
  if (!model_idx || !bin_model_offsets) { set_error("ckm_search_per_bin: bad argument"); return CKM_EINVAL; }
  return checked_search(e, m, model_idx, 0, bin_model_offsets, db, E, domE, hits_out, nhits_out);
}
int ckm_align(ckm_engine *e, const ckm_models *m, int32_t model, const ckm_seqdb *db, int32_t *state_out, float *oasc_out) {
  if (!e || !m || !db || !state_out) { set_error("ckm_align: bad argument"); return CKM_EINVAL; }
  if (model < 0 || model >= (int)m->models.size()) { set_error("ckm_align: model index out of range"); return CKM_EINVAL; }
  const int64_t all[2] = {0, db->nseq};
  return checked_align(e, m, &model, all, 1, db, state_out, oasc_out);
}
int ckm_align_groups(ckm_engine *e, const ckm_models *m, const int32_t *group_model, const int64_t *group_seq_off, int32_t ngroups,
                     const ckm_seqdb *db, int32_t *state_out, float *oasc_out) {
  if (!e || !m || !db || !state_out || ngroups < 0 || (ngroups > 0 && (!group_model || !group_seq_off))) {
    set_error("ckm_align_groups: bad argument"); return CKM_EINVAL;
  }
  for (int32_t g = 0; g < ngroups; ++g) {
    if (group_model[g] < 0 || group_model[g] >= (int)m->models.size()) { set_error("ckm_align_groups: model index out of range in group " + std::to_string(g)); return CKM_EINVAL; }
    if (group_seq_off[g] < 0 || group_seq_off[g + 1] < group_seq_off[g] || group_seq_off[g + 1] > db->nseq) {
      set_error("ckm_align_groups: group_seq_off must rise from >= 0 to <= nseq (group " + std::to_string(g) + ")"); return CKM_EINVAL;
    }
  }
  return checked_align(e, m, group_model, group_seq_off, ngroups, db, state_out, oasc_out);
}

// domtblout writer: the 22 columns + description CheckM's HMMERParser.readHitsDOM splits (checkm/hmmer.py:184-200)
int ckm_write_domtblout(const ckm_models *m, const ckm_hit *hits, int64_t nhits, int32_t bin, int32_t seq_base,
                        const char *const *names, const char *const *descs, const char *path) {
  if (!m || (!hits && nhits > 0) || !names || !path) { set_error("ckm_write_domtblout: bad argument"); return CKM_EINVAL; }
  FILE *fp = std::fopen(path, "w");
  if (!fp) { set_error(std::string("cannot write ") + path); return CKM_EIO; }
  int tnamew = 20, qnamew = 20, qaccw = 10, taccw = 10;
  for (int64_t i = 0; i < nhits; ++i) {
    if (hits[i].bin != bin) continue;
    const Model &md = m->models[hits[i].model];
    tnamew = std::max<int>(tnamew, (int)std::strlen(names[hits[i].seq - seq_base]));
    qnamew = std::max<int>(qnamew, (int)md.name.size());
    qaccw = std::max<int>(qaccw, (int)md.acc.size());
  }
  std::fprintf(fp, "#%*s %22s %40s %11s %11s %11s\n", tnamew + qnamew - 1 + 15 + taccw + qaccw, "", "--- full sequence ---",
               "-------------- this domain -------------", "hmm coord", "ali coord", "env coord");
  std::fprintf(fp, "#%-*s %-*s %5s %-*s %-*s %5s %9s %6s %5s %3s %3s %9s %9s %6s %5s %5s %5s %5s %5s %5s %5s %4s %s\n",
               tnamew - 1, " target name", taccw, "accession", "tlen", qnamew, "query name", qaccw, "accession", "qlen",
               "E-value", "score", "bias", "#", "of", "c-Evalue", "i-Evalue", "score", "bias", "from", "to", "from", "to", "from", "to", "acc", "description of target");
  std::fprintf(fp, "#%*s %*s ----- %*s %*s ----- --------- ------ ----- --- --- --------- --------- ------ ----- ----- ----- ----- ----- ----- ----- ---- ---------------------\n",
               tnamew - 1, "-------------------", taccw, "----------", qnamew, "--------------------", qaccw, "----------");
  for (int64_t i = 0; i < nhits; ++i) {
    const ckm_hit &h = hits[i];
    if (h.bin != bin) continue;
    const Model &md = m->models[h.model];
    const char *desc = (descs && descs[h.seq - seq_base] && descs[h.seq - seq_base][0]) ? descs[h.seq - seq_base] : "-";
    std::fprintf(fp, "%-*s %-*s %5d %-*s %-*s %5d %9.2g %6.1f %5.1f %3d %3d %9.2g %9.2g %6.1f %5.1f %5d %5d %5d %5d %5d %5d %4.2f %s\n",
                 tnamew, names[h.seq - seq_base], taccw, "-", h.tlen, qnamew, md.name.c_str(), qaccw, md.acc.empty() ? "-" : md.acc.c_str(), h.qlen,
                 h.full_evalue, h.full_score, h.full_bias, h.dom, h.ndom, h.c_evalue, h.i_evalue, h.dom_score, h.dom_bias,
                 h.hmm_from, h.hmm_to, h.ali_from, h.ali_to, h.env_from, h.env_to, h.acc, desc);
  }
  std::fprintf(fp, "#\n# Program:         checkm_b200 (libckm.so)\n# Pipeline mode:   SEARCH\n# [ok]\n");
  std::fclose(fp);
  return CKM_OK;
}

// test hooks: the cascade's per-pair scores as dense [query][sequence] arrays
int ckm_filter_scores(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, int32_t nmodels,
                      const ckm_seqdb *db, float *filtersc_out, float *vit_out, float *fwd_out, uint8_t *passed_out) {
  if (!e || !m || !db || !filtersc_out || !vit_out || !fwd_out || !passed_out) { set_error("ckm_filter_scores: bad argument"); return CKM_EINVAL; }
  const SearchKnobs k = read_knobs(false);
  const DeviceScope ws(e);
  QueryPlan q;
  int rc = plan_queries(m, db, model_idx, nmodels, nullptr, q, ws.st);
  if (rc) return rc;
  const int64_t n = q.n_pairs;
  DevBuf dfs, dvit, dfwd, dpass;
  const size_t nf = (size_t)n;
  // NaN-fill the float outputs, zero the flags
  for (DevBuf *b : {&dfs, &dvit, &dfwd}) CKM_TRY(b->fill(sizeof(float) * nf, 0xff, ws.st));
  CKM_TRY(dpass.fill(nf + 4, 0, ws.st));
  Stage1 s1; Stage2 s2;
  std::memset(&e->stats, 0, sizeof(e->stats));
  if ((rc = run_stage1(e, k, m, db, q.am, n, s1, nullptr))) return rc;
  if ((rc = run_stage2(e, k, m, db, q.am, s1, s2, dfs.as<float>(), dvit.as<float>(), dfwd.as<float>(), dpass.as<uint8_t>()))) return rc;
  int32_t ctr[CTR_N];
  CKM_TRY(copy_out(ctr, e->d_counters, CTR_N, ws.st));
  CKM_TRY(dfs.get(filtersc_out, nf, ws.st));
  CKM_TRY(dvit.get(vit_out, nf, ws.st));
  CKM_TRY(dfwd.get(fwd_out, nf, ws.st));
  CKM_TRY(dpass.get(passed_out, nf, ws.st));
  CKM_TRY(stream_sync(ws.st));
  if (ctr[CTR_CAND] > s1.cand_cap || ctr[CTR_MSV] > s1.pass_cap) { set_error("candidate queue overflow"); return CKM_ECAPACITY; }
  // MSV pass flags come from the stage-1 pass list
  std::vector<Candidate> pass1((size_t)ctr[CTR_MSV]);
  if (!pass1.empty()) CKM_CUDA(cudaMemcpy(pass1.data(), s1.pass.p, sizeof(Candidate) * pass1.size(), cudaMemcpyDeviceToHost));
  for (const Candidate &c : pass1) passed_out[(int64_t)q.qorder[0][c.model] * db->nseq + c.seq] |= 1;
  fill_filter_stats(e, n, ctr, /*cells: not counted by this hook*/ 0, 5);
  return CKM_OK;
}

int ckm_viterbi_scores(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, int32_t nmodels,
                       const ckm_seqdb *db, int32_t mode, float *vit_out) {
  if (!e || !m || !db || !vit_out) { set_error("ckm_viterbi_scores: bad argument"); return CKM_EINVAL; }
  const DeviceScope ws(e);
  const cudaStream_t st = ws.st;
  const int ndb = (int)m->models.size();
  if (model_idx == nullptr) nmodels = ndb;
  const int64_t n = (int64_t)nmodels * db->nseq;
  if (n > ((int64_t)1 << 30)) { set_error("ckm_viterbi_scores: too many pairs for one call"); return CKM_ECAPACITY; }
  ActiveMasks am; std::vector<int32_t> slot;
  int rc = build_masks(m, db, model_idx, nmodels, nullptr, am, slot, st);
  if (rc) return rc;
  std::vector<int32_t> slot_model((size_t)std::max(nmodels, 1));
  for (int i = 0; i < nmodels; ++i) slot_model[i] = model_idx ? model_idx[i] : i;
  const size_t nf = (size_t)n;
  DevBuf dsm, din, dout, dredo, dvit, dgrp;
  CKM_TRY(dsm.put(slot_model.data(), slot_model.size(), st));
  CKM_TRY(din.alloc(sizeof(Candidate) * nf));
  CKM_TRY(dout.alloc(sizeof(Candidate) * nf));
  CKM_TRY(dredo.alloc(sizeof(Candidate) * nf));
  CKM_TRY(set_bytes(e->d_counters, 0, CTR_N * sizeof(int32_t), st));
  CKM_TRY(dvit.fill(sizeof(float) * nf, 0xff, st));
  std::memset(&e->stats, 0, sizeof(e->stats));
  if (n > 0) {
    if ((rc = launch_all_pairs(din.as<Candidate>(), e->d_counters + CTR_BIAS, dsm.as<int32_t>(), nmodels, db->nseq, st))) return rc;
    FilterParams p = filter_params(m, db, am);
    p.use_blk = (mode == 2) ? 0 : 1;      // mode 2: every pair through the chunked shared-memory kernel
    p.dense_vit = dvit.as<float>();
    p.redo = dredo.as<Candidate>(); p.redo_count = e->d_counters + CTR_VREDO; p.redo_cap = (int32_t)nf;
    p.in = din.as<Candidate>(); p.in_count = e->d_counters + CTR_BIAS; p.in_cap = (int32_t)nf;
    p.out = dout.as<Candidate>(); p.out_count = e->d_counters + CTR_VIT; p.out_cap = (int32_t)nf;
    if ((rc = run_viterbi(e, m, p, mode == 0, dgrp))) return rc;
  }
  int32_t ctr[CTR_N];
  CKM_TRY(copy_out(ctr, e->d_counters, CTR_N, st));
  CKM_TRY(dvit.get(vit_out, nf, st));
  CKM_TRY(stream_sync(st));
  e->stats.n_pairs = n; e->stats.n_past_bias = ctr[CTR_BIAS]; e->stats.n_past_vit = ctr[CTR_VIT]; e->stats.n_vit_redo = ctr[CTR_VREDO];
  return CKM_OK;
}

int ckm_msv_scores(ckm_engine *e, const ckm_models *m, const int32_t *model_idx, int32_t nmodels,
                   const ckm_seqdb *db, int32_t *xj_out) {
  if (!e || !m || !db || !xj_out) { set_error("ckm_msv_scores: bad argument"); return CKM_EINVAL; }
  const SearchKnobs k = read_knobs(false);
  const DeviceScope ws(e);
  QueryPlan q;
  int rc = plan_queries(m, db, model_idx, nmodels, nullptr, q, ws.st);
  if (rc) return rc;
  const int64_t n = q.n_pairs;
  DevBuf dense;
  CKM_TRY(dense.fill(sizeof(int32_t) * (size_t)n, 0xff, ws.st));
  Stage1 s1;
  std::memset(&e->stats, 0, sizeof(e->stats));
  if ((rc = run_stage1(e, k, m, db, q.am, n, s1, dense.as<int32_t>()))) return rc;
  int32_t ctr[CTR_N];
  CKM_TRY(copy_out(ctr, e->d_counters, CTR_N, ws.st));
  unsigned long long cells = 0;
  CKM_TRY(s1.cells.get(&cells, 1, ws.st));
  CKM_TRY(dense.get(xj_out, (size_t)n, ws.st));
  CKM_TRY(stream_sync(ws.st));
  if (ctr[CTR_CAND] > s1.cand_cap || ctr[CTR_MSV] > s1.pass_cap) { set_error("candidate queue overflow"); return CKM_ECAPACITY; }
  fill_filter_stats(e, n, ctr, cells, 2);     // stage 1 only: the later counters are still zero
  return CKM_OK;
}

}  // extern "C"
