// Stand-alone driver of the C ABI (no Python, no torch) for compute-sanitizer runs of the kernels and of a fleet's lifetime:
//   g++ -O1 -std=c++17 -I/usr/local/cuda/include -o tools/sanitize/driver tools/sanitize/driver.cpp
//       -Lmodelmesh_b200/csrc -lmmplace -L/usr/local/cuda/lib64 -lcudart_static -ldl -lpthread -lrt -Wl,-rpath,'$ORIGIN/../../modelmesh_b200/csrc'
//   compute-sanitizer --tool memcheck|racecheck|synccheck [--leak-check full] tools/sanitize/driver [n_instances n_models n_decisions rounds]
// A small random fleet with type constraints, one commit, one traced batch (k_place, cooperative) and one untraced
// batch (k_place_lanes) whose results must agree; then every part of the fleet that holds CUDA resources of its own:
// a device-path commit, a batch under a call-wide exclude set, single decisions through the captured graph and the
// resident server (which must agree with the batch), stats, the reaper, the registry prune, and the closed loop (LRU
// init, churn init, two windows).  Each round destroys its fleet and prints how much device memory it did not give back
// (the first round also pays for the modules loaded on first use).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/mmplace.h"

static uint64_t rs = 88172645463325252ULL;
static uint32_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return (uint32_t)(rs >> 11); }

#define REQ(call, what)                                                              \
  do {                                                                               \
    if ((call) < 0) { fprintf(stderr, "%s: %s\n", what, mmp_last_error(f)); return 2; } \
  } while (0)

static int run(int NI, int NM, int ND) {
  mmp_config cfg = {2560, 600000, 2560, NI, NM, 0, 0, 1, 0, 0};
  mmp_fleet *f = nullptr;
  if (mmp_fleet_create(&cfg, &f) < 0) { fprintf(stderr, "create: %s\n", mmp_last_error(nullptr)); return 2; }
  mmp_types_set_json(f, "{\"ta\":{\"required\":[\"l1\"]},\"tb\":{\"preferred\":[\"l2\",\"l3\"]},\"tc\":{\"required\":[\"l2\"],\"preferred\":[\"l1\"]}}");
  const int ta = mmp_type_id(f, "ta"), tb = mmp_type_id(f, "tb"), tc = mmp_type_id(f, "tc");
  const int64_t now = 1760000000000LL;
  std::vector<mmp_instance_row> irows(NI);
  for (int i = 0; i < NI; i++) {
    mmp_instance_row r = {};
    r.capacity = 25600 + (rnd() % 4) * 1000;
    r.used = rnd() % 3 == 0 ? r.capacity - (rnd() % 3000) : rnd() % (uint32_t)r.capacity;
    r.lru_time = now - (int64_t)(rnd() % 7200000);
    r.count = rnd() % 30; r.l_threads = 8; r.l_in_prog = rnd() % 3; r.rpm = rnd() % 400; r.start_time = now - 86400000; r.vers = 1;
    r.active = 1;
    irows[i] = r;
    std::string id = "pod-" + std::to_string(100000 + i);
    const char *labs[3]; int nl = 0;
    if (rnd() % 2) labs[nl++] = "l1";
    if (rnd() % 3 == 0) labs[nl++] = "l2";
    if (rnd() % 4 == 0) labs[nl++] = "l3";
    REQ(mmp_instance_upsert(f, i, &r, id.c_str(), nullptr, (i % 3) ? "z1" : "z2", labs, nl), "upsert");
  }
  std::vector<int> long_models;  // more than 4 registrations: the closed loop needs them trimmed
  std::vector<mmp_model_row> mrows(NM);
  std::vector<std::vector<int32_t>> mids(NM);
  for (int m = 0; m < NM; m++) {
    mmp_model_row r = {};
    r.last_used = now - (int64_t)(rnd() % 100000000); r.size_units = 256 + rnd() % 4000;
    const int ts[4] = {0, ta, tb, tc};
    r.type_id = (uint16_t)ts[rnd() % 4];
    int32_t ids[6]; int n = rnd() % 7 == 0 ? 6 : rnd() % 4;
    for (int k = 0; k < n; k++) ids[k] = (int32_t)(rnd() % NI);
    r.copy_count = (uint8_t)n;
    mrows[m] = r; mids[m].assign(ids, ids + n);
    if (n > 4) long_models.push_back(m);
    REQ(mmp_model_upsert(f, m, &r, ids, n), "model");
  }
  REQ(mmp_fleet_commit(f), "commit");
  std::vector<mmp_decision_in> d(ND);
  std::vector<int32_t> extra;
  for (int i = 0; i < ND; i++) {
    d[i].model = (int32_t)(rnd() % NM); d[i].self = (int32_t)(rnd() % NI); d[i].last_used = now - (int64_t)(rnd() % 4000000);
    d[i].flags = (rnd() % 3 == 0 ? MMP_DF_FAVOUR_SELF : 0) | (rnd() % 2 ? MMP_DF_MODEL_LAST_USED : 0);
    d[i].fresh = -1; d[i].extra_off = (int32_t)extra.size(); d[i].extra_n = rnd() % 9 == 0 ? 2 : 0;
    for (int k = 0; k < d[i].extra_n; k++) extra.push_back((int32_t)(rnd() % NI));
  }
  std::vector<mmp_decision_out> a(ND), b(ND);
  std::vector<mmp_decision_trace> tr(ND);
  REQ(mmp_place_batch(f, d.data(), ND, nullptr, 0, extra.data(), (int32_t)extra.size(), a.data(), now, 7), "place");
  REQ(mmp_place_batch_trace(f, d.data(), ND, nullptr, 0, extra.data(), (int32_t)extra.size(), b.data(), tr.data(), nullptr, now, 7), "trace");
  int bad = 0, none = 0;
  for (int i = 0; i < ND; i++) { bad += a[i].target != b[i].target || a[i].n_candidates != b[i].n_candidates; none += a[i].target == MMP_TARGET_NONE; }
  // single decisions through the captured graph (one_mode 2) and the resident server (3): the batch's answer for decision 0
  for (int mode : {2, 3}) {
    mmp_decision_out one = {};
    REQ(mmp_tune(f, "one_mode", mode), "tune");
    REQ(mmp_place_one(f, &d[0], nullptr, extra.data(), &one, now, 7), "place_one");
    bad += one.target != a[0].target || one.n_candidates != a[0].n_candidates;
  }
  std::vector<int32_t> self(ND);
  for (int i = 0; i < ND; i++) self[i] = d[i].self;
  std::vector<mmp_decision_out> c(NM < ND ? NM : ND);
  REQ(mmp_place_sweep(f, 0, (int32_t)c.size(), self.data(), 1, nullptr, c.data(), now, 7), "sweep");
  // a device-path commit: numeric instance updates, and the models with more than 4 registrations cut to their first 4
  for (int i = 0; i < NI; i += 7) { irows[i].used = irows[i].used / 2; irows[i].lru_time -= 1000; REQ(mmp_instance_update(f, i, &irows[i]), "update"); }
  for (int m : long_models) { mrows[m].copy_count = 4; REQ(mmp_model_upsert(f, m, &mrows[m], mids[m].data(), 4), "trim"); }
  REQ(mmp_fleet_commit(f), "commit 2");
  int32_t path = 0;
  mmp_commit_info(f, &path, nullptr);
  if (path != 2) { fprintf(stderr, "second commit took path %d, not the device path\n", path); return 2; }
  // a batch under a call-wide exclude set
  std::vector<int32_t> excl;
  for (int k = 0; k < 40; k++) excl.push_back((int32_t)(rnd() % NI));
  REQ(mmp_place_batch_excluding(f, d.data(), ND, nullptr, 0, extra.data(), (int32_t)extra.size(), excl.data(), (int32_t)excl.size(), a.data(),
                                nullptr, nullptr, now, 9), "excluding");
  // stats, the reaper, the registry prune
  std::vector<mmp_cluster_stats> st(64);
  std::vector<int32_t> parts(64);
  REQ(mmp_stats(f, st.data(), parts.data(), 64), "stats");
  std::vector<uint8_t> taken(NM, 0);
  std::vector<int32_t> picked(NM);
  REQ(mmp_reaper_select(f, -1, now, taken.data(), picked.data(), NM), "reaper");
  std::vector<int64_t> missing(NI, 0);
  std::vector<uint8_t> masks(NM);
  REQ(mmp_registry_prune(f, 0, now, 600000, missing.data(), picked.data(), masks.data(), NM), "prune");
  // the closed loop: LRU store, churn state, two windows
  std::vector<int64_t> cap(NI);
  for (int i = 0; i < NI; i++) cap[i] = irows[i].capacity;
  REQ(mmp_lru_init(f, NI, cap.data(), 64), "lru_init");
  mmp_churn_config cc = {30000, now - 60000, 64, 0};
  REQ(mmp_churn_init(f, &cc), "churn_init");
  const int NE = 2000;
  std::vector<mmp_churn_event> ev(NE);
  std::vector<mmp_churn_decision> dec(4 * NE);
  std::vector<mmp_churn_eviction> evi(16 * NE);
  for (int w = 0; w < 2; w++) {
    const int64_t t0 = now + 2000 * w;
    for (int k = 0; k < NE; k++)
      ev[k] = mmp_churn_event{rnd() % 50 == 0 ? MMP_CHURN_REMOVE : MMP_CHURN_REQUEST, (int32_t)(rnd() % NM), (int32_t)(rnd() % NI), rnd(), t0 + k};
    int32_t n_dec = 0, n_evict = 0;
    REQ(mmp_churn_step(f, ev.data(), NE, t0, t0 + 2000, 11 + w, dec.data(), (int32_t)dec.size(), &n_dec, evi.data(), (int32_t)evi.size(),
                       &n_evict, nullptr, nullptr), "churn_step");
  }
  printf("driver: %d decisions, lanes vs traced (and single) mismatches %d, none %d, launches %lld\n", ND, bad, none,
         (long long)mmp_kernel_launches(f));
  mmp_fleet_destroy(f);
  return bad ? 1 : 0;
}

int main(int argc, char **argv) {
  const int NI = argc > 1 ? atoi(argv[1]) : 1500, NM = argc > 2 ? atoi(argv[2]) : 4000, ND = argc > 3 ? atoi(argv[3]) : 6000;
  const int rounds = argc > 4 ? atoi(argv[4]) : 2;
  int rc = 0;
  for (int r = 0; r < rounds && rc == 0; r++) {
    size_t free0 = 0, free1 = 0, total = 0;
    cudaMemGetInfo(&free0, &total);
    rc = run(NI, NM, ND);
    cudaMemGetInfo(&free1, &total);
    printf("round %d: device memory not given back after mmp_fleet_destroy: %.1f MiB\n", r, ((double)free0 - (double)free1) / (1 << 20));
  }
  return rc;
}
