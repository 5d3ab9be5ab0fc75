// Nodes that move in BuildState's list under ClusterUpgradeStateManagerImpl::ApplyStateIncremental. Two worlds as in
// membership_spec.hpp, one reconciled with ApplyState, one with ApplyStateIncremental, must stay indistinguishable after
// every reconcile (same error, labels, annotations, actuator calls) while the list order changes the way it does in a
// cluster:
//   (a) a rollout in which every restarted driver pod is re-created under a new name and the list is sorted by pod name
//   (b) several driver DaemonSets whose blocks swap places between reconciles, with joins and leaves
//   (c) a full shuffle on every reconcile, with a reconcile that aborts on a revision-hash error and one whose changed
//       outputs overflow the sparse-output arrays
// The cache must follow by moving its slots: one full upload in the whole run, exactly the changed and the joined nodes
// encoded per reconcile. (d) A ListIndex that contradicts a bucket's slice order is still rejected.
#pragma once
#include <algorithm>
#include <cstdio>

#include "membership_spec.hpp"

namespace spec {

// An MWorld with up to three driver DaemonSets. BuildState's list is w.list, regrouped into DaemonSet blocks in
// blockOrder when there is more than one.
struct RWorld : MWorld {
  DaemonSet dss[3];
  int nds = 1;
  std::vector<int> blockOrder{0};
  RWorld() {
    for (int d = 0; d < 3; d++) { dss[d].Name = "driver-" + std::to_string(d); dss[d].UID = "ds-uid-" + std::to_string(d); dss[d].ResourceVersion = "1"; }
  }
  int dsOf(size_t i) const { return (int)(i % (size_t)nds); }
  void reorderedSnapshot() {
    std::vector<size_t> l;
    for (int b : blockOrder)
      for (size_t i : list)
        if (dsOf(i) == b) l.push_back(i);
    state = ClusterUpgradeState();
    entries.clear();
    for (size_t p = 0; p < l.size(); p++) {
      const size_t i = l[p];
      if (nodes[i].Name.empty()) continue;
      entries.emplace_back();
      NodeUpgradeState& e = entries.back();
      e.Node = &nodes[i];
      e.ListIndex = (int64_t)p;
      e.DriverPod = &podObjs[i];
      e.DriverDaemonSet = (i % 17 == 3) ? nullptr : &dss[dsOf(i)];
      state.NodeStates[getNodeUpgradeState(&nodes[i])].push_back(&e);
    }
  }
  void sortByPodName() {
    std::stable_sort(list.begin(), list.end(), [&](size_t x, size_t y) { return podObjs[x].Name < podObjs[y].Name; });
  }
  // what evolve() does with restarted pods, for the pod manager the scenarios wire (it records restarts)
  std::vector<Pod*> lastRestarted;
  void handOverRestarts() { pods.restarted = lastRestarted = hashPods.restarted; hashPods.restarted.clear(); }
};

inline void rsetup(RWorld& w, const MakeFn& make, int n, uint64_t seed) {
  w.m = make({});
  w.wire();
  w.m->PodManager = &w.hashPods;
  mpopulate(w, n, seed);
}

inline DriverUpgradePolicySpec rpolicy() {
  DriverUpgradePolicySpec p;
  p.AutoUpgrade = true;
  p.MaxParallelUpgrades = 6;
  p.MaxUnavailable = IntOrString::FromString("30%");
  p.DrainSpec = upgrade::DrainSpec{};
  p.DrainSpec->Enable = true;
  return p;
}

// One reconcile of both worlds, compared. Returns false once something differs.
inline bool rcompare(Runner& R, RWorld& a, RWorld& b, const Error& ea, const Error& eb, const std::function<std::string()>& backendCheck) {
  EXPECT(R, ea.has_value() == eb.has_value());
  EXPECT(R, image(a) == image(b));
  EXPECT(R, names(a.cordon.cordoned) == names(b.cordon.cordoned));
  EXPECT(R, names(a.cordon.uncordoned) == names(b.cordon.uncordoned));
  EXPECT(R, pnames(a.hashPods.restarted) == pnames(b.hashPods.restarted));
  EXPECT(R, a.drain.calls == b.drain.calls && a.hashPods.evictionCalls == b.hashPods.evictionCalls && a.hashPods.waitCalls == b.hashPods.waitCalls);
  const std::string backend = backendCheck();
  if (!backend.empty()) std::printf("    %s\n", backend.c_str());
  EXPECT(R, backend.empty());
  return !R.failed_here;
}

// `rounds` reconciles; before each, `move(w, rec)` changes both worlds alike (after evolve). Checks the encode count per
// reconcile and one full upload over the run; prints the stats under `label`.
inline void rrun(Runner& R, RWorld& a, RWorld& b, const WorldApplyFn& applyFull, const WorldApplyFn& applyIncr,
                 const std::function<std::string()>& backendCheck, int rounds, DriverUpgradePolicySpec& p,
                 const std::function<void(RWorld&, int)>& move, const char* label, const std::function<void(int)>& after = nullptr) {
  VersionMap before;
  for (int rec = 0; rec < rounds; rec++) {
    if (rec == 5) p.MaxParallelUpgrades = 0;
    if (rec == 8) p.MaxUnavailable = IntOrString::FromString("60%");
    move(a, rec); move(b, rec);
    a.reorderedSnapshot(); b.reorderedSnapshot();
    const VersionMap now = versions(b);
    int64_t expectEncoded = 0;
    for (const auto& kv : now) {
      auto it = before.find(kv.first);
      if (it == before.end() || it->second != kv.second) expectEncoded++;
    }
    for (RWorld* w : {&a, &b}) { w->cordon.cordoned.clear(); w->cordon.uncordoned.clear(); w->hashPods.restarted.clear(); }
    const auto st0 = b.m->Stats();
    const Error ea = applyFull(a, &p), eb = applyIncr(b, &p);
    const auto& st = b.m->Stats();
    const bool ok = rcompare(R, a, b, ea, eb, backendCheck);
    EXPECT(R, st.encoded - st0.encoded == expectEncoded);  // the changed and the joined nodes, nothing else
    EXPECT(R, st.slots == (int64_t)b.entries.size());
    if (after) after(rec);
    if (!ok || R.failed_here) {
      std::printf("    (%s, reconcile %d: %lld encoded, %lld expected)\n", label, rec, (long long)(st.encoded - st0.encoded), (long long)expectEncoded);
      break;
    }
    before = now;
    // keep the actuator records for evolve(): what the DaemonSet controller and the cordons do next
    for (RWorld* w : {&a, &b}) {
      w->handOverRestarts();
      evolve(*w, Lcg{5000u + (uint64_t)rec});
    }
  }
  const auto& st = b.m->Stats();
  std::printf("    %s: %lld reconciles, %lld full uploads, %lld reorders, %lld encoded, %lld reused, %lld inserted, %lld removed, %lld outputs received\n",
              label, (long long)st.reconciles, (long long)st.full_uploads, (long long)st.reorders, (long long)st.encoded, (long long)st.reused,
              (long long)st.inserted, (long long)st.removed, (long long)st.outputs_received);
  EXPECT(R, st.full_uploads == 1);
  EXPECT(R, st.reorders > 0);
}

inline void run_reorder(Runner& R, const MakeFn& makeFull, const WorldApplyFn& applyFull, const MakeFn& makeIncr,
                        const WorldApplyFn& applyIncr, const std::function<std::string()>& backendCheck, int n_nodes) {
  SetDriverName("gpu");
  R.it("(a) ApplyStateIncremental == ApplyState while restarted driver pods come back under new names in a list sorted by pod name", [&] {
    RWorld a, b;
    rsetup(a, makeFull, n_nodes, 21); rsetup(b, makeIncr, n_nodes, 21);
    DriverUpgradePolicySpec p = rpolicy();
    int64_t renamed = 0;
    rrun(R, a, b, applyFull, applyIncr, backendCheck, 14, p, [&](RWorld& w, int rec) {
      // the pods evolve() brought back were deleted and re-created by the DaemonSet controller: new random suffix
      Lcg r{7000u + (uint64_t)rec};
      if (rec == 0)
        for (Pod& pd : w.podObjs) pd.Name = "driver-" + std::to_string(r.next() % 100000);
      for (Pod* pd : w.lastRestarted) {
        pd->Name = "driver-" + std::to_string(r.next() % 100000);
        renamed += &w == &b;
      }
      w.lastRestarted.clear();
      w.sortByPodName();
    }, "renamed pods");
    EXPECT(R, renamed > 0);
  });

  R.it("(b) ApplyStateIncremental == ApplyState while the blocks of three driver DaemonSets swap places, with joins and leaves", [&] {
    RWorld a, b;
    rsetup(a, makeFull, n_nodes, 22); rsetup(b, makeIncr, n_nodes, 22);
    for (RWorld* w : {&a, &b}) { w->nds = 3; w->blockOrder = {0, 1, 2}; }
    DriverUpgradePolicySpec p = rpolicy();
    rrun(R, a, b, applyFull, applyIncr, backendCheck, 14, p, [&](RWorld& w, int rec) {
      static const std::vector<int> orders[] = {{0, 1, 2}, {2, 0, 1}, {1, 0, 2}, {0, 2, 1}, {1, 2, 0}};
      w.blockOrder = rec % 3 == 2 ? w.blockOrder : orders[(size_t)rec % 5];
      if (rec > 0 && rec % 2 == 0) churn(w, Lcg{8000u + (uint64_t)rec}, rec);  // joins and leaves in the same reconcile
    }, "DaemonSet blocks");
  });

  R.it("(c) ApplyStateIncremental == ApplyState under a full shuffle of the list, with an abort and an overflow of the sparse outputs", [&] {
    RWorld a, b;
    rsetup(a, makeFull, n_nodes, 23); rsetup(b, makeIncr, n_nodes, 23);
    DriverUpgradePolicySpec p = rpolicy();
    std::string brokenPod;
    rrun(R, a, b, applyFull, applyIncr, backendCheck, 12, p, [&](RWorld& w, int rec) {
      Lcg r{9000u + (uint64_t)rec};
      if (rec == 4) {  // a node pool larger than the sparse outputs joins
        const int pool = 2 * n_nodes + 2000;
        for (int j = 0; j < pool; j++) join(w, r, "pool-" + std::to_string(j), r.next() % (w.list.size() + 1));
      }
      if (rec == 7) {  // an existing node, now in the upgrade-done pass, whose pod's revision hash cannot be read
        size_t i = 40;
        while (i % 17 == 3 || w.nodes[i].Name.empty()) i++;
        w.nodes[i].Labels[GetUpgradeStateLabelKey()] = UpgradeStateDone;
        VersionedProvider::bump(&w.nodes[i]);
        w.hashPods.broken.insert(w.podObjs[i].Name);
        brokenPod = w.podObjs[i].Name;
      }
      if (rec == 8) {  // the label appears: the pod object changes
        w.hashPods.broken.clear();
        for (Pod& pd : w.podObjs)
          if (pd.Name == brokenPod) pd.ResourceVersion = std::to_string(std::stoll(pd.ResourceVersion) + 1);
      }
      for (size_t k = w.list.size(); k > 1; k--) std::swap(w.list[k - 1], w.list[r.next() % k]);
    }, "shuffle", [&](int rec) {
      if (rec == 7) EXPECT(R, b.m->LastCounters().error_code == UST_ERR_REVISION_HASH);  // the reconcile did abort
      if (rec == 8) EXPECT(R, b.m->LastCounters().error_code == UST_OK);
    });
  });

  R.it("(d) ApplyStateIncremental rejects a ListIndex that contradicts a bucket's slice order", [&] {
    RWorld b;
    rsetup(b, makeIncr, n_nodes, 24);
    DriverUpgradePolicySpec p = rpolicy();
    for (int rec = 0; rec < 2; rec++) {
      b.reorderedSnapshot();
      applyIncr(b, &p);
      b.handOverRestarts();
      evolve(b, Lcg{6000u + (uint64_t)rec});
    }
    b.reorderedSnapshot();
    std::vector<NodeUpgradeState*>* bucket = nullptr;
    for (auto& kv : b.state.NodeStates)
      if (kv.second.size() >= 2 && (!bucket || kv.second.size() > bucket->size())) bucket = &kv.second;
    EXPECT(R, bucket != nullptr);
    if (!bucket) return;
    std::swap((*bucket)[0]->ListIndex, (*bucket)[1]->ListIndex);
    const Error e = applyIncr(b, &p);
    EXPECT(R, e.has_value() && e->find("a bucket's slice order contradicts the list order") != std::string::npos);
    // consistent input again: the cache starts over with a full upload
    b.reorderedSnapshot();
    const auto st0 = b.m->Stats();
    applyIncr(b, &p);
    EXPECT(R, b.m->Stats().full_uploads == st0.full_uploads + 1);
  });
}

}  // namespace spec
