// Membership changes under ClusterUpgradeStateManagerImpl::ApplyStateIncremental: the two-world scenario of
// incremental_spec.hpp, but between reconciles nodes also leave, join at random positions of BuildState's pod list and
// come back under the names of nodes that left. After every reconcile the world reconciled with ApplyStateIncremental
// must be indistinguishable from the one reconciled with ApplyState (same error, labels, annotations, actuator calls),
// and the cache must have followed the membership change by a splice: one full upload in the whole run, exactly the
// changed and the joined nodes encoded per reconcile, one slot per node of the current snapshot.
#pragma once
#include <set>

#include "incremental_spec.hpp"

namespace spec {

// A PodManager whose revision-hash lookup fails for chosen pods (pod_manager.go:84-89): ApplyState aborts with an error
// when its pass reaches such a node.
struct HashErrorPods : PodManagerMock {
  std::set<std::string> broken;  // pod names
  Error GetPodControllerRevisionHash(const Pod* pod, std::string* hash) override {
    if (broken.count(pod->Name)) return Errorf("controller-revision-hash label not present for pod " + pod->Name);
    return PodManagerMock::GetPodControllerRevisionHash(pod, hash);
  }
};

// A World whose pod-list order is kept apart from where the objects are stored, so that a node can join anywhere in it.
struct MWorld : World {
  HashErrorPods hashPods;          // wired instead of World::pods by the scenarios that need a failing lookup
  std::vector<size_t> list;        // BuildState's pod list: indices into nodes / podObjs
  std::vector<std::string> born;   // the name each stored node was created with
  std::vector<char> counted;       // stored node whose departure has been noted
  std::vector<std::string> gone;   // names of nodes that left (candidates to rejoin)
  int fresh = 0;
  void listSnapshot() {
    state = ClusterUpgradeState();
    entries.clear();
    for (size_t p = 0; p < list.size(); p++) {
      const size_t i = list[p];
      if (nodes[i].Name.empty()) continue;
      entries.emplace_back();
      NodeUpgradeState& e = entries.back();
      e.Node = &nodes[i];
      e.ListIndex = (int64_t)p;
      e.DriverPod = &podObjs[i];
      e.DriverDaemonSet = (i % 17 == 3) ? nullptr : &daemonSet;
      state.NodeStates[getNodeUpgradeState(&nodes[i])].push_back(&e);
    }
  }
};

inline void mpopulate(MWorld& w, int n, uint64_t seed) {
  populate(w, n, seed);
  for (int i = 0; i < n; i++) { w.list.push_back((size_t)i); w.born.push_back(w.nodes[(size_t)i].Name); w.counted.push_back(0); }
}

// a node that joins: a new object (what the API server hands out after a node is re-created), at list position `pos`
inline void join(MWorld& w, Lcg& r, const std::string& name, size_t pos) {
  const char* states[] = {"", UpgradeStateUpgradeRequired, UpgradeStateDone, UpgradeStateFailed, UpgradeStateCordonRequired,
                          UpgradeStatePodRestartRequired, "some-other-label"};
  // resourceVersions come from one counter of the API server: a re-created object never repeats its predecessor's
  const std::string rv = std::to_string(1000000 + 1000 * (int64_t)w.nodes.size());
  w.nodes.emplace_back();
  Node& nd = w.nodes.back();
  nd.Name = name;
  nd.ResourceVersion = rv;
  nd.Labels[GetUpgradeStateLabelKey()] = states[r.next() % (sizeof(states) / sizeof(states[0]))];
  nd.Unschedulable = r.chance(15);
  if (r.chance(5)) nd.Labels[GetUpgradeSkipNodeLabelKey()] = "true";
  if (r.chance(5)) nd.Annotations[GetUpgradeRequestedAnnotationKey()] = "true";
  if (r.chance(4)) nd.Conditions.push_back({"Ready", "False"});
  w.podObjs.emplace_back();
  Pod& p = w.podObjs.back();
  p.Name = "pod-of-" + name + "-" + std::to_string(w.podObjs.size());
  p.ResourceVersion = rv;
  p.NodeName = name;
  p.Labels[PodControllerRevisionHashLabelKey] = r.chance(50) ? "test-hash-12345" : "test-hash-outdated";
  p.Phase = r.chance(90) ? "Running" : "Pending";
  p.ContainerStatuses = {{r.chance(85), (int)(r.next() % 14)}};
  w.born.push_back(name);
  w.counted.push_back(0);
  w.list.insert(w.list.begin() + (std::ptrdiff_t)(pos < w.list.size() ? pos : w.list.size()), w.nodes.size() - 1);
}

// What the cluster's membership does between two reconciles (after evolve): joins, rejoins under the names of nodes that
// were gone at the last reconcile, leaves. (A node that leaves and comes back between two reconciles is, to the cache,
// one node that moved in the list: a reordering, which the cache answers with a full re-encode.)
inline void churn(MWorld& w, Lcg r, int rec) {
  const int joins = 1 + (int)(r.next() % 8);
  const size_t at = r.next() % (w.list.size() + 1);
  for (int j = 0; j < joins; j++) {
    size_t pos = r.next() % (w.list.size() + 1);
    if (rec % 4 == 1 && j < 2) pos = 0;               // at the head of the list
    if (rec % 4 == 2 && j < 2) pos = w.list.size();   // at its end
    if (rec % 4 == 3) pos = at;                       // many at one position
    std::string name;
    if (!w.gone.empty() && r.chance(40)) {  // a node that left comes back under its old name
      const size_t g = r.next() % w.gone.size();
      name = w.gone[g];
      w.gone.erase(w.gone.begin() + (std::ptrdiff_t)g);
    } else {
      name = "joined-" + std::to_string(w.fresh++);
    }
    join(w, r, name, pos);
  }
  for (size_t i = 0; i < w.nodes.size(); i++)
    if (!w.nodes[i].Name.empty() && r.chance(2)) w.nodes[i].Name.clear();  // more nodes leave than evolve() lets go
  for (size_t i = 0; i < w.nodes.size(); i++)
    if (w.nodes[i].Name.empty() && !w.counted[i]) { w.counted[i] = 1; w.gone.push_back(w.born[i]); }
}

// the resourceVersions an entry's encoding is keyed on, per node name
using VersionMap = std::map<std::string, std::pair<std::string, std::string>>;
inline VersionMap versions(const MWorld& w) {
  VersionMap v;
  for (const NodeUpgradeState& e : w.entries) v[e.Node->Name] = {e.Node->ResourceVersion, e.DriverPod->ResourceVersion};
  return v;
}

inline void run_membership(Runner& R, const MakeFn& makeFull, const WorldApplyFn& applyFull, const MakeFn& makeIncr,
                           const WorldApplyFn& applyIncr, const std::function<std::string()>& backendCheck, int n_nodes) {
  SetDriverName("gpu");
  R.it("ApplyStateIncremental == ApplyState while nodes leave, join anywhere in the list and rejoin (splice of the cache)", [&] {
    MWorld a, b;
    a.m = makeFull({}); a.wire();
    b.m = makeIncr({}); b.wire();
    mpopulate(a, n_nodes, 7); mpopulate(b, n_nodes, 7);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    p.MaxParallelUpgrades = 7;
    p.MaxUnavailable = IntOrString::FromString("25%");
    p.DrainSpec = upgrade::DrainSpec{};
    p.DrainSpec->Enable = true;
    VersionMap before;
    int64_t joinedTotal = 0, leftTotal = 0;
    for (int rec = 0; rec < 16; rec++) {
      if (rec == 6) p.MaxParallelUpgrades = 0;
      if (rec == 10) p.MaxUnavailable = IntOrString::FromString("60%");
      a.listSnapshot(); b.listSnapshot();
      const VersionMap now = versions(b);
      int64_t expectEncoded = 0, joined = 0;
      for (const auto& kv : now) {
        auto it = before.find(kv.first);
        if (it == before.end()) { expectEncoded++; joined++; } else if (it->second != kv.second) expectEncoded++;
      }
      int64_t left = 0;
      for (const auto& kv : before) left += now.count(kv.first) == 0;
      if (rec > 0) { joinedTotal += joined; leftTotal += left; }
      const auto st0 = b.m->Stats();
      const Error ea = applyFull(a, &p), eb = applyIncr(b, &p);
      const auto& st = b.m->Stats();
      EXPECT(R, ea.has_value() == eb.has_value());
      EXPECT(R, image(a) == image(b));
      EXPECT(R, names(a.cordon.cordoned) == names(b.cordon.cordoned));
      EXPECT(R, names(a.cordon.uncordoned) == names(b.cordon.uncordoned));
      EXPECT(R, pnames(a.pods.restarted) == pnames(b.pods.restarted));
      EXPECT(R, a.drain.calls == b.drain.calls && a.pods.evictionCalls == b.pods.evictionCalls && a.pods.waitCalls == b.pods.waitCalls);
      EXPECT(R, st.encoded - st0.encoded == expectEncoded);       // the changed and the joined nodes, nothing else
      EXPECT(R, st.slots == (int64_t)b.entries.size());           // one slot per node of this snapshot
      if (rec > 0) EXPECT(R, st.inserted - st0.inserted == joined && st.removed - st0.removed == left);
      const std::string backend = backendCheck();
      if (!backend.empty()) std::printf("    %s\n", backend.c_str());
      EXPECT(R, backend.empty());
      if (R.failed_here) { std::printf("    (reconcile %d: %lld encoded, %lld expected)\n", rec, (long long)(st.encoded - st0.encoded), (long long)expectEncoded); break; }
      before = now;
      evolve(a, Lcg{2000u + (uint64_t)rec}); evolve(b, Lcg{2000u + (uint64_t)rec});
      churn(a, Lcg{3000u + (uint64_t)rec}, rec); churn(b, Lcg{3000u + (uint64_t)rec}, rec);
    }
    const auto& st = b.m->Stats();
    std::printf("    membership: %lld reconciles, %lld full uploads, %lld encoded, %lld reused, %lld inserted, %lld removed, %lld outputs received\n",
                (long long)st.reconciles, (long long)st.full_uploads, (long long)st.encoded, (long long)st.reused, (long long)st.inserted,
                (long long)st.removed, (long long)st.outputs_received);
    EXPECT(R, st.full_uploads == 1);                      // joins and leaves never force a re-upload
    EXPECT(R, joinedTotal > 0 && leftTotal > 0);          // the scenario did change the membership
    EXPECT(R, st.inserted == joinedTotal && st.removed == leftTotal);
  });

  // A node pool joins in one reconcile: more new nodes than the incremental path's sparse-output arrays hold, so the
  // outputs must be fetched in full - and one of the new nodes aborts the reconcile, so the call returns the abort's code
  // rather than UST_ERR_TRUNCATED. The next reconcile, with the node repaired, must agree again.
  R.it("ApplyStateIncremental == ApplyState when a node pool larger than the sparse outputs joins together with a node that aborts", [&] {
    MWorld a, b;
    a.m = makeFull({}); a.wire(); a.m->PodManager = &a.hashPods;
    b.m = makeIncr({}); b.wire(); b.m->PodManager = &b.hashPods;
    mpopulate(a, n_nodes, 11); mpopulate(b, n_nodes, 11);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    p.MaxParallelUpgrades = 5;
    const int pool = 2 * n_nodes + 2000;  // > n_new / 4 + 1024 outputs, whatever n_nodes is
    auto compare = [&](const Error& ea, const Error& eb) {
      EXPECT(R, ea.has_value() == eb.has_value());
      EXPECT(R, image(a) == image(b));
      EXPECT(R, names(a.cordon.cordoned) == names(b.cordon.cordoned));
      EXPECT(R, names(a.cordon.uncordoned) == names(b.cordon.uncordoned));
      EXPECT(R, pnames(a.hashPods.restarted) == pnames(b.hashPods.restarted));
      EXPECT(R, a.drain.calls == b.drain.calls && a.hashPods.evictionCalls == b.hashPods.evictionCalls);
      const std::string backend = backendCheck();
      if (!backend.empty()) std::printf("    %s\n", backend.c_str());
      EXPECT(R, backend.empty());
    };
    a.listSnapshot(); b.listSnapshot();
    compare(applyFull(a, &p), applyIncr(b, &p));
    std::string brokenPod;
    for (MWorld* w : {&a, &b}) {
      w->cordon.cordoned.clear(); w->cordon.uncordoned.clear(); w->hashPods.restarted.clear();
      Lcg r{4242};
      const size_t first = w->nodes.size();
      for (int j = 0; j < pool; j++) join(*w, r, "pool-" + std::to_string(j), r.next() % (w->list.size() + 1));
      // a new node in the upgrade-done pass, owned by the DaemonSet, whose pod's revision hash cannot be read
      size_t i = first;
      while (i % 17 == 3) i++;
      w->nodes[i].Labels[GetUpgradeStateLabelKey()] = UpgradeStateDone;
      w->hashPods.broken.insert(w->podObjs[i].Name);
      brokenPod = w->podObjs[i].Name;
    }
    a.listSnapshot(); b.listSnapshot();
    const Error ea = applyFull(a, &p), eb = applyIncr(b, &p);
    compare(ea, eb);
    EXPECT(R, eb.has_value() && b.m->LastCounters().error_code == UST_ERR_REVISION_HASH);  // the reconcile did abort
    // the label appears: the pod object changes (and with it its resourceVersion)
    for (MWorld* w : {&a, &b}) {
      w->cordon.cordoned.clear(); w->cordon.uncordoned.clear(); w->hashPods.restarted.clear();
      w->hashPods.broken.clear();
      for (Pod& pd : w->podObjs)
        if (pd.Name == brokenPod) pd.ResourceVersion = std::to_string(std::stoll(pd.ResourceVersion) + 1);
    }
    a.listSnapshot(); b.listSnapshot();
    compare(applyFull(a, &p), applyIncr(b, &p));
    const auto& st = b.m->Stats();
    std::printf("    node pool: %lld full uploads, %lld inserted, %lld outputs received\n", (long long)st.full_uploads,
                (long long)st.inserted, (long long)st.outputs_received);
    EXPECT(R, st.full_uploads == 1 && st.inserted == pool);
  });
}

}  // namespace spec
