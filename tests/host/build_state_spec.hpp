// The whole reconcile loop incrementally: BuildStateIncremental + ApplyStateIncremental on one manager against
// BuildState + ApplyState on a fresh manager every reconcile. Two identical worlds of driver DaemonSets, nodes and driver
// pods behind K8sClientMock; between reconciles the world moves the way a cluster does:
//   pods change phase, unscheduled pending pods get scheduled, nodes join and leave, restarted driver pods come back under
//   new names (they move in a list sorted by name), a DaemonSet is re-created with a new UID (its pods become orphans,
//   then are replaced by pods of the new DaemonSet), a few pods are owned by something else (dropped from the snapshot),
//   and DesiredNumberScheduled sometimes disagrees (an error reconcile, then recovery).
// After every reconcile both worlds must agree on the error, the snapshot (buckets, entry order, ListIndex, driver pod,
// DaemonSet, NodeMaintenance), the node labels / annotations and the provider / actuator call sequence; over the whole run
// each cache makes one full upload.
#pragma once
#include <algorithm>
#include <cstdio>
#include <deque>

#include "mocks.hpp"

namespace spec {
using namespace upgrade;
using namespace mocks;

using MakeBuildFn = std::function<std::unique_ptr<ClusterUpgradeStateManagerImpl>()>;

struct BLcg {
  uint64_t s;
  uint32_t next() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); }
  bool chance(int pct) { return next() % 100 < (uint32_t)pct; }
};

// Provider and actuators that record every call, in order; label / annotation writes bump the node's resourceVersion.
struct LogProvider : NodeUpgradeStateProviderMock {
  std::vector<std::string>* log = nullptr;
  static void bump(Node* n) { n->ResourceVersion = std::to_string(std::stoll(n->ResourceVersion) + 1); }
  Error ChangeNodeUpgradeState(Node* n, const std::string& s) override {
    log->push_back("state " + n->Name + "=" + s);
    bump(n);
    return NodeUpgradeStateProviderMock::ChangeNodeUpgradeState(n, s);
  }
  Error ChangeNodeUpgradeAnnotation(Node* n, const std::string& k, const std::string& v) override {
    log->push_back("annotation " + n->Name + " " + k + "=" + v);
    bump(n);
    return NodeUpgradeStateProviderMock::ChangeNodeUpgradeAnnotation(n, k, v);
  }
};
struct LogCordon : CordonManager {
  std::vector<std::string>* log = nullptr;
  std::vector<Node*> cordoned, uncordoned;
  Error Cordon(Node* n) override { log->push_back("cordon " + n->Name); cordoned.push_back(n); return std::nullopt; }
  Error Uncordon(Node* n) override { log->push_back("uncordon " + n->Name); uncordoned.push_back(n); return std::nullopt; }
};
struct LogDrain : DrainManager {
  std::vector<std::string>* log = nullptr;
  Error ScheduleNodesDrain(const DrainConfiguration& c) override {
    std::string s = "drain";
    for (Node* n : c.Nodes) s += " " + n->Name;
    log->push_back(s);
    return std::nullopt;
  }
};
struct LogPods : PodManagerMock {
  std::vector<std::string>* log = nullptr;
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& c) override { log->push_back("wait " + std::to_string(c.Nodes.size())); return std::nullopt; }
  Error SchedulePodEviction(const PodManagerConfig& c) override { log->push_back("evict " + std::to_string(c.Nodes.size())); return std::nullopt; }
  Error SchedulePodsRestart(const std::vector<Pod*>& pods) override {
    std::string s = "restart";
    for (Pod* p : pods) s += " " + p->Name;
    log->push_back(s);
    restarted.insert(restarted.end(), pods.begin(), pods.end());
    return std::nullopt;
  }
};

struct BWorld {
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m;
  std::vector<std::string> log;
  LogProvider provider;
  LogCordon cordon;
  LogDrain drain;
  LogPods pods;
  ValidationManagerMock validation;
  SafeDriverLoadManagerImpl safeLoad{&provider};
  K8sClientMock client;
  std::deque<Node> nodes;
  std::deque<Pod> podObjs;
  std::vector<char> alive;       // per pod object
  std::deque<DaemonSet> dss;
  std::vector<size_t> liveDs;    // DaemonSets that exist, in the order ListDaemonSets returns them
  int64_t version = 100;         // the API server's resourceVersion counter
  int extraDesired = 0;          // added to DaemonSet 0's DesiredNumberScheduled on the next reconcile
  std::unique_ptr<ClusterUpgradeState> state;

  BWorld() { provider.log = cordon.log = drain.log = pods.log = &log; }
  void wire(ClusterUpgradeStateManagerImpl* mm) {
    mm->NodeUpgradeStateProvider = &provider; mm->DrainManager = &drain; mm->CordonManager = &cordon; mm->PodManager = &pods;
    mm->ValidationManager = &validation; mm->SafeDriverLoadManager = &safeLoad; mm->K8sClient = &client;
  }
  std::string rv() { return std::to_string(version++); }
  void bumpPod(Pod& p) { p.ResourceVersion = rv(); }
  DaemonSet& addDs(const std::string& name) {
    dss.emplace_back();
    dss.back().Name = name;
    dss.back().UID = "uid-" + name + "-" + rv();
    liveDs.push_back(dss.size() - 1);
    return dss.back();
  }
  void addPod(const std::string& name, const std::string& node, const std::string& ownerUid, bool pending, BLcg& r) {
    podObjs.emplace_back();
    Pod& p = podObjs.back();
    p.Name = name;
    p.Namespace = "gpu-operator";
    p.ResourceVersion = rv();
    p.NodeName = pending ? "" : node;
    if (!ownerUid.empty()) p.OwnerReferences.push_back({"DaemonSet", "driver", ownerUid});
    p.Labels[PodControllerRevisionHashLabelKey] = r.chance(60) ? "test-hash-12345" : "test-hash-outdated";
    p.Phase = pending ? "Pending" : (r.chance(90) ? "Running" : "Pending");
    p.ContainerStatuses = {{r.chance(85), (int)(r.next() % 14)}};
    alive.push_back(1);
  }
  void addNode(const std::string& name, BLcg& r) {
    const char* states[] = {"", UpgradeStateUpgradeRequired, UpgradeStateCordonRequired, UpgradeStateDrainRequired,
                            UpgradeStatePodRestartRequired, UpgradeStateValidationRequired, UpgradeStateUncordonRequired,
                            UpgradeStateDone, UpgradeStateDone, UpgradeStateFailed, "some-other-label"};
    nodes.emplace_back();
    Node& nd = nodes.back();
    nd.Name = name;
    nd.ResourceVersion = rv();
    nd.Labels[GetUpgradeStateLabelKey()] = states[r.next() % (sizeof(states) / sizeof(states[0]))];
    nd.Unschedulable = r.chance(10);
    if (r.chance(3)) nd.Labels[GetUpgradeSkipNodeLabelKey()] = "true";
    if (r.chance(4)) nd.Conditions.push_back({"Ready", "False"});
    provider.nodes[name] = &nd;
  }
  // what ListDaemonSets / ListPods return now: the pods sorted by name, DesiredNumberScheduled = owned pods (+ extraDesired)
  void publish() {
    client.daemonSets.clear();
    for (size_t d : liveDs) {
      int owned = 0;
      for (size_t i = 0; i < podObjs.size(); i++)
        owned += alive[i] && !podObjs[i].OwnerReferences.empty() && podObjs[i].OwnerReferences[0].UID == dss[d].UID;
      dss[d].DesiredNumberScheduled = owned + (d == liveDs[0] ? extraDesired : 0);
      client.daemonSets.push_back(&dss[d]);
    }
    client.pods.clear();
    for (size_t i = 0; i < podObjs.size(); i++)
      if (alive[i]) client.pods.push_back(&podObjs[i]);
    std::stable_sort(client.pods.begin(), client.pods.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
  }
};

inline void bpopulate(BWorld& w, int n, uint64_t seed) {
  BLcg r{seed};
  w.addDs("driver-a");
  w.addDs("driver-b");
  for (int i = 0; i < n; i++) {
    const std::string node = "node-" + std::to_string(i);
    w.addNode(node, r);
    // a few pods owned by something that is not a driver DaemonSet (index -2: not in the snapshot)
    const std::string owner = i % 29 == 5 ? "uid-some-replicaset" : w.dss[w.liveDs[(size_t)i % 2]].UID;
    w.addPod("drv-" + node, node, i % 23 == 7 ? "" : owner, false, r);
  }
}

// The cluster between two reconciles; identical on both worlds (same seed, same actuator records).
inline void bevolve(BWorld& w, int rec, BLcg r) {
  for (Node* n : w.cordon.cordoned) { n->Unschedulable = true; LogProvider::bump(n); }
  for (Node* n : w.cordon.uncordoned) { n->Unschedulable = false; LogProvider::bump(n); }
  w.cordon.cordoned.clear(); w.cordon.uncordoned.clear();
  for (Pod* p : w.pods.restarted) {  // deleted and re-created by the DaemonSet controller: a new name, the current revision
    p->Name = "drv-r" + std::to_string(r.next() % 1000000);
    p->Labels[PodControllerRevisionHashLabelKey] = "test-hash-12345";
    p->Phase = "Running"; p->ContainerStatuses = {{true, 0}};
    w.bumpPod(*p);
  }
  w.pods.restarted.clear();
  w.extraDesired = rec % 25 == 7 ? 1 : 0;  // the next reconcile finds a DaemonSet with unscheduled pods
  for (size_t i = 0; i < w.podObjs.size(); i++) {
    if (!w.alive[i]) continue;
    Pod& p = w.podObjs[i];
    if (p.NodeName.empty() && r.chance(60)) {  // an unscheduled pending pod gets scheduled
      p.NodeName = p.Name.substr(0, 4) == "drv-" && w.provider.nodes.count(p.Name.substr(4)) ? p.Name.substr(4) : p.NodeName;
      if (!p.NodeName.empty()) { p.Phase = "Running"; w.bumpPod(p); }
    } else if (r.chance(3)) {  // phase / readiness changes
      p.Phase = r.chance(80) ? "Running" : "Failed";
      p.ContainerStatuses = {{r.chance(70), (int)(r.next() % 14)}};
      w.bumpPod(p);
    }
  }
  // nodes leave (with their driver pods)
  for (Node& nd : w.nodes) {
    if (nd.Name.empty() || !r.chance(1)) continue;
    for (size_t i = 0; i < w.podObjs.size(); i++)
      if (w.alive[i] && (w.podObjs[i].NodeName == nd.Name || w.podObjs[i].Name == "drv-" + nd.Name)) w.alive[i] = 0;
    w.provider.nodes.erase(nd.Name);
    nd.Name.clear();
  }
  // nodes join; half of their driver pods are not scheduled yet
  const int joins = (int)(r.next() % 4);
  for (int j = 0; j < joins; j++) {
    const std::string node = "node-j" + std::to_string(rec) + "-" + std::to_string(j);
    w.addNode(node, r);
    w.addPod("drv-" + node, node, w.dss[w.liveDs[r.next() % w.liveDs.size()]].UID, r.chance(50), r);
  }
  // a DaemonSet is deleted with its pods orphaned and re-created with a new UID ...
  if (rec % 60 == 20) {
    const size_t old = w.liveDs.back();
    const std::string oldUid = w.dss[old].UID;
    w.liveDs.pop_back();
    w.addDs(w.dss[old].Name);
    std::swap(w.liveDs[0], w.liveDs.back());  // ListDaemonSets returns another order too
    for (size_t i = 0; i < w.podObjs.size(); i++)
      if (w.alive[i] && !w.podObjs[i].OwnerReferences.empty() && w.podObjs[i].OwnerReferences[0].UID == oldUid) {
        w.podObjs[i].OwnerReferences.clear();
        w.bumpPod(w.podObjs[i]);
      }
  }
  // ... and two reconciles later the new DaemonSet replaces the orphans with pods of its own, under new names
  if (rec % 60 == 22) {
    const std::string uid = w.dss[w.liveDs[0]].UID;
    const size_t n0 = w.podObjs.size();
    for (size_t i = 0; i < n0; i++) {
      if (!w.alive[i] || !w.podObjs[i].OwnerReferences.empty() || i % 23 == 7 || w.podObjs[i].NodeName.empty()) continue;
      w.alive[i] = 0;
      const std::string node = w.podObjs[i].NodeName;
      w.addPod("drv-n" + std::to_string(r.next() % 1000000) + "-" + node, node, uid, false, r);
    }
  }
}

// Everything of a snapshot a caller can see, by name.
inline std::string describe(const ClusterUpgradeState* s) {
  if (!s) return "(none)";
  std::string d;
  for (const auto& kv : s->NodeStates) {
    d += "[" + kv.first + "]";
    for (const NodeUpgradeState* e : kv.second)
      d += " " + e->Node->Name + "/" + e->DriverPod->Name + "/" + (e->DriverDaemonSet ? e->DriverDaemonSet->UID : "-") + "/" +
           std::to_string(e->ListIndex) + (e->NodeMaintenance ? "/NM" : "");
  }
  return d;
}
inline std::string bimage(const BWorld& w) {
  std::string s;
  for (const Node& n : w.nodes) {
    s += n.Name + "{" + (n.Labels.count(GetUpgradeStateLabelKey()) ? n.Labels.at(GetUpgradeStateLabelKey()) : "") + (n.Unschedulable ? ",U" : "");
    for (const auto& kv : n.Annotations) s += "," + kv.first + "=" + kv.second;
    s += "}";
  }
  return s;
}

using BuildFn = std::function<Error(BWorld&, std::unique_ptr<ClusterUpgradeState>*)>;
using ApplyFn = std::function<Error(BWorld&, ClusterUpgradeState*, const DriverUpgradePolicySpec*)>;

inline void run_build_state(Runner& R, const MakeBuildFn& makeFull, const BuildFn& buildFull, const ApplyFn& applyFull,
                            const MakeBuildFn& makeIncr, const BuildFn& buildIncr, const ApplyFn& applyIncr,
                            const std::function<std::string()>& backendCheck, int n_nodes, int rounds) {
  SetDriverName("gpu");
  R.it("BuildStateIncremental + ApplyStateIncremental == BuildState + ApplyState over a reconcile loop with joins, leaves, moves, "
       "re-created DaemonSets and unscheduled pods", [&] {
    BWorld a, b;
    bpopulate(a, n_nodes, 77); bpopulate(b, n_nodes, 77);
    b.m = makeIncr(); b.wire(b.m.get());
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    p.MaxParallelUpgrades = 8;
    p.MaxUnavailable = IntOrString::FromString("30%");
    p.DrainSpec = upgrade::DrainSpec{};
    p.DrainSpec->Enable = true;
    int errors = 0, orphans = 0, foreign = 0;
    for (int rec = 0; rec < rounds; rec++) {
      a.m = makeFull(); a.wire(a.m.get());  // the reference's way: a fresh manager, everything from scratch
      a.publish(); b.publish();
      a.log.clear(); b.log.clear();
      std::unique_ptr<ClusterUpgradeState> sa, sb;
      Error ea = buildFull(a, &sa), eb = buildIncr(b, &sb);
      EXPECT(R, ea == eb);
      EXPECT(R, describe(ea ? nullptr : sa.get()) == describe(eb ? nullptr : sb.get()));
      if (!ea && !eb) {
        for (const auto& kv : sa->NodeStates)
          for (const NodeUpgradeState* e : kv.second) orphans += e->DriverDaemonSet == nullptr;
        ea = applyFull(a, sa.get(), &p);
        eb = applyIncr(b, sb.get(), &p);
        EXPECT(R, ea == eb);
      } else {
        errors++;
      }
      for (const Pod* pd : b.client.pods) foreign += !pd->OwnerReferences.empty() && pd->OwnerReferences[0].UID == "uid-some-replicaset";
      EXPECT(R, a.log == b.log);
      EXPECT(R, bimage(a) == bimage(b));
      const std::string backend = backendCheck();
      if (!backend.empty()) std::printf("    %s\n", backend.c_str());
      EXPECT(R, backend.empty());
      if (R.failed_here) {
        std::printf("    (reconcile %d: %s / %s)\n", rec, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        break;
      }
      bevolve(a, rec, BLcg{9000u + (uint64_t)rec}); bevolve(b, rec, BLcg{9000u + (uint64_t)rec});
    }
    const auto& bs = b.m->BuildStateStats();
    const auto& as = b.m->Stats();
    std::printf("    build state: %lld reconciles, %lld full uploads, %lld re-derived, %lld reused, %lld inserted, %lld removed, %lld reorders, "
                "%lld outputs received; apply state: %lld full uploads, %lld reorders; %d error reconciles\n",
                (long long)bs.reconciles, (long long)bs.full_uploads, (long long)bs.rederived, (long long)bs.reused, (long long)bs.inserted,
                (long long)bs.removed, (long long)bs.reorders, (long long)bs.outputs_received, (long long)as.full_uploads,
                (long long)as.reorders, errors);
    EXPECT(R, bs.reconciles == rounds);
    EXPECT(R, bs.full_uploads == 1);   // BuildState's list never left the device ...
    EXPECT(R, as.full_uploads == 1);   // ... and neither did ApplyState's snapshot
    EXPECT(R, bs.reused > bs.rederived);
    EXPECT(R, bs.inserted > 0 && bs.removed > 0 && bs.reorders > rounds / 2);
    EXPECT(R, errors >= rounds / 30 && orphans > 0 && foreign > 0);
  });
}

}  // namespace spec
