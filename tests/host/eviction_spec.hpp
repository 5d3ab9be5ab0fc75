// StateOptions::EvictionOnDevice against the reference's PodManagerImpl.SchedulePodEviction (pod_manager.go:122-229,
// :393-403) and DrainManagerImpl.ScheduleNodesDrain (drain_manager.go:58-139), restated here over a fake pod and
// DaemonSet store with kubectl's drain filter chain written out from k8s.io/kubectl pkg/drain/filters.go. The goroutines
// run one after the other, to completion, before the call returns. The device-mode manager must make the same provider,
// cordon and evictor calls per node, in the same order, and return the same error.
#pragma once
#include <cstdio>
#include <mutex>

#include "wait_spec.hpp"

namespace espec {
using namespace upgrade;
using namespace mocks;

// The fake API server: SelectorClient's pods ("" selects every pod) plus the DaemonSets a namespace-wide List returns.
struct Store : vspec::SelectorClient {
  std::vector<DaemonSet*> workloadDs;  // what ListDaemonSets("", {}) returns
  Error dsError, selectorError;  // selectorError: what a List with a non-empty selector returns instead, when set
  int dsLists = 0, allLists = 0;
  Error ListDaemonSets(const std::string& ns, const StringMap& l, std::vector<DaemonSet*>* out) override {
    if (!ns.empty()) return vspec::SelectorClient::ListDaemonSets(ns, l, out);
    dsLists++;
    if (dsError) return dsError;
    *out = workloadDs;
    return std::nullopt;
  }
  Error ListPodsBySelector(const std::string& selector, const std::string& nodeName, std::vector<Pod*>* out) override {
    if (!selector.empty()) {
      if (selectorError) { lists++; return selectorError; }
      return vspec::SelectorClient::ListPodsBySelector(selector, nodeName, out);
    }
    lists++;
    allLists++;
    if (listError) return listError;
    out->clear();
    for (Pod* p : all)
      if (nodeName.empty() || p->NodeName == nodeName) out->push_back(p);
    return std::nullopt;
  }
  bool getDaemonSet(const std::string& ns, const std::string& name) const {  // a Get: found or NotFound
    for (const DaemonSet* d : workloadDs)
      if (d->Namespace == ns && d->Name == name) return true;
    return false;
  }
};

// A PodEvictor that records its calls and can be told to fail for one node.
struct LogEvictor : PodEvictor {
  std::vector<std::string>* log = nullptr;
  std::mutex* mu = nullptr;
  std::string failNode;
  Error DeleteOrEvictPods(const Node& node, const std::vector<Pod*>& pods, const EvictionOptions& o) override {
    std::string s = "evict " + node.Name + " force=" + std::to_string(o.Force) + " emptydir=" + std::to_string(o.DeleteEmptyDir) +
                    " timeout=" + std::to_string(o.TimeoutSecond) + " grace=" + std::to_string(o.GracePeriodSeconds) + ":";
    for (const Pod* p : pods) s += " " + p->Name;
    const bool fail = node.Name == failNode;
    std::unique_lock<std::mutex> l;
    if (mu) l = std::unique_lock<std::mutex>(*mu);
    log->push_back(fail ? "FAILED " + s : s);
    return fail ? Errorf("eviction failed") : std::nullopt;
  }
};

// kubectl drain.Helper (k8s.io/kubectl pkg/drain): GetPodsForDeletion with the filter chain, and DeleteOrEvictPods,
// whose pod deletions are the PodEvictor's.
struct DrainHelper {
  Store* client = nullptr;
  PodEvictor* evictor = nullptr;
  bool Force = false, DeleteEmptyDirData = false;
  int TimeoutSecond = 0;
  std::string PodSelector;
  PodDeletionFilter additional;  // AdditionalFilters: delete when true, skip otherwise
  enum Status { Okay, Skip, Fail };
  static bool finished(const Pod& p) { return p.Phase == "Succeeded" || p.Phase == "Failed"; }
  static const OwnerReference* GetControllerOf(const Pod& p) {
    for (const auto& o : p.OwnerReferences)
      if (o.Controller) return &o;
    return nullptr;
  }
  // filters.go: skipDeletedFilter (inactive: SkipWaitForDeleteTimeoutSeconds is 0), daemonSetFilter with
  // IgnoreAllDaemonSets, mirrorPodFilter, localStorageFilter, unreplicatedFilter, then the additional filters; the first
  // status that does not delete is the pod's.
  Status filter(const Pod& pod) const {
    if (const OwnerReference* c = GetControllerOf(pod))
      if (c->Kind == "DaemonSet" && !finished(pod)) {
        if (!client->getDaemonSet(pod.Namespace, c->Name)) {
          if (!Force) return Fail;  // NotFound without --force
        } else {
          return Skip;  // IgnoreAllDaemonSets: a warning, not deleted
        }
      }
    if (pod.Annotations.count("kubernetes.io/config.mirror")) return Skip;
    if (pod.HasEmptyDirVolume && !finished(pod) && !DeleteEmptyDirData) return Fail;
    if (!finished(pod) && GetControllerOf(pod) == nullptr && !Force) return Fail;
    if (additional && !additional(pod)) return Skip;
    return Okay;
  }
  // the pods to delete, or the errors
  int GetPodsForDeletion(const std::string& node, std::vector<Pod*>* pods) const {
    std::vector<Pod*> listed;
    if (Error e = client->ListPodsBySelector(PodSelector, node, &listed)) return 1;
    int errs = 0;
    for (Pod* p : listed) {
      const Status s = filter(*p);
      if (s == Okay) pods->push_back(p);
      errs += s == Fail;
    }
    return errs;
  }
  Error DeleteOrEvictPods(const Node& node, const std::vector<Pod*>& pods) const {
    if (pods.empty()) return std::nullopt;
    EvictionOptions o;
    o.Force = Force; o.DeleteEmptyDir = DeleteEmptyDirData; o.TimeoutSecond = TimeoutSecond;
    return evictor->DeleteOrEvictPods(node, pods, o);
  }
};

// pod_manager.go:122-229, :393-403, with the wait-for-completion check of wait_spec.hpp
struct PodManagerImpl : wspec::PodManagerImpl {
  Store* store = nullptr;
  PodEvictor* evictor = nullptr;
  PodDeletionFilter podDeletionFilter;
  std::set<std::string> nodesInProgress;  // stays empty between calls: the goroutines end before SchedulePodEviction returns
  int evictions = 0;
  void updateNodeToDrainOrFailed(Node node, bool drainEnabled) {
    (void)provider->ChangeNodeUpgradeState(&node, drainEnabled ? UpgradeStateDrainRequired : UpgradeStateFailed);
  }
  Error SchedulePodEviction(const PodManagerConfig& config) override {
    evictions++;
    if (config.Nodes.empty()) return std::nullopt;
    if (config.DeletionSpec == nullptr) return Errorf("pod deletion spec should not be empty");
    DrainHelper helper;
    helper.client = store; helper.evictor = evictor;
    helper.Force = config.DeletionSpec->Force; helper.DeleteEmptyDirData = config.DeletionSpec->DeleteEmptyDir;
    helper.TimeoutSecond = config.DeletionSpec->TimeoutSecond;
    helper.additional = podDeletionFilter;
    for (Node* n : config.Nodes) {
      if (nodesInProgress.count(n->Name)) continue;
      Node node = *n;  // go func(node corev1.Node)
      std::vector<Pod*> podList;
      if (store->ListPodsBySelector("", node.Name, &podList)) continue;  // logged, dropped
      int numPodsToDelete = 0;
      for (const Pod* p : podList) numPodsToDelete += podDeletionFilter(*p) ? 1 : 0;
      if (numPodsToDelete == 0) {
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
        continue;
      }
      std::vector<Pod*> podDeleteList;
      helper.GetPodsForDeletion(node.Name, &podDeleteList);
      if ((int)podDeleteList.size() != numPodsToDelete) {
        updateNodeToDrainOrFailed(node, config.DrainEnabled);
        continue;
      }
      if (helper.DeleteOrEvictPods(node, podDeleteList)) {
        updateNodeToDrainOrFailed(node, config.DrainEnabled);
        continue;
      }
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
    }
    return std::nullopt;
  }
};

// drain_manager.go:58-139; the cordon is RunCordonOrUncordon, the CordonManager's call (cordon_manager.go:40-47)
struct DrainManagerImpl : DrainManager {
  Store* store = nullptr;
  PodEvictor* evictor = nullptr;
  CordonManager* cordon = nullptr;
  NodeUpgradeStateProvider* provider = nullptr;
  std::set<std::string> drainingNodes;
  int calls = 0;
  Error ScheduleNodesDrain(const DrainConfiguration& c) override {
    calls++;
    if (c.Nodes.empty()) return std::nullopt;
    if (c.Spec == nullptr) return Errorf("drain spec should not be empty");
    if (!c.Spec->Enable) return std::nullopt;
    DrainHelper helper;
    helper.client = store; helper.evictor = evictor;
    helper.Force = c.Spec->Force; helper.DeleteEmptyDirData = c.Spec->DeleteEmptyDir; helper.TimeoutSecond = c.Spec->TimeoutSecond;
    helper.PodSelector = c.Spec->PodSelector;
    for (Node* n : c.Nodes) {
      if (drainingNodes.count(n->Name)) continue;
      Node node = *n;  // the mirror hands its worker a copy; the log and the store see the same node name
      if (cordon->Cordon(&node)) {
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
        continue;
      }
      std::vector<Pod*> pods;
      if (helper.GetPodsForDeletion(node.Name, &pods) || helper.DeleteOrEvictPods(node, pods)) {  // RunNodeDrain
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
        continue;
      }
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
    }
    return std::nullopt;
  }
};

// A cordon that records its calls (under `mu`, when set) and fails for one node.
struct FailingCordon : CordonManager {
  std::vector<std::string>* log = nullptr;
  std::mutex* mu = nullptr;
  std::string failNode;
  Error Cordon(Node* n) override {
    std::unique_lock<std::mutex> l;
    if (mu) l = std::unique_lock<std::mutex>(*mu);
    const bool fail = n->Name == failNode;
    log->push_back((fail ? "FAILED cordon " : "cordon ") + n->Name);
    return fail ? Errorf("cordon failed") : std::nullopt;
  }
  Error Uncordon(Node* n) override {
    std::unique_lock<std::mutex> l;
    if (mu) l = std::unique_lock<std::mutex>(*mu);
    log->push_back("uncordon " + n->Name);
    return std::nullopt;
  }
};

// The logging PodManager and DrainManager, locked: their log is the one the mirror's workers write to.
struct LockedPods : wspec::CountingPods {
  std::mutex* mu = nullptr;
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& c) override { std::lock_guard<std::mutex> l(*mu); return CountingPods::ScheduleCheckOnPodCompletion(c); }
  Error SchedulePodEviction(const PodManagerConfig& c) override { std::lock_guard<std::mutex> l(*mu); return CountingPods::SchedulePodEviction(c); }
  Error SchedulePodsRestart(const std::vector<Pod*>& pods) override { std::lock_guard<std::mutex> l(*mu); return CountingPods::SchedulePodsRestart(pods); }
};
struct LockedDrain : spec::LogDrain {
  std::mutex* mu = nullptr;
  Error ScheduleNodesDrain(const DrainConfiguration& c) override { std::lock_guard<std::mutex> l(*mu); return spec::LogDrain::ScheduleNodesDrain(c); }
};

// The API-server provider of wait_spec.hpp, callable from the mirror's workers.
struct LockedProvider : wspec::ApiProvider {
  std::mutex mu;
  Error GetNode(const std::string& name, Node** out) override { std::lock_guard<std::mutex> l(mu); return ApiProvider::GetNode(name, out); }
  Error ChangeNodeUpgradeState(Node* n, const std::string& s) override { std::lock_guard<std::mutex> l(mu); return ApiProvider::ChangeNodeUpgradeState(n, s); }
  Error ChangeNodeUpgradeAnnotation(Node* n, const std::string& k, const std::string& v) override {
    std::lock_guard<std::mutex> l(mu);
    return ApiProvider::ChangeNodeUpgradeAnnotation(n, k, v);
  }
};

// A log split by node (the text after the verb's first space up to the next space or '='), each node's calls in order:
// the workers of different nodes run concurrently, as the reference's goroutines do.
inline std::map<std::string, std::vector<std::string>> perNode(const std::vector<std::string>& log) {
  std::map<std::string, std::vector<std::string>> out;
  for (const std::string& s : log) {
    std::string t = s.rfind("FAILED ", 0) == 0 ? s.substr(7) : s;
    const size_t a = t.find(' ');
    const size_t b = a == std::string::npos ? a : t.find_first_of(" =", a + 1);
    const std::string verb = t.substr(0, a);
    const std::string who = (verb == "restart" || verb == "drain" || verb == "wait" || a == std::string::npos) ? "*" : t.substr(a + 1, b - a - 1);
    out[who].push_back(s);
  }
  return out;
}

// The calls the option replaces, as the logging PodManager and DrainManager record them: "evict <n>" and "drain ...".
inline int managerCalls(const std::vector<std::string>& log) {
  int n = 0;
  for (const std::string& s : log) n += s.rfind("drain", 0) == 0 || (s.rfind("evict ", 0) == 0 && s.size() > 6 && s[6] >= '0' && s[6] <= '9');
  return n;
}

inline Pod makeWorkloadPod(const std::string& name, const std::string& node, const std::string& phase, int64_t rv) {
  Pod p;
  p.Name = name;
  p.Namespace = "apps";
  p.NodeName = node;
  p.ResourceVersion = std::to_string(rv);
  p.Phase = phase;
  return p;
}

}  // namespace espec
