// The events of the managers the three on-device options replace, restated: ValidationManagerImpl.Validate
// (validation_manager.go:97-101), PodManagerImpl.ScheduleCheckOnPodCompletion (pod_manager.go:290-306), SchedulePodEviction
// (:210-222, :393-403) and DrainManagerImpl.ScheduleNodesDrain (drain_manager.go:104-131), over the restatements of
// validation_spec.hpp, wait_spec.hpp and eviction_spec.hpp. Each one records through an optional EventRecorder (nullptr:
// none, and the calls are those of the restatement it extends). The drain's error text comes from this file's own
// evaluation of kubectl's filter chain, with its messages.
#pragma once
#include <atomic>
#include <mutex>

#include "eviction_spec.hpp"

namespace evspec {
using namespace upgrade;
using namespace mocks;

// A recorder that writes "event <node> <type> <reason>: <message>" into a call log (under `mu`, when set), so that
// espec::perNode files each event among its node's calls.
struct LogRecorder : EventRecorder {
  std::vector<std::string>* log = nullptr;
  std::mutex* mu = nullptr;
  std::atomic<int> events{0};
  void Event(const Node& n, const std::string& type, const std::string& reason, const std::string& message) override {
    std::unique_lock<std::mutex> l;
    if (mu) l = std::unique_lock<std::mutex>(*mu);
    events++;
    log->push_back("event " + n.Name + " " + type + " " + reason + ": " + message);
  }
};
// util.go:162-176
inline void logEvent(EventRecorder* r, const Node& n, const char* type, const std::string& message) {
  if (r) r->Event(n, type, GetEventReason(), message);
}

// validation_manager.go:71-116
struct ValidationManagerImpl : vspec::ValidationManagerImpl {
  EventRecorder* recorder = nullptr;
  Error Validate(Node* node, bool* done) override {
    calls++;
    *done = false;
    if (podSelector.empty()) { *done = true; return std::nullopt; }
    std::vector<Pod*> pods;
    if (Error e = client->ListPodsBySelector(podSelector, node->Name, &pods)) return e;
    if (pods.empty()) return std::nullopt;
    bool ok = true;
    for (Pod* p : pods) {
      if (!isPodReady(*p)) {
        if (Error e = handleTimeout(node, 600)) {
          // logEventf(..., "Failed to handle timeout for validation state", err.Error()): a format without a verb
          logEvent(recorder, *node, EventTypeWarning, "Failed to handle timeout for validation state%!(EXTRA string=" + *e + ")");
          return Errorf("unable to handle timeout for validation state: " + *e);
        }
        ok = false;
        break;
      }
      if (Error e = provider->ChangeNodeUpgradeAnnotation(node, GetValidationStartTimeAnnotationKey(), "null")) { *done = ok; return e; }
    }
    *done = ok;
    return std::nullopt;
  }
};

// kubectl drain.Helper.GetPodsForDeletion with the filters' messages (k8s.io/kubectl pkg/drain/filters.go, drain.go) and
// RunNodeDrain's utilerrors.NewAggregate: "cannot delete <message>: <ns/name, ...>" per message, messages in the order of
// their first pod, "[a, b]" for more than one.
struct DrainHelper : espec::DrainHelper {
  // the chain of espec::DrainHelper::filter, and the message of a Fail
  Status filter(const Pod& pod, std::string* message) const {
    if (const OwnerReference* c = GetControllerOf(pod))
      if (c->Kind == "DaemonSet" && !finished(pod)) {
        if (!client->getDaemonSet(pod.Namespace, c->Name)) {
          if (!Force) { *message = "daemonsets.apps \"" + c->Name + "\" not found"; return Fail; }
        } else {
          return Skip;
        }
      }
    if (pod.Annotations.count("kubernetes.io/config.mirror")) return Skip;
    if (pod.HasEmptyDirVolume && !finished(pod) && !DeleteEmptyDirData) {
      *message = "Pods with local storage (use --delete-emptydir-data to override)";
      return Fail;
    }
    if (!finished(pod) && GetControllerOf(pod) == nullptr && !Force) {
      *message = "Pods declare no controller (use --force to override)";
      return Fail;
    }
    if (additional && !additional(pod)) return Skip;
    return Okay;
  }
  Error GetPodsForDeletion(const std::string& node, std::vector<Pod*>* pods) const {
    std::vector<Pod*> listed;
    if (Error e = client->ListPodsBySelector(PodSelector, node, &listed)) return e;
    std::vector<std::pair<std::string, std::string>> failed;
    for (Pod* p : listed) {
      std::string msg;
      const Status s = filter(*p, &msg);
      if (s == Okay) pods->push_back(p);
      if (s != Fail) continue;
      size_t k = 0;
      while (k < failed.size() && failed[k].first != msg) k++;
      if (k == failed.size()) failed.push_back({msg, ""});
      else failed[k].second += ", ";
      failed[k].second += p->Namespace + "/" + p->Name;
    }
    if (failed.empty()) return std::nullopt;
    std::string s;
    for (size_t k = 0; k < failed.size(); k++) s += (k ? ", " : "") + ("cannot delete " + failed[k].first + ": " + failed[k].second);
    return Errorf(failed.size() == 1 ? s : "[" + s + "]");
  }
};

// pod_manager.go:122-317, :393-403
struct PodManagerImpl : espec::PodManagerImpl {
  EventRecorder* recorder = nullptr;
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& config) override {  // :256-317
    checks++;
    for (Node* n : config.Nodes) {
      std::vector<Pod*> podList;
      if (Error err = ListPods(config.WaitForCompletionSpec->PodSelector, n->Name, &podList)) return err;
      Node node = *n;
      bool running = false;
      for (const Pod* pod : podList) {
        running = IsPodRunningOrPending(*pod);
        if (running) break;
      }
      if (running) {
        if (config.WaitForCompletionSpec->TimeoutSecond != 0)
          if (Error err = HandleTimeoutOnPodCompletions(&node, (int64_t)config.WaitForCompletionSpec->TimeoutSecond))
            logEvent(recorder, node, EventTypeWarning, "Failed to handle timeout for job completions, " + *err);  // :290-296
        continue;
      }
      if (Error err = provider->ChangeNodeUpgradeAnnotation(&node, GetWaitForPodCompletionStartTimeAnnotationKey(), "null")) {
        logEvent(recorder, node, EventTypeWarning, "Failed to remove annotation used to track job completions: " + *err);  // :301-306
        continue;
      }
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);
    }
    return std::nullopt;
  }
  void updateNodeToDrainOrFailed(Node node, bool drainEnabled) {  // :393-403
    if (drainEnabled)
      logEvent(recorder, node, EventTypeWarning, "Pod deletion failed but drain is enabled in spec. Will attempt a node drain");
    (void)provider->ChangeNodeUpgradeState(&node, drainEnabled ? UpgradeStateDrainRequired : UpgradeStateFailed);
  }
  Error SchedulePodEviction(const PodManagerConfig& config) override {  // :122-229
    evictions++;
    if (config.Nodes.empty()) return std::nullopt;
    if (config.DeletionSpec == nullptr) return Errorf("pod deletion spec should not be empty");
    espec::DrainHelper helper;
    helper.client = store; helper.evictor = evictor;
    helper.Force = config.DeletionSpec->Force; helper.DeleteEmptyDirData = config.DeletionSpec->DeleteEmptyDir;
    helper.TimeoutSecond = config.DeletionSpec->TimeoutSecond;
    helper.additional = podDeletionFilter;
    for (Node* n : config.Nodes) {
      if (nodesInProgress.count(n->Name)) continue;
      Node node = *n;
      std::vector<Pod*> podList;
      if (store->ListPodsBySelector("", node.Name, &podList)) continue;
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
      if (Error err = helper.DeleteOrEvictPods(node, podDeleteList)) {
        logEvent(recorder, node, EventTypeWarning, "Failed to delete workload pods on the node for the driver upgrade, " + *err);
        updateNodeToDrainOrFailed(node, config.DrainEnabled);
        continue;
      }
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
      logEvent(recorder, node, EventTypeNormal, "Deleted workload pods on the node for the driver upgrade");
    }
    return std::nullopt;
  }
};

// drain_manager.go:58-139
struct DrainManagerImpl : espec::DrainManagerImpl {
  EventRecorder* recorder = nullptr;
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
      logEvent(recorder, *n, EventTypeNormal, "Scheduling drain of the node");
      Node node = *n;
      if (Error err = cordon->Cordon(&node)) {
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
        logEvent(recorder, node, EventTypeWarning, "Failed to cordon the node, " + *err);
        continue;
      }
      std::vector<Pod*> pods;
      Error err = helper.GetPodsForDeletion(node.Name, &pods);  // RunNodeDrain
      if (!err) err = helper.DeleteOrEvictPods(node, pods);
      if (err) {
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
        logEvent(recorder, node, EventTypeWarning, "Failed to drain the node, " + *err);
        continue;
      }
      logEvent(recorder, node, EventTypeNormal, "Successfully drained the node");
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
    }
    return std::nullopt;
  }
};

// The rows of the events table (INTEGRATION.md, "Events"): the message each row's events start with.
inline const std::vector<std::string>& rows() {
  static const std::vector<std::string> r = {
      "Warning Failed to handle timeout for validation state%!(EXTRA string=",
      "Warning Failed to handle timeout for job completions, ",
      "Warning Failed to remove annotation used to track job completions: ",
      "Warning Failed to delete workload pods on the node for the driver upgrade, ",
      "Normal Deleted workload pods on the node for the driver upgrade",
      "Warning Pod deletion failed but drain is enabled in spec. Will attempt a node drain",
      "Normal Scheduling drain of the node",
      "Warning Failed to cordon the node, ",
      "Warning Failed to drain the node, ",
      "Normal Successfully drained the node"};
  return r;
}
// The row of a LogRecorder line, -1 for anything else.
inline int rowOf(const std::string& line) {
  if (line.rfind("event ", 0) != 0) return -1;
  const size_t a = line.find(' ', 6);  // after the node
  const size_t b = line.find(' ', a + 1);  // after the type
  const size_t c = line.find(": ", b + 1);  // after the reason
  if (a == std::string::npos || b == std::string::npos || c == std::string::npos) return -1;
  const std::string key = line.substr(a + 1, b - a) + line.substr(c + 2);
  for (size_t i = 0; i < rows().size(); i++)
    if (key.rfind(rows()[i], 0) == 0) return (int)i;
  return -1;
}

}  // namespace evspec
