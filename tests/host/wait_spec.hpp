// StateOptions::WaitForCompletionOnDevice against the reference's PodManagerImpl.ScheduleCheckOnPodCompletion
// (pod_manager.go:256-391), restated here over the same mocks: one List per wait-for-jobs-required node through the
// client, a check per node on a copy of the node with every error dropped, and a return at the first failing List. The
// device-mode manager must make the same provider calls, in the same order, and return the same error.
#pragma once
#include <cstdio>

#include "validation_spec.hpp"

namespace wspec {
using namespace upgrade;
using namespace mocks;

// The failing, logging provider of validation_spec.hpp as an API server would be: a write names a node, and it lands on
// the cluster's node object of that name, whichever copy the caller holds (both sides hand the wait check's calls a copy
// of the node, as the reference does). `copies` counts the writes that came with a copy.
struct ApiProvider : vspec::FailingProvider {
  int copies = 0;
  Node* stored(Node* n) {
    auto it = nodes.find(n->Name);
    if (it == nodes.end() || it->second == n) return n;
    copies++;
    return it->second;
  }
  Error ChangeNodeUpgradeState(Node* n, const std::string& s) override { return FailingProvider::ChangeNodeUpgradeState(stored(n), s); }
  Error ChangeNodeUpgradeAnnotation(Node* n, const std::string& k, const std::string& v) override {
    return FailingProvider::ChangeNodeUpgradeAnnotation(stored(n), k, v);
  }
};

// The logging PodManager of build_state_spec.hpp that counts the checks it is asked for.
struct CountingPods : spec::LogPods {
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& c) override { waitCalls++; return spec::LogPods::ScheduleCheckOnPodCompletion(c); }
};

// pod_manager.go:256-391; eviction, restarts and revision hashes as spec::LogPods has them
struct PodManagerImpl : spec::LogPods {
  vspec::SelectorClient* client = nullptr;
  NodeUpgradeStateProvider* provider = nullptr;
  std::function<int64_t()> now;
  int checks = 0, lists = 0;
  // :371-391
  static bool IsPodRunningOrPending(const Pod& pod) { return pod.Phase == "Running" || pod.Phase == "Pending"; }
  // :320-329
  Error ListPods(const std::string& selector, const std::string& nodeName, std::vector<Pod*>* out) {
    lists++;
    return client->ListPodsBySelector(selector, nodeName, out);
  }
  // :331-368
  Error HandleTimeoutOnPodCompletions(Node* node, int64_t timeoutSeconds) {
    const std::string annotationKey = GetWaitForPodCompletionStartTimeAnnotationKey();
    const int64_t currentTime = now();
    if (!node->Annotations.count(annotationKey))  // :336-346
      return provider->ChangeNodeUpgradeAnnotation(node, annotationKey, std::to_string(currentTime));
    int64_t startTime = 0;
    if (Error err = vspec::ValidationManagerImpl::parseInt(node->Annotations[annotationKey], &startTime)) return err;  // :348-353
    if (currentTime > (int64_t)((uint64_t)startTime + (uint64_t)timeoutSeconds)) {  // :354, Go's wrapping int64 sum
      (void)provider->ChangeNodeUpgradeState(node, UpgradeStatePodDeletionRequired);  // :356
      if (Error err = provider->ChangeNodeUpgradeAnnotation(node, annotationKey, "null")) return err;  // :360-365
    }
    return std::nullopt;
  }
  // :256-317. The goroutines run one after the other here: each one only touches its own node.
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& config) override {
    checks++;
    for (Node* n : config.Nodes) {
      std::vector<Pod*> podList;
      if (Error err = ListPods(config.WaitForCompletionSpec->PodSelector, n->Name, &podList)) return err;  // :263-268
      Node node = *n;  // go func(node corev1.Node) (:275, :312)
      bool running = false;
      for (const Pod* pod : podList) {  // :279-284
        running = IsPodRunningOrPending(*pod);
        if (running) break;
      }
      if (running) {  // :287-299
        if (config.WaitForCompletionSpec->TimeoutSecond != 0)
          (void)HandleTimeoutOnPodCompletions(&node, (int64_t)config.WaitForCompletionSpec->TimeoutSecond);  // error: an event
        continue;
      }
      const std::string annotationKey = GetWaitForPodCompletionStartTimeAnnotationKey();  // :300-307
      if (provider->ChangeNodeUpgradeAnnotation(&node, annotationKey, "null")) continue;  // error: an event
      (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);    // :309
    }
    return std::nullopt;  // :315-316
  }
};

inline Pod makeWaitPod(const std::string& name, const std::string& node, const std::string& phase, int64_t rv) {
  Pod p;
  p.Name = name;
  p.Namespace = "jobs";
  p.NodeName = node;
  p.ResourceVersion = std::to_string(rv);
  p.Labels["app"] = "my-app";
  p.Phase = phase;
  return p;
}

}  // namespace wspec
