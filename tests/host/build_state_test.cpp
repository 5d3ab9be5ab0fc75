// The incremental reconcile loop, BuildStateIncremental + ApplyStateIncremental (build_state_spec.hpp).
//   build_state_test         host halves only: the oracle stands behind BuildState's device call and behind both caches; the
//                            runs and overwrites the driver-pod cache hands down are checked and replayed on the oracle's copy
//                            of the previous reconcile's arrays, and its sparse owner indices are diffed against them
//   build_state_test --gpu   through the C ABI and the H100 kernels (ust_build_state_uids, ust_build_state_delta,
//                            ust_apply_state*, the ApplyState delta entry points)
#include <climits>
#include <cstring>

#include "build_state_spec.hpp"

extern "C" int ust_oracle_apply_state(int variant, const ust_policy* policy, int64_t n, const uint8_t* state,
                                      const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                                      const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                                      uint8_t* actuator_outcome, ust_counters* out);
extern "C" int ust_oracle_build_state_uids(int64_t n_pods, const uint8_t* state, const uint64_t* owner_uid, int32_t n_ds,
                                           const uint64_t* ds_uid, const int32_t* ds_desired, int32_t* ds_idx_out, ust_counters* out);

namespace {

// BuildState with the oracle behind its device call.
struct OracleBuild : upgrade::ClusterUpgradeStateManagerImpl {
  int BuildStateDevice(int64_t n, const uint8_t* state, const uint64_t* owner, int32_t n_ds, const uint64_t* ds_uid,
                       const int32_t* desired, int32_t* owner_idx, ust_counters* c) override {
    return ust_oracle_build_state_uids(n, state, owner, n_ds, ds_uid, desired, owner_idx, c);
  }
};

// Both caches with the oracle behind them. The driver-pod cache's hand-down is checked against the contract of
// ust_build_state_delta: its runs and overwrites, replayed on the previous reconcile's arrays, must give the cache's arrays,
// and the owner indices it carried over must be the previous ones; the sparse outputs (or, beyond the cache's capacity, all
// indices) are what the device would return.
struct CheckingOracle : upgrade::ClusterUpgradeStateManagerImpl {
  std::vector<uint8_t> state;
  std::vector<uint64_t> owner;
  std::vector<int32_t> prev;
  std::string problem;
  static inline int64_t reorders = 0, patched = 0, fetched = 0;

  int BuildStateCached(int32_t n_ds, const uint64_t* ds_uid, const int32_t* desired, PodCache* cache, ust_counters* c) override {
    PodCache& k = *cache;
    auto note = [&](const std::string& s) { if (problem.empty()) problem = s; };
    const size_t n = k.state.size(), nOld = state.size();
    std::vector<uint8_t> st;
    std::vector<uint64_t> ow;
    std::vector<int32_t> pv;
    if (k.reorder) {
      std::vector<char> named(nOld, 0);
      size_t ins = 0;
      if (k.run_src.size() != k.run_len.size()) note("run_src / run_len sizes differ");
      for (size_t r = 0; r < k.run_src.size() && problem.empty(); r++) {
        const int64_t s = k.run_src[r], l = k.run_len[r];
        if (l < 1 || s < -1) { note("run length below 1 or source below -1"); break; }
        if (r > 0 && ((s < 0 && k.run_src[r - 1] < 0) || (s >= 0 && k.run_src[r - 1] >= 0 && k.run_src[r - 1] + k.run_len[r - 1] == s)))
          note("runs are not maximal");
        for (int64_t e = 0; e < l && problem.empty(); e++) {
          if (s < 0) {
            if (ins >= k.insert_at.size()) { note("the inserted runs take more than the joined pods"); break; }
            const size_t i = (size_t)k.insert_at[ins++];
            if (i != st.size()) note("a joined pod is not where its run puts it");
            st.push_back(k.state[i]); ow.push_back(k.owner[2 * i]); ow.push_back(k.owner[2 * i + 1]); pv.push_back(INT32_MIN);
            continue;
          }
          const size_t q = (size_t)(s + e);
          if (q >= nOld || named[q]) { note("an old run leaves the previous list or names a pod twice"); break; }
          named[q] = 1;
          st.push_back(state[q]); ow.push_back(owner[2 * q]); ow.push_back(owner[2 * q + 1]); pv.push_back(prev[q]);
        }
      }
      if (ins != k.insert_at.size()) note("the inserted runs do not take every joined pod");
      reorders++;
    } else {
      st = state; ow = owner; pv = prev;
      if (!k.insert_at.empty()) note("joined pods without a reorder");
    }
    std::vector<char> seen(n, 0);
    for (int64_t i : k.changed) {
      if (i < 0 || (size_t)i >= st.size() || seen[(size_t)i]) { note("changed index outside the new list or named twice"); break; }
      seen[(size_t)i] = 1;
      st[(size_t)i] = k.state[(size_t)i]; ow[2 * i] = k.owner[2 * i]; ow[2 * i + 1] = k.owner[2 * i + 1];
    }
    if (!problem.empty()) return UST_ERR_INVALID_ARGUMENT;
    if (st != k.state || ow != k.owner) note("the replayed reorder + overwrites differ from the cache's arrays");
    if (pv != k.ownerIdx) note("the owner indices did not move with their pods");
    std::vector<int32_t> idx(n + 1);
    std::vector<uint8_t> s1 = k.state; s1.push_back(0);
    std::vector<uint64_t> o1 = k.owner; o1.push_back(0); o1.push_back(0);
    const int rc = ust_oracle_build_state_uids((int64_t)n, s1.data(), o1.data(), n_ds, ds_uid, desired, idx.data(), c);
    if (rc == UST_ERR_INVALID_ARGUMENT) return rc;
    idx.resize(n);
    size_t changed = 0;
    for (size_t i = 0; i < n; i++) changed += idx[i] != pv[i];
    if (changed > n / 4 + 1024) {  // what BuildStateCached does beyond its capacity: fetch every index
      k.ownerIdx = idx;
      fetched++;
    } else {
      for (size_t i = 0; i < n; i++)
        if (idx[i] != pv[i]) k.ownerIdx[i] = idx[i];
      patched++;
    }
    if (k.ownerIdx != idx) note("the patched owner indices differ from the oracle's");
    state = k.state; owner = k.owner; prev = idx;
    return rc;
  }

  int EvaluateCached(const ust_policy& policy, bool, const std::vector<int64_t>&, Cache* cache, ust_counters* c) override {
    Cache& k = *cache;
    const size_t n = k.slots.size();
    k.next.assign(n + 1, 0);
    k.actions.assign(n + 1, 0);
    std::vector<uint8_t> st = k.state; st.push_back(0);
    std::vector<uint32_t> fl = k.flags; fl.push_back(0);
    std::vector<int32_t> rv = k.pod_rev, di = k.ds_idx, dr = k.ds_rev;
    rv.push_back(0); di.push_back(0); dr.push_back(0);
    const int rc = ust_oracle_apply_state(0, &policy, (int64_t)n, st.data(), fl.data(), rv.data(), di.data(), (int32_t)k.ds_rev.size(),
                                          dr.data(), nullptr, k.next.data(), k.actions.data(), nullptr, c);
    k.next.resize(n);
    k.actions.resize(n);
    return rc;
  }
};

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  mocks::Runner R;
  bool device_ok = true;
  CheckingOracle* oracle = nullptr;
  spec::MakeBuildFn makeFull, makeIncr;
  spec::BuildFn buildFull = [](spec::BWorld& w, std::unique_ptr<upgrade::ClusterUpgradeState>* s) { return w.m->BuildState("gpu-operator", {}, s); };
  spec::BuildFn buildIncr = [](spec::BWorld& w, std::unique_ptr<upgrade::ClusterUpgradeState>* s) {
    return w.m->BuildStateIncremental("gpu-operator", {}, s);
  };
  spec::ApplyFn applyFull, applyIncr = [](spec::BWorld& w, upgrade::ClusterUpgradeState* s, const upgrade::DriverUpgradePolicySpec* p) {
    return w.m->ApplyStateIncremental(s, p);
  };
  std::function<std::string()> backendCheck = [] { return std::string(); };
  if (gpu) {
    makeFull = [&]() {
      std::unique_ptr<upgrade::ClusterUpgradeStateManagerImpl> m;
      if (auto e = upgrade::ClusterUpgradeStateManagerImpl::New(0, {}, &m)) {
        std::printf("cannot create manager: %s\n", e->c_str());
        device_ok = false;
        return upgrade::ClusterUpgradeStateManagerImpl::NewDetached({});
      }
      return m;
    };
    makeIncr = makeFull;
    applyFull = [](spec::BWorld& w, upgrade::ClusterUpgradeState* s, const upgrade::DriverUpgradePolicySpec* p) { return w.m->ApplyState(s, p); };
  } else {
    makeFull = [] { return std::unique_ptr<upgrade::ClusterUpgradeStateManagerImpl>(new OracleBuild()); };
    makeIncr = [&] {
      oracle = new CheckingOracle();
      return std::unique_ptr<upgrade::ClusterUpgradeStateManagerImpl>(oracle);
    };
    applyFull = [](spec::BWorld& w, upgrade::ClusterUpgradeState* s, const upgrade::DriverUpgradePolicySpec* p) -> upgrade::Error {
      upgrade::EncodedSnapshot enc;
      if (auto err = w.m->Encode(*s, *p, &enc)) return err;
      const size_t n = enc.entries.size();
      std::vector<uint8_t> next(n + 1);
      std::vector<uint16_t> actions(n + 1);
      enc.state.push_back(0); enc.flags.push_back(0); enc.pod_rev.push_back(0); enc.ds_idx.push_back(0); enc.ds_rev.push_back(0);
      ust_counters c;
      const int rc = ust_oracle_apply_state(0, &enc.policy, (int64_t)n, enc.state.data(), enc.flags.data(), enc.pod_rev.data(),
                                            enc.ds_idx.data(), (int32_t)enc.ds_rev.size() - 1, enc.ds_rev.data(), nullptr,
                                            next.data(), actions.data(), nullptr, &c);
      return w.m->Replay(enc, *p, next.data(), actions.data(), rc, c);
    };
    backendCheck = [&] { return oracle ? oracle->problem : std::string("no oracle-backed manager"); };
  }
  spec::run_build_state(R, makeFull, buildFull, applyFull, makeIncr, buildIncr, applyIncr, backendCheck, gpu ? 3000 : 300, 300);
  if (!gpu) {
    R.it("the oracle-backed evaluation saw the reorders and sparse patches it checked", [&] {
      std::printf("    %lld reorders, %lld sparse patches, %lld full fetches checked\n", (long long)CheckingOracle::reorders,
                  (long long)CheckingOracle::patched, (long long)CheckingOracle::fetched);
      EXPECT(R, CheckingOracle::reorders >= 150 && CheckingOracle::patched >= 150);
    });
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && device_ok) ? 0 : 1;
}
