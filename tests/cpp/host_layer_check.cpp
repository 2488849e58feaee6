// Compiles the C++ host layer (include/serfsim.hpp) against libserfsim.so and checks, without a GPU, that the boundary
// behaves as documented: the library loads, the ABI version matches, and creating a cluster fails loudly with
// SERFSIM_E_NO_DEVICE (there is no CPU execution path).  On an H100 it runs the configs[0] scenario instead.
#include <cstdio>
#include <cstring>

#include "serfsim.hpp"

int main() {
  using namespace serf;
  if (serfsim_abi_version() != SERFSIM_ABI_VERSION) { std::printf("abi mismatch\n"); return 2; }
  if (std::strcmp(as_str(MemberStatus::Leaving), "leaving") != 0) return 3;
  Options o;
  o.with_nodes(256).with_tracked_subjects(2).with_gossip_nodes(3).with_seed(7);
  try {
    Serf s(o);
    // GPU present: 256-node full mesh, node 0 leaves, node 1 re-announces its join
    std::vector<uint64_t> rp(257);
    std::vector<uint32_t> col;
    for (uint32_t v = 0; v < 256; ++v) { rp[v] = col.size(); for (uint32_t w = 0; w < 256; ++w) if (w != v) col.push_back(w); }
    rp[256] = col.size();
    s.set_topology(rp, col);
    s.track({0, 1});
    int leaves = 0;
    s.subscribe([&](uint32_t, MemberEventType ty, const std::vector<uint32_t>& ids) { if (ty == MemberEventType::Leave) leaves += (int)ids.size(); });
    s.leave(0); s.join(1);
    auto r = s.run_until_converged(500);
    auto m = s.members(0);
    int left = 0;
    for (auto st : m) left += st == MemberStatus::Left;
    std::printf("converged=%d ticks=%u left=%d leave_events=%d\n", (int)r.second, r.first, left, leaves);
    if (!(r.second && left == 255 && leaves == 1)) return 4;
    // Serf::user_event on a second cluster: two tracked events fired by nodes 7 and 9, every node delivers both
    Serf u(o);
    u.set_topology(rp, col);
    u.track({0, 1});
    u.track_user_events({11, 22});
    u.user_event(7, 0, 0);
    u.user_event(9, 1, 2);
    auto ru = u.run_until_converged(500);
    int seen0 = 0, seen1 = 0;
    for (auto b : u.user_event_seen(0)) seen0 += b;
    for (auto b : u.user_event_seen(1)) seen1 += b;
    const auto us = u.user_event_stats();
    std::printf("user events: converged=%d seen=%d/%d delivered=%llu event_time=%llu\n", (int)ru.second, seen0, seen1,
                (unsigned long long)us.delivered, (unsigned long long)us.event_time);
    return (ru.second && seen0 == 256 && seen1 == 256 && us.delivered == 512 && us.event_queue == 0) ? 0 : 6;
  } catch (const Error& e) {
    std::printf("%s\n", e.what());
    return e.code == SERFSIM_E_NO_DEVICE ? 10 : 5;
  }
}
