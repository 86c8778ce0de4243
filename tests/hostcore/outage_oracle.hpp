// outage_oracle.hpp — TEST INFRASTRUCTURE: the link oracle (link_oracle.hpp, the oracle's Simulator with link latencies) with one
// outage window per node, the reference of one parameter set of an outage sweep (lbft_create_sweep_outages).  The oracle itself
// stays the restatement of the reference, which has no timed outages; this derives from LinkSimulator and restates loop_until
// only, as LinkSimulator has it, with one change: the silent test after the pop (after the max_clock test and the clock update)
// reads "silent, or down at the pop clock".  A node keeps its whole state across its window and nothing is scheduled at
// recovery, so a window only filters which pops are handled.  No window gives LinkSimulator's run; [0, > max_clock) gives the
// oracle's run with that node silent.  tests/test_outage_sweep.py pins both on a trace of every pop.
#pragma once
#include <functional>
#include <utility>
#include <vector>

#include "link_oracle.hpp"

namespace lbft_oracle {

// Why a pop was not handled, or that it was: the pop-trace codes (OutageSimulator::on_pop).
enum PopFate {
  POP_HANDLED = 0,          // handled by its node
  POP_CANCELLED = 1,        // a timer cancelled by ignore_scheduled_updates_until
  POP_RECEIVER_SILENT = 2,  // dropped: its receiver is silent
  POP_RECEIVER_DOWN = 3,    // dropped: its receiver is down
  POP_SENDER_SILENT = 4,    // dropped: a request whose sender (the node it was sent to) is silent
  POP_SENDER_DOWN = 5,      // dropped: a request whose sender is down
};

struct OutageSimulator : LinkSimulator {
  std::vector<std::pair<int64_t, int64_t>> windows;  // [num_nodes] {down_from, down_until}, or empty: none
  // Called for every pop up to max_clock: (kind, receiver, sender, pop clock, PopFate).
  std::function<void(int, Author, Author, int64_t, int)> on_pop;

  OutageSimulator(uint64_t seed, const SimConfig& c, std::vector<uint32_t> m, std::vector<std::pair<int64_t, int64_t>> w)
      : LinkSimulator(seed, c, std::move(m)), windows(std::move(w)) {}

  bool is_down(Author a, int64_t clk) const {
    return !windows.empty() && windows[a].first <= clk && clk < windows[a].second;
  }

  void loop_until(int64_t max_clock) {  // LinkSimulator::loop_until with the outage test
    while (!pending_events.empty()) {
      Event ev = pending_events.top();
      pending_events.pop();
      if (ev.time > max_clock) break;
      int64_t clk = std::max(ev.time, clock);
      clock = clk;
      counters.processed[ev.kind]++;
      int fate = POP_HANDLED;
      if (is_silent(ev.receiver)) fate = POP_RECEIVER_SILENT;
      else if (is_down(ev.receiver, clk)) fate = POP_RECEIVER_DOWN;
      else if (ev.kind == EV_REQUEST && is_silent(ev.sender)) fate = POP_SENDER_SILENT;
      else if (ev.kind == EV_REQUEST && is_down(ev.sender, clk)) fate = POP_SENDER_DOWN;
      if (fate == POP_HANDLED && ev.kind == EV_TIMER && clk <= nodes[ev.receiver].ignore_scheduled_updates_until)
        fate = POP_CANCELLED;
      if (on_pop) on_pop(ev.kind, ev.receiver, ev.sender, clk, fate);
      if (fate != POP_HANDLED && fate != POP_CANCELLED) continue;
      switch (ev.kind) {
        case EV_TIMER: {
          SimulatedNode& node = nodes[ev.receiver];
          if (clk <= node.ignore_scheduled_updates_until) {
            counters.timers_cancelled++;
            continue;
          }
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
        case EV_NOTIFY: {
          SimulatedNode& node = nodes[ev.receiver];
          std::optional<DataSyncRequest> result = node.node.handle_notification(node.context, notif_pool[ev.payload]);
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          if (result) {
            int p = (int)req_pool.size();
            req_pool.push_back(*result);
            schedule_network_event(EV_REQUEST, ev.receiver, ev.sender, p);
          }
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
        case EV_REQUEST: {
          SimulatedNode& node = nodes[cfg.true_data_sync ? ev.sender : ev.receiver];
          int p = (int)resp_pool.size();
          resp_pool.push_back(node.node.handle_request(req_pool[ev.payload]));
          schedule_network_event(EV_RESPONSE, ev.receiver, ev.sender, p);
          break;
        }
        case EV_RESPONSE: {
          SimulatedNode& node = nodes[ev.receiver];
          node.node.handle_response(node.context, resp_pool[ev.payload], to_node_time(clk, node.startup_time));
          if (payload_free) resp_pool[ev.payload] = DataSyncResponse();
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
      }
    }
  }
};

}  // namespace lbft_oracle
