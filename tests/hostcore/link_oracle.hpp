// link_oracle.hpp — TEST INFRASTRUCTURE: the oracle's Simulator (oracle/lbft_oracle.hpp) with link latencies, the reference of one
// parameter set of a links sweep (lbft_create_sweep_links).  The oracle itself stays the restatement of the reference, which has
// no link latencies; this derives from it and restates the three members a network send passes through — loop_until,
// process_node_actions and schedule_network_event, each as the oracle has it — with one change: schedule_network_event adds
// links[sender * num_nodes + receiver] to the event's time right after its delay is drawn, before the partition test.  (They are
// not virtual: LinkSimulator::loop_until calls the restated ones.)  The constructor's startup delays and the timers get no term.
// An empty matrix gives the oracle's run; tests/test_link_sweep.py pins that, and the term, on a trace of every network event.
#pragma once
#include <functional>
#include <vector>

#include "../../oracle/lbft_oracle.hpp"

namespace lbft_oracle {

struct LinkSimulator : Simulator {
  std::vector<uint32_t> links;  // [num_nodes * num_nodes], or empty: none
  // Called for every network event at its scheduling, partitioned or not: (kind, receiver, sender, send clock, due time).
  std::function<void(int, Author, Author, int64_t, int64_t)> on_network_event;

  LinkSimulator(uint64_t seed, const SimConfig& c, std::vector<uint32_t> m) : Simulator(seed, c), links(std::move(m)) {}

  void schedule_network_event(int kind, Author receiver, Author sender, int payload) {  // Simulator::schedule_network_event
    int64_t t = clock + cfg.delay.sample(rng);
    if (!links.empty()) t += links[(size_t)sender * cfg.num_nodes + receiver];
    if (on_network_event) on_network_event(kind, receiver, sender, clock, t);
    if (!cfg.partitions.empty() && partitioned(receiver, sender)) {
      event_count++;
      counters.dropped_partition++;
      return;
    }
    push_event(t, kind, receiver, sender, payload);
  }

  void process_node_actions(int64_t clk, Author author, const NodeUpdateActions& actions) {  // Simulator::process_node_actions
    SimulatedNode& node = nodes[author];
    int64_t from_node =
        actions.next_scheduled_update == NODE_TIME_NEVER ? INT64_MAX : from_node_time(actions.next_scheduled_update, node.startup_time);
    int64_t new_scheduled_time = std::max(from_node, clk + 1);
    node.ignore_scheduled_updates_until = new_scheduled_time - 1;
    push_event(new_scheduled_time, EV_TIMER, author, author, -1);
    std::vector<Author> receivers;
    if (actions.should_broadcast) {
      for (uint32_t i = 0; i < cfg.num_nodes; i++)
        if ((Author)i != author) receivers.push_back((Author)i);
    } else {
      for (Author r : actions.should_send)
        if (r != author) receivers.push_back(r);
    }
    shuffle(receivers, rng);
    if (!receivers.empty()) {
      int p = (int)notif_pool.size();
      notif_pool.push_back(node.node.create_notification(node.context));
      counters.scheduled_notify += receivers.size();
      for (Author r : receivers) schedule_network_event(EV_NOTIFY, r, author, p);
    }
    std::vector<Author> senders;
    if (actions.should_query_all) {
      for (uint32_t i = 0; i < cfg.num_nodes; i++)
        if ((Author)i != author) senders.push_back((Author)i);
    }
    shuffle(senders, rng);
    if (!senders.empty()) {
      int p = (int)req_pool.size();
      req_pool.push_back(node.node.create_request());
      for (Author s : senders) schedule_network_event(EV_REQUEST, author, s, p);
    }
  }

  void loop_until(int64_t max_clock) {  // Simulator::loop_until (single-epoch runs of the sweeps: no DataWriter)
    while (!pending_events.empty()) {
      Event ev = pending_events.top();
      pending_events.pop();
      if (ev.time > max_clock) break;
      int64_t clk = std::max(ev.time, clock);
      clock = clk;
      counters.processed[ev.kind]++;
      if (is_silent(ev.receiver) || (ev.kind == EV_REQUEST && is_silent(ev.sender))) continue;
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
