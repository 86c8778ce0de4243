/* multi_handle.c — ONE host thread keeps several handles busy through lbft_run_async / lbft_wait (include/lbft.h): the way a
 * single-threaded C or Rust caller drives every GPU of a box (bft-lib-gpu: GpuSimulator::on_devices).  Handle h lives on
 * device h % (number of devices); on a one-GPU box the eight handles share device 0.  Each handle runs two batches:
 * while batch 1 is in flight the results of batch 0 must stay readable and the seeds of batch 1 are staged with
 * lbft_set_seeds.  Everything is compared with synchronous lbft_run on a ninth handle, and the bulk commit-log
 * export (lbft_commit_logs) with lbft_commit_log.  Then one batch of BIG instances per device (at least two handles), which
 * selects the thread-per-instance kernel with its shared-memory queues (a per-device opt-in beyond 48 KB of shared
 * memory per block), run concurrently; every handle must agree with the first.  Built and run by tests/test_gpu_cabi_c.py. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "lbft.h"

#define H 8
#define I 96
#define N 4
#define CAP 64
#define BIG 65536
#define MAXB 16

static void config(lbft_config* c, const uint64_t* seeds, uint32_t count, int device) {
  memset(c, 0, sizeof *c);
  c->struct_size = sizeof *c;
  c->num_instances = count;
  c->num_nodes = N;
  c->seeds = seeds;
  c->max_clock = 1000;
  c->delay_mean = 10.0;
  c->delay_variance = 4.0;
  c->target_commit_interval = 100000;
  c->delta = 20;
  c->gamma = 2.0;
  c->lambda = 0.5;
  c->commands_per_epoch = 30000;
  c->device = device;
}
#define CHECK(x)                                                                     \
  do {                                                                               \
    if ((x) != LBFT_OK) { fprintf(stderr, "%s: %s\n", #x, lbft_last_error()); return 1; } \
  } while (0)

int main(void) {
  static uint64_t seeds[H][2][I];
  static uint64_t states[H][2][I * N], want[I * N];
  static uint32_t counts[I * N], lens[I * N];
  static lbft_commit rows[I * CAP], one[CAP];
  lbft_sim* sim[H];
  lbft_sim* ref = NULL;
  int ndev = 1;
  const char* e = getenv("LBFT_TEST_DEVICES");
  if (e) ndev = atoi(e) > 0 ? atoi(e) : 1;
  for (int h = 0; h < H; h++)
    for (int b = 0; b < 2; b++)
      for (int i = 0; i < I; i++) seeds[h][b][i] = 1000u * (unsigned)h + 100000u * (unsigned)b + (unsigned)i + 7u;
  lbft_config c;
  for (int h = 0; h < H; h++) {
    config(&c, seeds[h][0], I, h % ndev);
    CHECK(lbft_create(&c, &sim[h]));
  }
  /* batch 0 on every handle at once */
  for (int h = 0; h < H; h++) CHECK(lbft_run_async(sim[h]));
  for (int h = 0; h < H; h++) {
    uint32_t tmp[I];
    if (lbft_status(sim[h], tmp) != LBFT_ERR_STATE && h == H - 1) { /* no results before the first wait */
      fprintf(stderr, "results readable before lbft_wait\n");
      return 1;
    }
  }
  for (int h = 0; h < H; h++) CHECK(lbft_wait(sim[h]));
  /* batch 1: stage the seeds and launch, THEN read batch 0's results while batch 1 runs */
  for (int h = 0; h < H; h++) {
    CHECK(lbft_set_seeds(sim[h], seeds[h][1]));
    CHECK(lbft_run_async(sim[h]));
  }
  for (int h = 0; h < H; h++) CHECK(lbft_last_states(sim[h], states[h][0]));
  if (lbft_run(sim[0]) != LBFT_ERR_STATE) { fprintf(stderr, "lbft_run accepted while a run is in flight\n"); return 1; }
  for (int h = 0; h < H; h++) CHECK(lbft_wait(sim[h]));
  for (int h = 0; h < H; h++) CHECK(lbft_last_states(sim[h], states[h][1]));
  /* the same batches, synchronously, on one more handle */
  config(&c, seeds[0][0], I, 0);
  CHECK(lbft_create(&c, &ref));
  int bad = 0;
  for (int h = 0; h < H; h++)
    for (int b = 0; b < 2; b++) {
      CHECK(lbft_set_seeds(ref, seeds[h][b]));
      CHECK(lbft_run(ref));
      CHECK(lbft_last_states(ref, want));
      if (memcmp(want, states[h][b], sizeof want)) { fprintf(stderr, "handle %d batch %d differs from the synchronous run\n", h, b); bad = 1; }
    }
  /* bulk commit logs of the last synchronous run against the per-node reader */
  CHECK(lbft_commit_counts(ref, counts));
  CHECK(lbft_commit_logs(ref, rows, CAP, lens));
  if (memcmp(counts, lens, sizeof counts)) { fprintf(stderr, "lens differ from lbft_commit_counts\n"); bad = 1; }
  size_t total = 0;
  for (uint32_t i = 0; i < I; i++)
    for (uint32_t n = 0; n < N; n++) {
      size_t len = 0;
      CHECK(lbft_commit_log(ref, i, n, one, CAP, &len));
      if (len != lens[i * N + n] || memcmp(one, rows + (size_t)i * CAP, len * sizeof(lbft_commit))) {
        fprintf(stderr, "instance %u node %u: bulk log differs\n", i, n);
        bad = 1;
      }
      total += len;
    }
  printf("%d handles x 2 batches on %d device(s) from one thread; %zu commit-log rows checked\n", H, ndev, total);
  for (int h = 0; h < H; h++) lbft_destroy(sim[h]);
  lbft_destroy(ref);
  /* BIG instances per handle, one handle per device (two on a one-GPU box), launched together */
  static uint64_t big_seeds[BIG], big_states[MAXB][BIG * N];
  lbft_sim* big[MAXB];
  const int nb = ndev < 2 ? 2 : (ndev > MAXB ? MAXB : ndev);
  for (int i = 0; i < BIG; i++) big_seeds[i] = (uint64_t)i;
  char kernel[128];
  for (int b = 0; b < nb; b++) {
    config(&c, big_seeds, BIG, b % ndev);
    CHECK(lbft_create(&c, &big[b]));
  }
  CHECK(lbft_kernel_info(big[0], kernel, sizeof kernel));
  for (int b = 0; b < nb; b++) CHECK(lbft_run_async(big[b]));
  for (int b = 0; b < nb; b++) CHECK(lbft_wait(big[b]));
  for (int b = 0; b < nb; b++) {
    CHECK(lbft_last_states(big[b], big_states[b]));
    if (memcmp(big_states[b], big_states[0], sizeof big_states[0])) { fprintf(stderr, "big handle %d differs from handle 0\n", b); bad = 1; }
    lbft_destroy(big[b]);
  }
  printf("%d handles of %d instances (%s) on %d device(s)\n", nb, BIG, kernel, ndev);
  puts(bad ? "MISMATCH" : "async handles agree with synchronous runs");
  return bad;
}
