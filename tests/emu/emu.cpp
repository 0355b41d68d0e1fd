// tests/emu/emu.cpp -- TEST INFRASTRUCTURE: cooperative scheduler of the host SIMT emulator (see shim/cuda_runtime.h).
#include <cuda_runtime.h>

namespace emu {
Cta* g_cta = nullptr;
unsigned long long g_events = 0;
static const size_t kStack = 512 * 1024;

static void retire(Cta& c, Thread& t) {
  t.done = true;
  Warp& w = c.warp[t.tid >> 5];
  w.alive--;
  c.cta_alive--;
  if (w.alive > 0 && w.arrived >= w.alive) { w.arrived = 0; w.gen++; }
  if (c.cta_alive > 0 && c.cta_arrived >= c.cta_alive) { c.cta_arrived = 0; c.cta_gen++; }
  g_events++;
}

static void trampoline() {
  Cta& c = *g_cta;
  c.body();
  Thread& t = c.th[c.cur];
  retire(c, t);
  swapcontext(&t.ctx, &c.sched);
  abort();
}

void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
  int nt = (int)block.x;
  Cta c;
  c.nthreads = nt;
  c.th.resize(nt);
  c.warp.resize((nt + 31) / 32);
  c.bdim = block; c.gdim = grid;
  c.smem = (char*)aligned_alloc(128, ((smem + 127) / 128 + 1) * 128);
  c.body = body;
  for (int i = 0; i < nt; i++) c.th[i].stack = (char*)malloc(kStack);
  Cta* prev = g_cta;
  g_cta = &c;
  for (unsigned b = 0; b < grid.x; b++) {
    c.bidx = dim3(b, 0, 0);
    memset(c.smem, 0xcd, smem);   // poison: reads of uninitialised shared memory show up as garbage, as on hardware
    c.cta_arrived = 0; c.cta_gen = 0; c.cta_alive = nt; c.or_acc[0] = c.or_acc[1] = 0;
    for (auto& w : c.warp) { w.arrived = 0; w.gen = 0; w.alive = 0; }
    for (int i = 0; i < nt; i++) {
      Thread& t = c.th[i];
      t.tid = i; t.done = false; t.wait_kind = 0; t.orcalls = 0;
      c.warp[i >> 5].alive++;
      getcontext(&t.ctx);
      t.ctx.uc_stack.ss_sp = t.stack; t.ctx.uc_stack.ss_size = kStack; t.ctx.uc_link = nullptr;
      makecontext(&t.ctx, trampoline, 0);
    }
    int ndone = 0;
    while (ndone < nt) {
      unsigned long long ev0 = g_events;
      bool any_runnable = false;
      ndone = 0;
      for (int i = 0; i < nt; i++) {
        Thread& t = c.th[i];
        if (t.done) { ndone++; continue; }
        if (t.wait_kind == 0) any_runnable = true;
        c.cur = i;
        swapcontext(&c.sched, &t.ctx);
        if (t.done) ndone++;
      }
      if (ndone < nt && g_events == ev0 && !any_runnable) {
        // a second look: waiting threads re-check their generation on resume, so one silent pass can be legitimate only
        // if someone was runnable; otherwise nobody can ever arrive
        bool all_wait = true;
        for (int i = 0; i < nt; i++) if (!c.th[i].done && c.th[i].wait_kind == 0) all_wait = false;
        if (all_wait) {
          fprintf(stderr, "emu: DEADLOCK in block %u (divergent warp collective or barrier)\n", b);
          for (int i = 0; i < nt; i++) if (!c.th[i].done) fprintf(stderr, "  tid %d waits at %s\n", i, c.th[i].wait_kind == 1 ? "warp rendezvous" : "cta barrier");
          abort();
        }
      }
    }
  }
  g_cta = prev;
  for (int i = 0; i < nt; i++) free(c.th[i].stack);
  free(c.smem);
}
}  // namespace emu
