/* cuda_emu.cc -- fiber scheduler behind cuda_emu.h (TEST INFRASTRUCTURE ONLY). */
#define MZ_EMU 1
#include "cuda_emu.h"

#include <pthread.h>
#include <sys/mman.h>

#include <array>

emu_dim3 threadIdx, blockIdx, blockDim, gridDim;
uint8_t *emu_dyn_smem;

__asm__(
    ".text\n"
    ".globl emu_switch\n"
    ".type emu_switch,@function\n"
    "emu_switch:\n"
    "  pushq %rbp\n  pushq %rbx\n  pushq %r12\n  pushq %r13\n  pushq %r14\n  pushq %r15\n"
    "  movq %rsp, (%rdi)\n"
    "  movq %rsi, %rsp\n"
    "  popq %r15\n  popq %r14\n  popq %r13\n  popq %r12\n  popq %rbx\n  popq %rbp\n"
    "  ret\n");

static const size_t kStack = 256 * 1024;
static std::vector<emu_fiber> g_fibers;
static std::vector<emu_warp_state> g_warps;
static void *g_sched_sp;
static int g_cur = -1;
static unsigned g_nthreads, g_live;
static unsigned g_bar_count, g_bar_gen;
static unsigned long g_progress;
static void (*g_entry)(void *);
static void *g_arg;
static std::vector<uint8_t> g_dyn;
static size_t g_dyn_bytes;

/* ---- seeded schedules (MZ_EMU_SCHED) -------------------------------------------------------------- */
/* a fiber yields at a preemption point with probability 1 / EMU_PREEMPT_ONE_IN */
static const unsigned EMU_PREEMPT_ONE_IN = 32;
int emu_sched_on, emu_race_on, emu_hooks_on;
static uint64_t g_rng;
static unsigned long g_launches, g_blocks_run;

static uint64_t rng_next(void) { /* splitmix64 */
    uint64_t z = (g_rng += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static void rng_fill(uint8_t *p, size_t n) {
    for (size_t i = 0; i < n; i += 8) {
        uint64_t r = rng_next();
        memcpy(p + i, &r, n - i < 8 ? n - i : 8);
    }
}
template <typename T> static void rng_shuffle(std::vector<T> &v) {
    for (size_t i = v.size(); i > 1; i--) std::swap(v[i - 1], v[rng_next() % i]);
}

__attribute__((constructor)) static void emu_env_init(void) {
    const char *s = getenv("MZ_EMU_SCHED");
    const uint64_t seed = s ? strtoull(s, NULL, 0) : 0;
    emu_sched_on = seed != 0;
    g_rng = seed * 0x2545F4914F6CDD1Dull;
    const char *r = getenv("MZ_EMU_RACE");
    emu_race_on = r && atoi(r) != 0;
    emu_hooks_on = emu_sched_on || emu_race_on;
}

/* static __shared__ storage of the library this file is linked into (weak: a library may have none) */
extern uint8_t __start_mz_emu_shared[] __attribute__((weak, visibility("hidden")));
extern uint8_t __stop_mz_emu_shared[] __attribute__((weak, visibility("hidden")));

const std::vector<uint64_t> &emu_block_order(uint64_t nblocks) {
    static std::vector<uint64_t> order;
    order.resize(nblocks);
    for (uint64_t i = 0; i < nblocks; i++) order[i] = i;
    if (emu_sched_on) rng_shuffle(order);
    g_launches++;
    return order;
}

emu_warp_state *emu_cur_warp(void) { return &g_warps[g_cur >> 5]; }
int emu_lane(void) { return g_cur & 31; }

void emu_yield(void) {
    emu_fiber *f = &g_fibers[g_cur];
    emu_switch(&f->sp, g_sched_sp);
}

void emu_preempt_slow(void) {
    if (g_cur < 0 || rng_next() % EMU_PREEMPT_ONE_IN) return;
    g_progress++; /* a fiber that yields here is runnable: not a deadlock */
    emu_yield();
}

/* ---- race checker (MZ_EMU_RACE) ------------------------------------------------------------------- */
/* Happens-before at two granularities. Across warps: ne[w] counts the block and named barriers warp w completed with all its
 * live lanes, and know[a][w] is the count of warp w that warp a has synchronised with (a vector clock over warps, joined at
 * every such barrier). Within a warp: wfe[w] counts warp barriers that held every live lane, and the lanes' vector clocks
 * lvc over lanes are joined at warp barriers that held only some. An access by thread t recorded at (ne, wfe, lc) is
 * ordered before the current thread u when u == t, or know[wu][wt] > ne for another warp, or for the same warp when the warp
 * passed a block/named or full warp barrier since, or lvc[u][lane t] > lc. */
static const int EMU_RACE_READERS = 4;
struct RaceRec {
    int32_t tid;
    uint32_t ne, wfe, lc;
    uint32_t mask; /* bytes of the word it touched */
};
struct RaceWord {
    unsigned long stamp; /* g_blocks_run of the CTA the record belongs to */
    RaceRec w;
    int w_atomic;
    int nr;
    unsigned rr;
    RaceRec r[EMU_RACE_READERS];
};
static std::vector<RaceWord> g_shadow_dyn, g_shadow_static;
static uint32_t g_ne[32], g_wfe[32], g_know[32][32];
static std::vector<uint32_t> g_lc;                  /* per thread */
static std::vector<std::array<uint32_t, 32>> g_lvc; /* per thread, over the lanes of its warp */
static unsigned g_nb_arr[16][32];                   /* lanes that arrived at named barrier id in its current generation */

static void race_reset_block(unsigned nthreads) {
    memset(g_ne, 0, sizeof(g_ne));
    memset(g_wfe, 0, sizeof(g_wfe));
    memset(g_know, 0, sizeof(g_know));
    memset(g_nb_arr, 0, sizeof(g_nb_arr));
    g_lc.assign(nthreads, 0);
    g_lvc.assign(nthreads, std::array<uint32_t, 32>());
}

/* a barrier that every live lane of each warp in `warps` passed */
static void race_warps_sync(uint32_t warps) {
    uint32_t join[32] = {0};
    for (int p = 0; p < 32; p++)
        if (warps >> p & 1) {
            g_ne[p]++;
            for (int x = 0; x < 32; x++) join[x] = std::max(join[x], g_know[p][x]);
        }
    for (int p = 0; p < 32; p++)
        if (warps >> p & 1) join[p] = g_ne[p];
    for (int p = 0; p < 32; p++)
        if (warps >> p & 1) memcpy(g_know[p], join, sizeof(join));
}

static void race_warp_barrier(int w, unsigned lanes) {
    if ((lanes & g_warps[w].live_mask) == g_warps[w].live_mask) {
        g_wfe[w]++;
        return;
    }
    std::array<uint32_t, 32> join{};
    for (int l = 0; l < 32; l++)
        if (lanes >> l & 1) {
            uint32_t t = (uint32_t)w * 32 + l;
            g_lc[t]++;
            for (int x = 0; x < 32; x++) join[x] = std::max(join[x], g_lvc[t][x]);
        }
    for (int l = 0; l < 32; l++)
        if (lanes >> l & 1) join[l] = g_lc[w * 32 + l];
    for (int l = 0; l < 32; l++)
        if (lanes >> l & 1) g_lvc[w * 32 + l] = join;
}

static RaceRec race_now(uint32_t mask) {
    const int w = g_cur >> 5;
    RaceRec r = {g_cur, g_ne[w], g_wfe[w], g_lc[g_cur], mask};
    return r;
}

static bool ordered(const RaceRec &a, int u) {
    if (a.tid == u) return true;
    const int wa = a.tid >> 5, wu = u >> 5;
    if (wa != wu) return g_know[wu][wa] > a.ne;
    return g_ne[wa] > a.ne || g_wfe[wa] > a.wfe || g_lvc[u][a.tid & 31] > a.lc;
}

static void race_report(const char *what, const char *region, size_t word, const RaceRec &a, const char *a_kind, const char *b_kind) {
    fprintf(stderr,
            "cuda_emu: shared-memory race (%s) in launch %lu, block (%u,%u,%u), %s shared word at byte offset 0x%zx: thread %d (%s) "
            "and thread %d (%s) with no barrier between them\n",
            what, g_launches, blockIdx.x, blockIdx.y, blockIdx.z, region, word * 4, a.tid, a_kind, g_cur, b_kind);
    fflush(stderr);
    abort();
}

static void race_word(RaceWord &s, const char *region, size_t word, uint32_t mask, int kind, const uint8_t *oldb, const uint8_t *newb) {
    if (s.stamp != g_blocks_run) {
        s.stamp = g_blocks_run;
        s.w.tid = -1;
        s.nr = 0;
        s.rr = 0;
    }
    const int u = g_cur;
    if (kind == EMU_ACC_READ) {
        if (s.w.tid >= 0 && !s.w_atomic && (s.w.mask & mask) && !ordered(s.w, u)) race_report("write then read", region, word, s.w, "plain write", "read");
        const RaceRec now = race_now(mask);
        for (int i = 0; i < s.nr; i++)
            if (s.r[i].tid == u) {
                s.r[i] = now;
                return;
            }
        if (s.nr < EMU_RACE_READERS) {
            s.r[s.nr++] = now;
            return;
        }
        for (int i = 0; i < s.nr; i++) /* a read ordered before this one is covered by it */
            if (ordered(s.r[i], u)) {
                s.r[i] = now;
                return;
            }
        s.r[s.rr++ % EMU_RACE_READERS] = now;
        return;
    }
    const bool atomic = kind == EMU_ACC_ATOMIC;
    for (int i = 0; i < s.nr; i++)
        if ((s.r[i].mask & mask) && !ordered(s.r[i], u)) race_report("read then write", region, word, s.r[i], "read", atomic ? "atomic" : "plain write");
    if (s.w.tid >= 0 && (s.w.mask & mask) && !(atomic && s.w_atomic) && !ordered(s.w, u)) {
        bool same = !atomic && !s.w_atomic;
        for (int b = 0; b < 4 && same; b++)
            if (mask >> b & 1) same = oldb[b] == newb[b];
        if (!same) race_report("write then write", region, word, s.w, s.w_atomic ? "atomic" : "plain write", atomic ? "atomic" : "plain write");
    }
    s.w = race_now(mask);
    s.w_atomic = atomic;
    s.nr = 0;
}

static void race_access(const void *ptr, unsigned bytes, int kind, const void *newval) {
    const uint8_t *p = (const uint8_t *)ptr;
    const uint8_t *base;
    std::vector<RaceWord> *shadow;
    const char *region;
    size_t span;
    if (p >= emu_dyn_smem && p < emu_dyn_smem + g_dyn_bytes) {
        base = emu_dyn_smem, shadow = &g_shadow_dyn, region = "dynamic", span = g_dyn_bytes;
    } else if (__start_mz_emu_shared && p >= __start_mz_emu_shared && p < __stop_mz_emu_shared) {
        base = (const uint8_t *)((uintptr_t)__start_mz_emu_shared & ~(uintptr_t)3), shadow = &g_shadow_static, region = "static";
        span = (size_t)(__stop_mz_emu_shared - base);
    } else {
        return; /* global memory: not checked */
    }
    if (shadow->size() < (span + 3) / 4) shadow->resize((span + 3) / 4, RaceWord());
    const size_t first = (size_t)(p - base), last = first + bytes - 1;
    for (size_t w = first / 4; w <= last / 4; w++) {
        uint32_t mask = 0;
        uint8_t oldb[4] = {0}, newb[4] = {0};
        for (int b = 0; b < 4; b++) {
            const size_t at = w * 4 + b;
            if (at < first || at > last) continue;
            mask |= 1u << b;
            oldb[b] = base[at];
            if (newval) newb[b] = ((const uint8_t *)newval)[at - first];
        }
        race_word((*shadow)[w], region, w, mask, kind, oldb, newb);
    }
}

void emu_access_slow(const void *p, unsigned bytes, int kind, const void *newval) {
    if (g_cur < 0) return;
    if (emu_sched_on) emu_preempt_slow();
    if (emu_race_on) race_access(p, bytes, kind, newval);
}

/* ---- barriers ------------------------------------------------------------------------------------- */
static void release_check_block(void) {
    if (g_live > 0 && g_bar_count >= g_live) {
        g_bar_count = 0;
        g_bar_gen++;
        g_progress++;
        if (emu_race_on) race_warps_sync((uint32_t)(((uint64_t)1 << g_warps.size()) - 1));
    }
}

void emu_block_barrier(void) {
    unsigned gen = g_bar_gen;
    g_bar_count++;
    release_check_block();
    while (g_bar_gen == gen) emu_yield();
}

static unsigned g_nb_count[16], g_nb_gen[16];
void emu_named_barrier(int id, int nthreads) {
    unsigned gen = g_nb_gen[id];
    g_nb_count[id]++;
    g_nb_arr[id][g_cur >> 5] |= 1u << (g_cur & 31);
    if (g_nb_count[id] >= (unsigned)nthreads) {
        g_nb_count[id] = 0;
        g_nb_gen[id]++;
        g_progress++;
        if (emu_race_on) { /* warps whose every live lane arrived in this generation */
            uint32_t warps = 0;
            for (size_t w = 0; w < g_warps.size(); w++)
                if (g_nb_arr[id][w] && (g_nb_arr[id][w] & g_warps[w].live_mask) == g_warps[w].live_mask) warps |= 1u << w;
            race_warps_sync(warps);
        }
        memset(g_nb_arr[id], 0, sizeof(g_nb_arr[id]));
        return;
    }
    while (g_nb_gen[id] == gen) emu_yield();
}

/* release lane l's group when every lane its mask names has arrived (lanes that exited are not waited for) */
static void warp_try_release(emu_warp_state *w, int l) {
    const unsigned m = (w->want[l] & w->live_mask) | (1u << l);
    if ((w->arrived & m) != m) return;
    w->arrived &= ~m;
    for (unsigned b = m; b; b &= b - 1) w->gen[__builtin_ctz(b)]++;
    g_progress++;
    if (emu_race_on) race_warp_barrier((int)(w - g_warps.data()), m);
}

void emu_warp_barrier(unsigned mask) {
    emu_warp_state *w = emu_cur_warp();
    const int lane = emu_lane();
    const unsigned gen = w->gen[lane];
    w->want[lane] = mask | (1u << lane);
    w->arrived |= 1u << lane;
    warp_try_release(w, lane);
    while (w->gen[lane] == gen) emu_yield();
}

static void trampoline(void) {
    g_entry(g_arg);
    emu_fiber *f = &g_fibers[g_cur];
    f->done = 1;
    g_live--;
    emu_warp_state *w = emu_cur_warp();
    w->live_mask &= ~(1u << emu_lane());
    g_progress++;
    /* an exiting thread may complete a barrier others wait on */
    release_check_block();
    for (unsigned b = w->arrived; b; b &= b - 1)
        if (w->arrived >> __builtin_ctz(b) & 1) warp_try_release(w, __builtin_ctz(b));
    emu_switch(&f->sp, g_sched_sp);
    abort();
}

static pthread_mutex_t g_launch_mu = PTHREAD_MUTEX_INITIALIZER;
void emu_launch_lock(void) { pthread_mutex_lock(&g_launch_mu); }
void emu_launch_unlock(void) { pthread_mutex_unlock(&g_launch_mu); }

void emu_run_block(unsigned nthreads, void (*entry)(void *), void *arg, size_t dyn_smem) {
    if (g_fibers.size() < nthreads) {
        size_t old = g_fibers.size();
        g_fibers.resize(nthreads);
        for (size_t i = old; i < nthreads; i++) {
            g_fibers[i].stack = mmap(NULL, kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
            if (g_fibers[i].stack == MAP_FAILED) { perror("mmap"); abort(); }
        }
    }
    g_warps.assign((nthreads + 31) / 32, emu_warp_state());
    g_dyn.assign(dyn_smem + 64, 0xCD); /* garbage like the device */
    emu_dyn_smem = (uint8_t *)(((uintptr_t)g_dyn.data() + 15) & ~(uintptr_t)15);
    g_dyn_bytes = dyn_smem;
    if (emu_sched_on) {
        rng_fill(g_dyn.data(), g_dyn.size());
        if (__start_mz_emu_shared) rng_fill(__start_mz_emu_shared, (size_t)(__stop_mz_emu_shared - __start_mz_emu_shared));
    }
    g_blocks_run++;
    if (emu_race_on) race_reset_block(nthreads);
    g_entry = entry;
    g_arg = arg;
    g_nthreads = g_live = nthreads;
    g_bar_count = 0;
    for (int i = 0; i < 16; i++) g_nb_count[i] = 0;
    for (unsigned i = 0; i < nthreads; i++) {
        emu_fiber *f = &g_fibers[i];
        f->done = 0;
        f->tid = (int)i;
        uintptr_t top = ((uintptr_t)f->stack + kStack) & ~(uintptr_t)15;
        void **sp = (void **)top;
        *--sp = NULL;                 /* keeps rsp%16==8 at trampoline entry */
        *--sp = (void *)trampoline;   /* return address for emu_switch's ret */
        for (int k = 0; k < 6; k++) *--sp = NULL; /* r15 r14 r13 r12 rbx rbp */
        f->sp = sp;
        g_warps[i >> 5].live_mask |= 1u << (i & 31);
    }
    std::vector<unsigned> order(nthreads);
    for (unsigned i = 0; i < nthreads; i++) order[i] = i;
    while (g_live > 0) {
        unsigned long before = g_progress;
        if (emu_sched_on) rng_shuffle(order);
        for (unsigned i : order) {
            if (g_fibers[i].done) continue;
            g_cur = (int)i;
            threadIdx = emu_dim3(i % blockDim.x, (i / blockDim.x) % blockDim.y, i / (blockDim.x * blockDim.y));
            emu_switch(&g_sched_sp, g_fibers[i].sp);
        }
        if (g_progress == before && g_live > 0) {
            fprintf(stderr, "cuda_emu: deadlock in block (%u,%u,%u): %u threads stuck (barrier count %u)\n", blockIdx.x,
                    blockIdx.y, blockIdx.z, g_live, g_bar_count);
            abort();
        }
    }
    g_cur = -1;
}
