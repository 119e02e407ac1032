/* mz_strm_cuda.c -- minizip-ng codec stream whose DEFLATE / inflate / CRC arithmetic runs on an H100.
 *
 * Host side in C, mirroring mz_strm_zlib.c function for function (citations at each entry point); the
 * arithmetic lives in the sm_90a kernels behind include/mz_cuda_batch.h. There is no CPU codec here:
 * if the GPU runtime cannot be initialised open() fails with MZ_SUPPORT_ERROR.
 *
 * Write path (mz_strm_zlib.c:203-264 equivalent): caller bytes accumulate in a pinned staging buffer;
 * a full batch goes H2D, is cut into independent <=64 KiB chunks, compressed by K2+K3, joined by K4,
 * comes back D2H and is handed to the base stream. Batches written before close() end with a sync
 * marker; close() compresses what is left as the final batch (BFINAL) -- an empty one if need be --
 * and appends the gzip / zlib trailer.
 *
 * Read path (mz_strm_zlib.c:116-193 equivalent): compressed bytes are pulled from the base stream
 * into a pinned window, the resumable K5 decoder runs until it needs input or output space, decoded
 * bytes come back into a host buffer from which read() calls are served. TOTAL_IN counts consumed
 * compressed bytes exactly at end of stream, as mz_zip.c:2090-2112 relies on.
 */
#include "mz_strm_cuda.h"

#include <pthread.h>
#include <sched.h>
#include <stdatomic.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "mz_abi.h"
#include "mz_cuda_batch.h"

#define CU_CHUNK 65536u

/* ---- workspaces: pinned + device buffers are expensive to create, so streams borrow them ---------- */
#define CU_NSLOT 3 /* write pipeline depth: upload of batch k+1 overlaps compute of k and download of k-1 */
#define CU_CRC_RING 64
#define CU_CRC_SEG ((uint64_t)16384)

typedef struct cu_slot_s {
    void *stream;   /* cudaStream_t */
    void *ev_h2d;   /* input upload finished: caller memory may be reused */
    void *ev_d2h[2]; /* download pieces: piece i+1 travels while piece i is handed to base */
    uint8_t *h_in;  /* pinned staging for pageable / small writes */
    uint8_t *d_in, *d_slots, *d_out, *h_out;
    uint32_t *d_out_len, *d_residue, *d_crc2;
    uint64_t *d_offsets;
    uint64_t *h_total; /* pinned: [0] joined bytes, [1] low word = crc32 of the batch */
    size_t n;          /* input bytes of the batch in flight */
    int busy;
} cu_slot;

typedef struct cu_ws_s {
    int device; /* CUDA device the buffers, streams and events belong to */
    struct cu_ws_s *next;
    int kind; /* 1 write, 2 read */
    size_t batch;
    /* write */
    cu_slot slot[CU_NSLOT];
    int cur; /* slot being filled */
    uint32_t max_chunks;
    uint64_t slot_stride;
    /* read */
    uint8_t *h_cin, *d_cin, *d_win, *h_dec;
    uint8_t *d_win2; /* long streams: second output window, so that decoding can go on while the first is still being delivered */
    size_t cin_cap, win_cap;
    size_t ring_cap; /* h_cin is a ring of this many bytes (+ 64 zero bytes behind it): the compressed window is cin_cap of it at most, the
                      * rest holds bytes read ahead from base while a round is in flight (long streams: 2 x cin_cap) */
    mz_cuda_inflate_job *h_job, *d_job;
    mz_cuda_inflate_state *h_state, *d_state;
    /* read, long streams: segment-speculative rounds (K6) */
    int large;
    void *d_spec;
    uint32_t spec_max_seg;
    size_t spec_seg_bytes;
    mz_cuda_spec_summary *h_sum, *d_sum;
    void *rstream;  /* decode stream: uploads, K5/K6 launches, state copies */
    void *dstream;  /* delivery stream: CRC + download of finished output, overlaps a round in flight */
    void *rev;      /* K6 round in flight finished (summary is in h_sum) */
    /* gzip members: the CRC-32 of every delivered piece is computed on a THIRD stream and folded when it is there -- on the
     * delivery stream the kernel would queue behind a K6 round that fills the SMs, and the caller's thread with it */
    void *cstream;
    void *cev[CU_CRC_RING];
    uint32_t *d_cres;          /* per ring slot: segment residues + 2 words of fold output */
    uint32_t *h_cres;          /* pinned, 2 words per slot: {residue, crc of the piece from 0} */
    uint64_t clen[CU_CRC_RING];
    uint64_t c_head, c_tail;   /* pieces folded / enqueued so far (slot = count % CU_CRC_RING) */
    int pending;    /* a K6 round is in flight */
    uint64_t pend_nseg;
} cu_ws;

static pthread_mutex_t g_pool_mu = PTHREAD_MUTEX_INITIALIZER;
static cu_ws *g_pool;

static size_t env_size(const char *name, size_t dflt, size_t unit) {
    const char *v = getenv(name);
    if (!v || !*v)
        return dflt;
    long long n = atoll(v);
    return n > 0 ? (size_t)n * unit : dflt;
}

/* words of CRC scratch per ring slot: one residue per 16 KiB segment of a delivery piece (half the host buffer) + fold output */
static size_t cu_crc_slot_words(size_t batch) {
    return (size_t)((batch / 2 + CU_CRC_SEG - 1) / CU_CRC_SEG) + 8;
}

static void ws_destroy(cu_ws *w) {
    if (!w)
        return;
    for (int i = 0; i < CU_NSLOT; i++) {
        cu_slot *s = &w->slot[i];
        mz_cuda_host_free(s->h_in);
        mz_cuda_free(s->d_in);
        mz_cuda_free(s->d_slots);
        mz_cuda_free(s->d_out);
        mz_cuda_host_free(s->h_out);
        mz_cuda_free(s->d_out_len);
        mz_cuda_free(s->d_residue);
        mz_cuda_free(s->d_crc2);
        mz_cuda_free(s->d_offsets);
        mz_cuda_host_free(s->h_total);
        mz_cuda_event_destroy(s->ev_h2d);
        mz_cuda_event_destroy(s->ev_d2h[0]);
        mz_cuda_event_destroy(s->ev_d2h[1]);
        mz_cuda_stream_destroy(s->stream);
    }
    mz_cuda_host_free(w->h_cin);
    mz_cuda_free(w->d_cin);
    mz_cuda_free(w->d_win);
    mz_cuda_free(w->d_win2);
    mz_cuda_host_free(w->h_dec);
    mz_cuda_host_free(w->h_job);
    mz_cuda_free(w->d_job);
    mz_cuda_host_free(w->h_state);
    mz_cuda_free(w->d_state);
    mz_cuda_free(w->d_spec);
    mz_cuda_host_free(w->h_sum);
    mz_cuda_free(w->d_sum);
    mz_cuda_event_destroy(w->rev);
    for (int i = 0; i < CU_CRC_RING; i++)
        mz_cuda_event_destroy(w->cev[i]);
    mz_cuda_free(w->d_cres);
    mz_cuda_host_free(w->h_cres);
    mz_cuda_stream_destroy(w->rstream);
    mz_cuda_stream_destroy(w->dstream);
    mz_cuda_stream_destroy(w->cstream);
    free(w);
}

#define CU_POOL_MAX 8
static cu_ws *ws_acquire(int kind) {
    cu_ws *w = NULL, **pp;
    size_t batch = env_size("MZ_CUDA_BATCH_KB", 32u << 20, 1024);
    batch = (batch + CU_CHUNK - 1) / CU_CHUNK * CU_CHUNK;
    const int device = mz_cuda_get_device();
    pthread_mutex_lock(&g_pool_mu);
    for (pp = &g_pool; *pp; pp = &(*pp)->next)
        if ((*pp)->kind == kind && (*pp)->batch == batch && (*pp)->device == device) { /* never hand out another device's workspace */
            w = *pp;
            *pp = w->next;
            break;
        }
    pthread_mutex_unlock(&g_pool_mu);
    if (w)
        return w;
    w = (cu_ws *)calloc(1, sizeof(cu_ws));
    if (!w)
        return NULL;
    w->kind = kind;
    w->batch = batch;
    w->device = device;
    if (kind == 1) {
        w->max_chunks = (uint32_t)(batch / CU_CHUNK);
        w->slot_stride = mz_cuda_deflate_slot_bound(CU_CHUNK);
        size_t slots = (size_t)w->max_chunks * w->slot_stride;
        for (int i = 0; i < CU_NSLOT; i++) {
            cu_slot *s = &w->slot[i];
            s->stream = mz_cuda_stream_create();
            s->ev_h2d = mz_cuda_event_create();
            s->ev_d2h[0] = mz_cuda_event_create();
            s->ev_d2h[1] = mz_cuda_event_create();
            s->h_in = (uint8_t *)mz_cuda_host_alloc(batch);
            s->d_in = (uint8_t *)mz_cuda_malloc(batch + 64);
            s->d_slots = (uint8_t *)mz_cuda_malloc(slots);
            s->d_out = (uint8_t *)mz_cuda_malloc(slots);
            s->h_out = (uint8_t *)mz_cuda_host_alloc(slots);
            s->d_out_len = (uint32_t *)mz_cuda_malloc((size_t)w->max_chunks * 4);
            s->d_residue = (uint32_t *)mz_cuda_malloc((size_t)w->max_chunks * 4);
            s->d_crc2 = (uint32_t *)mz_cuda_malloc(8);
            s->d_offsets = (uint64_t *)mz_cuda_malloc(((size_t)w->max_chunks + 1) * 8);
            s->h_total = (uint64_t *)mz_cuda_host_alloc(16);
            if (!s->stream || !s->ev_h2d || !s->ev_d2h[0] || !s->ev_d2h[1] || !s->h_in || !s->d_in || !s->d_slots || !s->d_out || !s->h_out || !s->d_out_len ||
                !s->d_residue || !s->d_crc2 || !s->d_offsets || !s->h_total) {
                ws_destroy(w);
                return NULL;
            }
        }
    } else {
        w->cin_cap = batch / 4 > (1u << 20) ? batch / 4 : (1u << 20);
        w->win_cap = 32768 + batch;
        w->ring_cap = w->cin_cap;
        w->h_cin = (uint8_t *)mz_cuda_host_alloc(w->ring_cap + 64);
        if (w->h_cin)
            memset(w->h_cin + w->ring_cap, 0, 64); /* the pad uploaded behind the window; never written again */
        w->d_cin = (uint8_t *)mz_cuda_malloc(w->cin_cap + 64);
        w->d_win = (uint8_t *)mz_cuda_malloc(w->win_cap + 512);
        w->h_dec = (uint8_t *)mz_cuda_host_alloc(batch);
        w->h_job = (mz_cuda_inflate_job *)mz_cuda_host_alloc(sizeof(mz_cuda_inflate_job));
        w->d_job = (mz_cuda_inflate_job *)mz_cuda_malloc(sizeof(mz_cuda_inflate_job));
        w->h_state = (mz_cuda_inflate_state *)mz_cuda_host_alloc(sizeof(mz_cuda_inflate_state));
        w->d_state = (mz_cuda_inflate_state *)mz_cuda_malloc(sizeof(mz_cuda_inflate_state));
        w->rstream = mz_cuda_stream_create();
        w->dstream = mz_cuda_stream_create();
        w->rev = mz_cuda_event_create();
        w->cstream = mz_cuda_stream_create();
        w->d_cres = (uint32_t *)mz_cuda_malloc((size_t)CU_CRC_RING * cu_crc_slot_words(batch) * 4);
        w->h_cres = (uint32_t *)mz_cuda_host_alloc((size_t)CU_CRC_RING * 8);
        int cev_ok = 1;
        for (int i = 0; i < CU_CRC_RING; i++) {
            w->cev[i] = mz_cuda_event_create();
            cev_ok &= w->cev[i] != NULL;
        }
        if (!cev_ok || !w->cstream || !w->d_cres || !w->h_cres || !w->h_cin || !w->d_cin || !w->d_win || !w->h_dec || !w->h_job || !w->d_job || !w->h_state || !w->d_state || !w->rstream ||
            !w->dstream || !w->rev) {
            ws_destroy(w);
            return NULL;
        }
    }
    return w;
}

static void ws_release(cu_ws *w) {
    if (!w)
        return;
    if (w->kind == 2) {
        if (w->pending)
            mz_cuda_stream_sync(w->rstream);
        w->pending = 0;
        mz_cuda_stream_sync(w->dstream); /* a piece may still be on its way into h_dec (abandoned read) */
        mz_cuda_stream_sync(w->cstream);
        w->c_head = w->c_tail = 0;
    }
    if (w->kind == 1) {
        for (int i = 0; i < CU_NSLOT; i++) {
            if (w->slot[i].busy)
                mz_cuda_stream_sync(w->slot[i].stream);
            w->slot[i].busy = 0;
        }
        w->cur = 0;
    }
    /* keep the pool bounded: at most CU_POOL_MAX idle workspaces per kind, and at most one of the big read workspaces
     * (128 MiB pinned + ~640 MiB device, taken by one long stream) -- the rest is given back */
    int same = 0, large = 0;
    pthread_mutex_lock(&g_pool_mu);
    for (cu_ws *q = g_pool; q; q = q->next) {
        same += q->kind == w->kind;
        large += q->kind == 2 && q->large;
    }
    const int keep = same < CU_POOL_MAX && !(w->kind == 2 && w->large && large >= 1);
    if (keep) {
        w->next = g_pool;
        g_pool = w;
    }
    pthread_mutex_unlock(&g_pool_mu);
    if (!keep)
        ws_destroy(w);
}

/* ---- the stream object ------------------------------------------------------------------------------ */
typedef struct mz_stream_cuda_s {
    mz_stream stream; /* must be first: mz_strm.h:69-72 */
    int32_t error;
    int8_t initialized;
    int16_t level;
    int32_t window_bits;
    int32_t mode;
    int64_t total_in;
    int64_t total_out;
    int64_t max_total_in;
    cu_ws *ws;
    /* write */
    size_t in_len;      /* bytes staged in the current slot's h_in */
    uint32_t crc;       /* running CRC-32 of the plaintext (gzip trailer) */
    uint64_t crc_bytes; /* plaintext bytes folded into crc so far */
    uint32_t adler_a, adler_b;
    int8_t header_done;
    /* read */
    int8_t hdr_parsed, ended, base_eof;
    int wrap;           /* 0 raw, 1 zlib, 2 gzip */
    int64_t hdr_size;   /* framing bytes before the raw stream */
    uint64_t cin_base;  /* raw-stream offset of the first byte of the compressed window */
    size_t cin_len;     /* bytes in the window (what the kernels see: d_cin[0 .. cin_len)) */
    size_t cin_off;     /* where the window starts in the ring ws->h_cin */
    size_t ahead_len;   /* bytes read from base beyond the window (behind it in the ring), not yet uploaded */
    int8_t verify_copy; /* MZ_CUDA_VERIFY_COPY=1: compare every copy into the caller's buffer with its source (debug aid) */
    int8_t ahead_force; /* MZ_CUDA_READ_AHEAD=2: read ahead whether or not the round is still running (tests: on the emulator it never is) */
    uint64_t win_base;  /* output offset of byte 0 of the window being decoded into */
    int dwin, lwin;     /* which window (0 = ws->d_win, 1 = ws->d_win2) is decoded into / delivered from */
    uint64_t lwin_base; /* output offset of byte 0 of the delivery window, while it is not the decode window */
    uint64_t lwin_end;  /* ... and where its bytes end */
    size_t dec_pos, dec_len; /* decoded bytes waiting in ws->h_dec + dec_base */
    size_t dec_base;         /* which half of h_dec the caller is reading */
    size_t pre_len;          /* bytes of the NEXT piece already on their way into the other half (0 = none) */
    uint64_t fed_in;    /* compressed bytes pulled from base (framing included) */
    uint64_t deliv_pos; /* output bytes already copied out of ws->d_win */
    uint64_t spec_resume_bit; /* no speculative round before the decoder has passed this stream bit */
    double ratio_est;   /* output bytes per compressed byte seen so far (sizes the rounds) */
    int8_t cin_dirty;   /* ws->h_cin changed since the last upload */
    /* MZ_CUDA_TRACE: where the caller's thread spent its time on the read path (ns), printed by close() */
    int8_t trace;
    uint64_t t_base, t_move, t_round, t_piece, t_serial, t_copy, t_ahead, n_round, n_serial, n_ahead, n_wrap;
} mz_stream_cuda;

/* ---- copying decoded bytes to the caller --------------------------------------------------------------------------
 * On a long member the caller's thread spends more time in this memcpy than in anything else (pinned staging -> the caller's
 * pageable buffer, one core: ~8 GB/s). Copies of 256 KiB and more are therefore split over a few helper threads
 * (MZ_CUDA_COPY_THREADS, default 4 including the caller; 1 = plain memcpy). The helpers spin for a moment after a job -- a
 * reader that calls read() in a loop finds them awake -- and sleep on a condition variable otherwise. One parallel copy at a
 * time per process; a second stream reading concurrently simply copies on its own thread. */
#define CU_COPY_MAX 8
static struct {
    pthread_mutex_t use;  /* held by the stream that is copying */
    pthread_mutex_t mu;
    pthread_cond_t cv;
    pthread_t th[CU_COPY_MAX];
    int n;                /* helpers running */
    int want;             /* -1 = environment not read yet */
    atomic_uint gen, done;
    uint8_t *dst;
    const uint8_t *src;
    size_t part, total;
    int parts;
} g_cp = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, {0}, 0, -1, 0, 0, NULL, NULL, 0, 0, 0};

static void cp_slice(int k) {
    const size_t o = (size_t)k * g_cp.part;
    if (o < g_cp.total)
        memcpy(g_cp.dst + o, g_cp.src + o, g_cp.total - o < g_cp.part ? g_cp.total - o : g_cp.part);
}

static void *cp_helper(void *arg) {
    const int me = (int)(intptr_t)arg; /* slice index 1.. */
    unsigned seen = 0;
    for (;;) {
        unsigned g = atomic_load_explicit(&g_cp.gen, memory_order_acquire);
        if (g == seen) { /* spin briefly, then sleep */
            for (int i = 0; i < 20000 && g == seen; i++) {
                if ((i & 63) == 63)
                    sched_yield();
                g = atomic_load_explicit(&g_cp.gen, memory_order_acquire);
            }
            if (g == seen) {
                pthread_mutex_lock(&g_cp.mu);
                while ((g = atomic_load_explicit(&g_cp.gen, memory_order_acquire)) == seen)
                    pthread_cond_wait(&g_cp.cv, &g_cp.mu);
                pthread_mutex_unlock(&g_cp.mu);
            }
        }
        seen = g;
        if (me < g_cp.parts)
            cp_slice(me);
        atomic_fetch_add_explicit(&g_cp.done, 1, memory_order_release);
    }
    return NULL;
}

static void cu_copy_out(uint8_t *dst, const uint8_t *src, size_t n) {
    if (n < (256u << 10) || pthread_mutex_trylock(&g_cp.use) != 0) {
        memcpy(dst, src, n);
        return;
    }
    if (g_cp.want < 0) {
        const char *v = getenv("MZ_CUDA_COPY_THREADS");
        int w = (v && *v) ? atoi(v) : 4;
        g_cp.want = w < 1 ? 1 : (w > CU_COPY_MAX ? CU_COPY_MAX : w);
        for (int i = 1; i < g_cp.want; i++) {
            if (pthread_create(&g_cp.th[i], NULL, cp_helper, (void *)(intptr_t)i) != 0)
                break;
            pthread_detach(g_cp.th[i]);
            g_cp.n++;
        }
    }
    if (g_cp.n == 0) {
        memcpy(dst, src, n);
        pthread_mutex_unlock(&g_cp.use);
        return;
    }
    g_cp.parts = g_cp.n + 1;
    g_cp.part = (((n + (size_t)g_cp.parts - 1) / (size_t)g_cp.parts) + 4095) & ~(size_t)4095; /* parts * part >= n: round the quotient UP first */
    g_cp.total = n;
    g_cp.dst = dst;
    g_cp.src = src;
    atomic_store_explicit(&g_cp.done, 0, memory_order_relaxed);
    pthread_mutex_lock(&g_cp.mu);
    atomic_fetch_add_explicit(&g_cp.gen, 1, memory_order_release);
    pthread_cond_broadcast(&g_cp.cv);
    pthread_mutex_unlock(&g_cp.mu);
    cp_slice(0);
    while (atomic_load_explicit(&g_cp.done, memory_order_acquire) < (unsigned)g_cp.n)
        sched_yield();
    pthread_mutex_unlock(&g_cp.use);
}

static inline uint64_t now_ns(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}
#define CU_TIMED(cu, acc, stmt)          \
    do {                                 \
        if ((cu)->trace) {               \
            const uint64_t t0_ = now_ns(); \
            stmt;                        \
            (cu)->acc += now_ns() - t0_; \
        } else {                         \
            stmt;                        \
        }                                \
    } while (0)

static mz_stream_vtbl mz_stream_cuda_vtbl = {
    mz_stream_cuda_open,   mz_stream_cuda_is_open, mz_stream_cuda_read,           mz_stream_cuda_write,
    mz_stream_cuda_tell,   mz_stream_cuda_seek,    mz_stream_cuda_close,          mz_stream_cuda_error,
    mz_stream_cuda_create, mz_stream_cuda_delete,  mz_stream_cuda_get_prop_int64, mz_stream_cuda_set_prop_int64};

static int valid_window_bits(int32_t wb) {
    /* what zlib's deflateInit2 / inflateInit2 accept (zlib.h:539-572, 834-870); 8 is bumped to 9 by deflate */
    return (wb >= -15 && wb <= -8) || (wb >= 8 && wb <= 15) || (wb >= 24 && wb <= 31);
}

static int wrap_of(int32_t wb) {
    return wb < 0 ? 0 : (wb > 15 ? 2 : 1);
}

/* mz_strm_zlib.c:65-107. Does not touch `base` (minigzip.c:92-93 opens before set_base). */
int32_t mz_stream_cuda_open(void *stream, const char *path, int32_t mode) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    (void)path;
    cu->total_in = 0;
    cu->total_out = 0;
    cu->error = 0;
    if (mode & MZ_OPEN_MODE_WRITE) {
#ifdef MZ_ZIP_NO_COMPRESSION
        return MZ_SUPPORT_ERROR;
#else
        int lvl = (int8_t)cu->level; /* the reference passes (int8_t)level to deflateInit2, :87 */
        if (lvl == -1)
            lvl = 6;
        if (lvl < 0 || lvl > 9 || !valid_window_bits(cu->window_bits)) {
            cu->error = MZ_STREAM_ERROR; /* Z_STREAM_ERROR from deflateInit2 */
            return MZ_OPEN_ERROR;
        }
#endif
    } else if (mode & MZ_OPEN_MODE_READ) {
#ifdef MZ_ZIP_NO_DECOMPRESSION
        return MZ_SUPPORT_ERROR;
#else
        if (!valid_window_bits(cu->window_bits)) {
            cu->error = MZ_STREAM_ERROR;
            return MZ_OPEN_ERROR;
        }
#endif
    }
    if (mz_cuda_init() != MZ_OK) {
        cu->error = MZ_SUPPORT_ERROR;
        fprintf(stderr, "mz_strm_cuda: no usable sm_90 GPU (%s); there is no CPU fallback\n", mz_cuda_last_error());
        return MZ_SUPPORT_ERROR;
    }
    cu->in_len = 0;
    cu->crc = 0;
    cu->crc_bytes = 0;
    cu->adler_a = 1;
    cu->adler_b = 0;
    cu->header_done = 0;
    cu->hdr_parsed = cu->ended = cu->base_eof = 0;
    cu->wrap = wrap_of(cu->window_bits);
    cu->hdr_size = 0;
    cu->cin_base = 0;
    cu->cin_len = 0;
    cu->cin_off = cu->ahead_len = 0;
    cu->verify_copy = getenv("MZ_CUDA_VERIFY_COPY") != NULL;
    {
        const char *ra = getenv("MZ_CUDA_READ_AHEAD"); /* 0 = off, 1 = while a round is in flight (default), 2 = always (tests) */
        cu->ahead_force = ra ? (ra[0] == '2' ? 1 : (ra[0] == '0' ? -1 : 0)) : 0;
    }
    cu->win_base = 0;
    cu->dwin = cu->lwin = 0;
    cu->lwin_base = cu->lwin_end = 0;
    cu->dec_pos = cu->dec_len = 0;
    cu->dec_base = cu->pre_len = 0;
    cu->fed_in = 0;
    cu->deliv_pos = 0;
    cu->spec_resume_bit = 0;
    cu->ratio_est = 4.0;
    cu->cin_dirty = 1;
    cu->trace = getenv("MZ_CUDA_TRACE") != NULL || getenv("MZ_CUDA_READ_STATS") != NULL; /* (TRACE also serialises the K6 kernels to time them) */
    cu->t_base = cu->t_move = cu->t_round = cu->t_piece = cu->t_serial = cu->t_copy = cu->t_ahead = cu->n_round = cu->n_serial = cu->n_ahead = cu->n_wrap = 0;
    cu->initialized = 1;
    cu->mode = mode;
    return MZ_OK;
}

/* mz_strm_zlib.c:109-114 */
int32_t mz_stream_cuda_is_open(void *stream) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    if (cu->initialized != 1)
        return MZ_OPEN_ERROR;
    return MZ_OK;
}

/* ---- gzip framing, shared by the vtbl and the device-memory calls (mz_cuda_gzip_*_device) ------------------------------------ */
/* what zlib writes for windowBits 31 (RFC1952): no name, MTIME 0, XFL 2 for level 9, 4 for level < 2, OS 3 */
static void cu_gzip_header(int lvl, uint8_t h[10]) {
    static const uint8_t base[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};
    memcpy(h, base, 10);
    h[8] = (uint8_t)(lvl == 9 ? 2 : (lvl < 2 ? 4 : 0));
}

/* the header at p[0 .. n): *hdr_size = its length; MZ_DATA_ERROR for bad magic, method or flags, MZ_BUF_ERROR when it runs past n */
static int32_t cu_gzip_parse(const uint8_t *p, size_t n, size_t *hdr_size) {
    size_t i;
    if (n < 10)
        return n >= 2 && (p[0] != 0x1f || p[1] != 0x8b) ? MZ_DATA_ERROR : MZ_BUF_ERROR;
    if (p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || (p[3] & 0xe0))
        return MZ_DATA_ERROR;
    i = 10;
    if (p[3] & 4) {
        if (i + 2 > n)
            return MZ_BUF_ERROR;
        i += 2 + ((size_t)p[i] | ((size_t)p[i + 1] << 8));
    }
    if (p[3] & 8) {
        while (i < n && p[i])
            i++;
        i++;
    }
    if (p[3] & 16) {
        while (i < n && p[i])
            i++;
        i++;
    }
    if (p[3] & 2)
        i += 2;
    if (i > n)
        return MZ_BUF_ERROR;
    *hdr_size = i;
    return MZ_OK;
}

/* ---- write side --------------------------------------------------------------------------------------- */
#ifndef MZ_ZIP_NO_COMPRESSION
static int32_t cu_emit(mz_stream_cuda *cu, const uint8_t *p, uint64_t n) {
    /* the base interface takes int32 sizes; mz_strm_zlib.c:196-201 maps a short write to MZ_WRITE_ERROR */
    while (n > 0) {
        int32_t part = n > (1u << 30) ? (int32_t)(1u << 30) : (int32_t)n;
        if (mz_abi_base_write(cu->stream.base, p, part) != part)
            return MZ_WRITE_ERROR;
        p += part;
        n -= (uint64_t)part;
        cu->total_out += part;
    }
    return MZ_OK;
}

static int32_t cu_write_header(mz_stream_cuda *cu) {
    int lvl = (int8_t)cu->level == -1 ? 6 : (int8_t)cu->level;
    if (cu->header_done)
        return MZ_OK;
    cu->header_done = 1;
    if (cu->wrap == 2) {
        uint8_t h[10];
        cu_gzip_header(lvl, h);
        return cu_emit(cu, h, 10);
    }
    if (cu->wrap == 1) {
        /* RFC1950: CMF = deflate + window, FLG = level hint + check bits */
        int wb = cu->window_bits < 9 ? 9 : cu->window_bits;
        uint32_t cmf = 8u | ((uint32_t)(wb - 8) << 4);
        uint32_t flevel = lvl < 2 ? 0 : (lvl < 6 ? 1 : (lvl == 6 ? 2 : 3));
        uint32_t hdr = (cmf << 8) | (flevel << 6);
        hdr += 31 - (hdr % 31);
        uint8_t h[2] = {(uint8_t)(hdr >> 8), (uint8_t)hdr};
        return cu_emit(cu, h, 2);
    }
    return MZ_OK;
}

static void cu_adler_update(mz_stream_cuda *cu, const uint8_t *p, size_t n) {
    uint32_t a = cu->adler_a, b = cu->adler_b;
    while (n > 0) {
        size_t k = n > 5552 ? 5552 : n;
        n -= k;
        while (k--) {
            a += *p++;
            b += a;
        }
        a %= 65521u;
        b %= 65521u;
    }
    cu->adler_a = a;
    cu->adler_b = b;
}

/* Enqueue one batch on its slot's stream: upload, K2+K3, K4, K1 (gzip), and the 16 bytes of results.
 * `src` is pinned host memory (the slot's staging buffer or the caller's own pinned buffer). */
static int32_t cu_submit(mz_stream_cuda *cu, cu_slot *s, const uint8_t *src, size_t n, int final) {
    cu_ws *w = cu->ws;
    int lvl = (int8_t)cu->level == -1 ? 6 : (int8_t)cu->level;
    uint32_t nchunks = n == 0 ? 1 : (uint32_t)((n + CU_CHUNK - 1) / CU_CHUNK);
    int32_t err = MZ_OK;
    if (n > 0)
        err = mz_cuda_memcpy_h2d(s->d_in, src, n, s->stream);
    if (err == MZ_OK)
        err = mz_cuda_event_record(s->ev_h2d, s->stream);
    if (err == MZ_OK)
        err = mz_cuda_deflate_chunks(s->d_in, n, CU_CHUNK, NULL, NULL, NULL, nchunks, (final ? MZ_CUDA_FLAG_FINAL : 0) | MZ_CUDA_FLAG_DICT /* one stream: chunks see the 32 KiB before them */, lvl, s->d_slots,
                                     w->slot_stride, s->d_out_len, s->stream);
    if (err == MZ_OK)
        err = mz_cuda_concat(s->d_slots, w->slot_stride, s->d_out_len, nchunks, s->d_offsets, s->d_out, s->stream);
    if (err == MZ_OK && cu->wrap == 2 && n > 0) {
        err = mz_cuda_crc32_segments(s->d_in, n, CU_CHUNK, NULL, NULL, nchunks, s->d_residue, NULL, s->stream);
        if (err == MZ_OK)
            err = mz_cuda_crc32_fold(s->d_residue, nchunks, CU_CHUNK, n, s->d_crc2, s->stream);
        if (err == MZ_OK)
            err = mz_cuda_memcpy_d2h(&s->h_total[1], &s->d_crc2[1], 4, s->stream);
    }
    if (err == MZ_OK)
        err = mz_cuda_memcpy_d2h(&s->h_total[0], s->d_offsets + nchunks, 8, s->stream);
    if (err != MZ_OK)
        return err;
    if (cu->wrap == 1 && n > 0)
        cu_adler_update(cu, src, n); /* zlib framing is unused by minizip-ng callers; host Adler-32 */
    s->n = n;
    s->busy = 1;
    return MZ_OK;
}

/* Wait for a batch, bring its joined stream to the host and hand it to base. In-order by construction. */
static int32_t cu_retire(mz_stream_cuda *cu, cu_slot *s) {
    int32_t err;
    if (!s->busy)
        return MZ_OK;
    s->busy = 0;
    err = mz_cuda_stream_sync(s->stream);
    if (err)
        return err;
    uint64_t total = s->h_total[0];
    if (cu->wrap == 2 && s->n > 0) /* crc(A||B) from crc(A), crc(B), |B| */
        cu->crc = cu->crc_bytes == 0 ? (uint32_t)s->h_total[1] : mz_cuda_crc32_combine(cu->crc, (uint32_t)s->h_total[1], s->n);
    cu->crc_bytes += s->n;
    /* the joined stream comes down in pieces: while base (the caller's thread, usually a memcpy or a file write) takes piece i,
     * piece i+1 is already crossing PCIe */
    const uint64_t piece = 4u << 20;
    const uint64_t np = (total + piece - 1) / piece;
    for (uint64_t i = 0; i < np && i < 2; i++) {
        const uint64_t o = i * piece, k = total - o < piece ? total - o : piece;
        err = mz_cuda_memcpy_d2h(s->h_out + o, s->d_out + o, k, s->stream);
        if (!err) err = mz_cuda_event_record(s->ev_d2h[i & 1], s->stream);
        if (err)
            return err;
    }
    for (uint64_t i = 0; i < np; i++) {
        const uint64_t o = i * piece, k = total - o < piece ? total - o : piece;
        err = mz_cuda_event_sync(s->ev_d2h[i & 1]);
        if (err)
            return err;
        if (i + 2 < np) {
            const uint64_t o2 = (i + 2) * piece, k2 = total - o2 < piece ? total - o2 : piece;
            err = mz_cuda_memcpy_d2h(s->h_out + o2, s->d_out + o2, k2, s->stream);
            if (!err) err = mz_cuda_event_record(s->ev_d2h[i & 1], s->stream);
            if (err)
                return err;
        }
        err = cu_emit(cu, s->h_out + o, k);
        if (err)
            return err;
    }
    return MZ_OK;
}

/* submit the slot being filled and advance the ring; the next slot is the oldest in flight */
static int32_t cu_push(mz_stream_cuda *cu, const uint8_t *src, size_t n, int final) {
    cu_ws *w = cu->ws;
    int32_t err = cu_submit(cu, &w->slot[w->cur], src, n, final);
    if (err != MZ_OK)
        return err;
    w->cur = (w->cur + 1) % CU_NSLOT;
    return cu_retire(cu, &w->slot[w->cur]);
}

static int32_t cu_drain(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    int32_t err = MZ_OK;
    for (int k = 0; k < CU_NSLOT && err == MZ_OK; k++)
        err = cu_retire(cu, &w->slot[(w->cur + k) % CU_NSLOT]); /* cur is the oldest after a push */
    return err;
}
#endif

/* mz_strm_zlib.c:243-264: all-or-error, total_in += size */
int32_t mz_stream_cuda_write(void *stream, const void *buf, int32_t size) {
#ifdef MZ_ZIP_NO_COMPRESSION
    (void)stream; (void)buf; (void)size;
    return MZ_SUPPORT_ERROR;
#else
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    const uint8_t *p = (const uint8_t *)buf;
    int32_t left = size, err;
    if (size < 0)
        return MZ_PARAM_ERROR;
    if (!cu->ws) {
        cu->ws = ws_acquire(1);
        if (!cu->ws) {
            cu->error = MZ_MEM_ERROR;
            return MZ_MEM_ERROR;
        }
    }
    err = cu_write_header(cu);
    if (err != MZ_OK)
        return err;
    /* zero-copy: whole batches straight out of a page-locked caller buffer (no staging memcpy) */
    if (cu->in_len == 0 && (size_t)left >= cu->ws->batch && mz_cuda_host_is_pinned(p)) {
        void *pending[CU_NSLOT];
        int npend = 0;
        while ((size_t)left >= cu->ws->batch) {
            cu_slot *s = &cu->ws->slot[cu->ws->cur];
            if (npend == CU_NSLOT) { /* ring wrapped: the oldest upload of this call is long done */
                memmove(pending, pending + 1, sizeof(void *) * (CU_NSLOT - 1));
                npend--;
            }
            pending[npend++] = s->ev_h2d;
            err = cu_push(cu, p, cu->ws->batch, 0);
            if (err != MZ_OK)
                goto fail;
            p += cu->ws->batch;
            left -= (int32_t)cu->ws->batch;
        }
        /* the caller may reuse its buffer when we return: wait for the uploads (not for the compute) */
        for (int i = 0; i < npend; i++)
            if (mz_cuda_event_sync(pending[i]) != MZ_OK) {
                err = MZ_INTERNAL_ERROR;
                goto fail;
            }
    }
    while (left > 0) {
        cu_slot *s = &cu->ws->slot[cu->ws->cur];
        size_t room = cu->ws->batch - cu->in_len;
        size_t k = (size_t)left < room ? (size_t)left : room;
        cu_copy_out(s->h_in + cu->in_len, p, k); /* (large writes: split over the copy helpers) */
        cu->in_len += k;
        p += k;
        left -= (int32_t)k;
        if (cu->in_len == cu->ws->batch) {
            err = cu_push(cu, s->h_in, cu->in_len, 0);
            cu->in_len = 0;
            if (err != MZ_OK)
                goto fail;
        }
    }
    cu->total_in += size;
    return size;
fail:
    if (err != MZ_WRITE_ERROR)
        cu->error = err;
    return err == MZ_WRITE_ERROR ? err : MZ_DATA_ERROR;
#endif
}

/* ---- read side ------------------------------------------------------------------------------------------ */
#ifndef MZ_ZIP_NO_DECOMPRESSION
/* pull more compressed bytes from base into the pinned window; honours TOTAL_IN_MAX (mz_strm_zlib.c:140-144) */
/* ring position of byte x of the compressed window (x may run past cin_len into the read-ahead bytes) */
static inline size_t cu_ring_pos(const mz_stream_cuda *cu, size_t x) { return (cu->cin_off + x) % cu->ws->ring_cap; }

/* one bounded read from base to ring offset x (relative to the window start): <= 1 MiB like the reference asks in bounded pieces,
 * clipped by TOTAL_IN_MAX and by the end of the ring. Returns bytes read, 0 at the end of base (base_eof is set), < 0 on error. */
static int32_t cu_base_read_at(mz_stream_cuda *cu, size_t x, size_t room) {
    cu_ws *w = cu->ws;
    const size_t p = cu_ring_pos(cu, x);
    int64_t want = (int64_t)room;
    if (want > (1 << 20))
        want = 1 << 20;
    if (want > (int64_t)(w->ring_cap - p))
        want = (int64_t)(w->ring_cap - p);
    if (cu->max_total_in > 0 && want > cu->max_total_in - (int64_t)cu->fed_in)
        want = cu->max_total_in - (int64_t)cu->fed_in;
    if (want <= 0) {
        cu->base_eof = 1;
        return 0;
    }
    int32_t got = mz_abi_base_read(cu->stream.base, w->h_cin + p, (int32_t)want);
    if (got < 0)
        return got;
    if (got == 0) {
        cu->base_eof = 1;
        return 0;
    }
    cu->fed_in += (uint64_t)got;
    return got;
}

/* top the compressed window up: first with the bytes already read ahead (they lie right behind it in the ring), then from base */
static int32_t cu_refill(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    if (cu->ahead_len && cu->cin_len < w->cin_cap) {
        size_t take = w->cin_cap - cu->cin_len;
        if (take > cu->ahead_len)
            take = cu->ahead_len;
        cu->cin_len += take;
        cu->ahead_len -= take;
        cu->cin_dirty = 1;
    }
    while (cu->cin_len < w->cin_cap && !cu->base_eof && cu->ahead_len == 0) {
        int32_t got;
        CU_TIMED(cu, t_base, got = cu_base_read_at(cu, cu->cin_len, w->cin_cap - cu->cin_len));
        if (got < 0)
            return got;
        if (got == 0)
            break;
        cu->cin_len += (size_t)got;
        cu->cin_dirty = 1;
    }
    return MZ_OK;
}

/* While a round is in flight the caller's thread has nothing to do but wait: pull the bytes the NEXT window will need from
 * base meanwhile (into the part of the ring behind the window; the upload of the window in flight is long done -- its round
 * has started). Stops as soon as the round has finished, the ring is full or base is at its end. */
static int32_t cu_read_ahead(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    while (!cu->base_eof && cu->cin_len + cu->ahead_len + 4096 <= w->ring_cap && cu->ahead_len < w->cin_cap) {
        if (!cu->ahead_force && mz_cuda_event_query(w->rev) != 0)
            break;
        int32_t got;
        CU_TIMED(cu, t_ahead, got = cu_base_read_at(cu, cu->cin_len + cu->ahead_len, w->ring_cap - cu->cin_len - cu->ahead_len));
        if (got < 0)
            return got;
        if (got == 0)
            break;
        cu->ahead_len += (size_t)got;
        cu->n_ahead += (uint64_t)got;
    }
    return MZ_OK;
}

/* gzip / zlib framing in front of the raw stream (what inflateInit2's windowBits selects, :97) */
static int32_t cu_parse_header(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    const uint8_t *p = w->h_cin + cu->cin_off; /* the first window starts at the ring's byte 0: contiguous */
    size_t n = cu->cin_len, i;
    if (cu->wrap == 0) {
        cu->hdr_size = 0;
    } else if (cu->wrap == 1) {
        if (n < 2)
            return MZ_BUF_ERROR;
        if ((p[0] & 0x0f) != 8 || (p[0] >> 4) > 7 || (((uint32_t)p[0] << 8) | p[1]) % 31 != 0 || (p[1] & 0x20))
            return MZ_DATA_ERROR;
        cu->hdr_size = 2;
    } else {
        const int32_t err = cu_gzip_parse(p, n, &i);
        if (err != MZ_OK)
            return err;
        cu->hdr_size = (int64_t)i;
    }
    /* drop the framing: the window starts at raw-stream byte 0 */
    cu->cin_off = cu_ring_pos(cu, (size_t)cu->hdr_size);
    cu->cin_len -= (size_t)cu->hdr_size;
    cu->cin_base = 0;
    cu->hdr_parsed = 1;
    memset(w->h_state, 0, sizeof(*w->h_state));
    return mz_cuda_memcpy_h2d(w->d_state, w->h_state, sizeof(*w->h_state), w->rstream);
}

/* A stream that fills the first (small) compressed window is a long one: switch the workspace to big windows and
 * give it the scratch memory of the segment-speculative decoder (K6). Called before the first byte is decoded. */
/* the K6 segment size in bytes, 0 when speculative rounds are off (MZ_CUDA_SPEC=0, or MZ_CUDA_SPEC_SEG_KB below 1 KiB) */
static size_t cu_spec_seg(void) {
    const char *off = getenv("MZ_CUDA_SPEC");
    if (off && off[0] == '0')
        return 0;
    size_t seg = env_size("MZ_CUDA_SPEC_SEG_KB", 16u << 10, 1024);
    return seg < 1024 ? 0 : seg;
}

static void ws_read_upgrade(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    size_t cin_cap = env_size("MZ_CUDA_READ_WINDOW_KB", 128u << 20, 1024);
    size_t seg = cu_spec_seg();
    if (!seg || cin_cap <= w->cin_cap)
        return;
    size_t mult = env_size("MZ_CUDA_READ_OUT_MULT", 4, 1); /* output window = this many compressed windows (tests shrink it) */
    size_t win_cap = 32768 + (mult ? mult : 4) * cin_cap;
    uint32_t max_seg = (uint32_t)(cin_cap / seg) + 1;
    if (max_seg > 12288) /* K6c keeps 16 bytes of shared memory per segment */
        max_seg = 12288;
    const size_t ring_cap = 2 * cin_cap; /* window + as much again read ahead while a round is in flight */
    uint8_t *h_cin = (uint8_t *)mz_cuda_host_alloc(ring_cap + 64);
    uint8_t *d_cin = (uint8_t *)mz_cuda_malloc(cin_cap + 64);
    uint8_t *d_win = (uint8_t *)mz_cuda_malloc(win_cap + 512);
    uint8_t *d_win2 = (uint8_t *)mz_cuda_malloc(win_cap + 512); /* (optional: without it rounds simply wait for the delivery) */
    void *d_spec = mz_cuda_malloc((size_t)mz_cuda_inflate_spec_workspace_bytes(max_seg));
    mz_cuda_spec_summary *h_sum = (mz_cuda_spec_summary *)mz_cuda_host_alloc(sizeof(mz_cuda_spec_summary));
    mz_cuda_spec_summary *d_sum = (mz_cuda_spec_summary *)mz_cuda_malloc(sizeof(mz_cuda_spec_summary));
    if (!h_cin || !d_cin || !d_win || !d_spec || !h_sum || !d_sum) { /* stay small */
        mz_cuda_host_free(h_cin);
        mz_cuda_free(d_cin);
        mz_cuda_free(d_win);
        mz_cuda_free(d_win2);
        mz_cuda_free(d_spec);
        mz_cuda_host_free(h_sum);
        mz_cuda_free(d_sum);
        return;
    }
    {
        const size_t n = cu->cin_len + cu->ahead_len, n1 = n < w->ring_cap - cu->cin_off ? n : w->ring_cap - cu->cin_off;
        memcpy(h_cin, w->h_cin + cu->cin_off, n1);
        memcpy(h_cin + n1, w->h_cin, n - n1);
        memset(h_cin + ring_cap, 0, 64);
        cu->cin_off = 0;
    }
    mz_cuda_host_free(w->h_cin);
    mz_cuda_free(w->d_cin);
    mz_cuda_free(w->d_win);
    mz_cuda_free(w->d_spec); /* the small-window K6 scratch, if a medium stream used this workspace before */
    mz_cuda_host_free(w->h_sum);
    mz_cuda_free(w->d_sum);
    w->h_cin = h_cin;
    w->d_cin = d_cin;
    w->d_win = d_win;
    mz_cuda_free(w->d_win2);
    w->d_win2 = d_win2;
    w->cin_cap = cin_cap;
    w->ring_cap = ring_cap;
    w->win_cap = win_cap;
    w->d_spec = d_spec;
    w->spec_max_seg = max_seg;
    w->spec_seg_bytes = seg;
    w->h_sum = h_sum;
    w->d_sum = d_sum;
    w->large = 1;
}

/* K6 scratch for the current (small) windows: medium streams -- a zip entry of a few megabytes -- are decoded by
 * speculative rounds too, without the big windows of a long stream. Allocated on first use, kept with the workspace. */
static int ws_spec_ensure(cu_ws *w) {
    if (w->d_spec)
        return 1;
    size_t seg = cu_spec_seg();
    if (!seg)
        return 0;
    uint32_t max_seg = (uint32_t)(w->cin_cap / seg) + 1;
    if (max_seg > 12288)
        max_seg = 12288;
    w->d_spec = mz_cuda_malloc((size_t)mz_cuda_inflate_spec_workspace_bytes(max_seg));
    w->h_sum = (mz_cuda_spec_summary *)mz_cuda_host_alloc(sizeof(mz_cuda_spec_summary));
    w->d_sum = (mz_cuda_spec_summary *)mz_cuda_malloc(sizeof(mz_cuda_spec_summary));
    if (!w->d_spec || !w->h_sum || !w->d_sum) {
        mz_cuda_free(w->d_spec);
        mz_cuda_host_free(w->h_sum);
        mz_cuda_free(w->d_sum);
        w->d_spec = NULL;
        w->h_sum = NULL;
        w->d_sum = NULL;
        return 0;
    }
    w->spec_max_seg = max_seg;
    w->spec_seg_bytes = seg;
    return 1;
}

static int32_t cu_crc_fold(mz_stream_cuda *cu, int wait, int one);

/* end of the raw stream: account for consumed bytes, verify the trailer (gzip CRC-32 + ISIZE, zlib Adler-32) */
static int32_t cu_finish_stream(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    mz_cuda_inflate_state *st = w->h_state;
    uint64_t raw_bytes = (st->in_bitpos + 7) >> 3;
    uint64_t tsize = cu->wrap == 2 ? 8 : (cu->wrap == 1 ? 4 : 0);
    int32_t err;
    cu->ended = 1;
    cu->total_in = cu->hdr_size + (int64_t)raw_bytes + (int64_t)tsize;
    if (cu->wrap == 2) {
        err = cu_crc_fold(cu, 1, 0);
        if (err)
            return err;
    }
    if (tsize) {
        size_t off = (size_t)(raw_bytes - cu->cin_base);
        if (off + tsize > cu->cin_len) {
            /* trailer not in the window yet: slide and pull */
            cu->cin_off = cu_ring_pos(cu, off);
            cu->cin_len -= off;
            cu->cin_base += off;
            cu->cin_dirty = 1;
            off = 0;
            err = cu_refill(cu);
            if (err != MZ_OK)
                return err;
            if (tsize > cu->cin_len) {
                cu->total_in = cu->hdr_size + (int64_t)raw_bytes + (int64_t)cu->cin_len;
                return MZ_BUF_ERROR;
            }
        }
        uint8_t t[8];
        for (size_t i = 0; i < (size_t)tsize; i++)
            t[i] = w->h_cin[cu_ring_pos(cu, off + i)];
        if (cu->wrap == 2) {
            uint32_t crc = t[0] | (t[1] << 8) | (t[2] << 16) | ((uint32_t)t[3] << 24);
            uint32_t isz = t[4] | (t[5] << 8) | (t[6] << 16) | ((uint32_t)t[7] << 24);
            if (crc != cu->crc || isz != (uint32_t)st->out_pos)
                return MZ_DATA_ERROR;
        } else {
            uint32_t ad = ((uint32_t)t[0] << 24) | (t[1] << 16) | (t[2] << 8) | t[3];
            if (ad != ((cu->adler_b << 16) | cu->adler_a))
                return MZ_DATA_ERROR;
        }
    }
    return MZ_OK;
}

/* Slide the compressed window to the decoder's position, top it up from base, and make the device copy current.
 * Only called while no round is in flight. */
static int32_t cu_prepare_input(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    mz_cuda_inflate_state *st = w->h_state;
    int32_t err;
    /* keep only bytes at or after the decoder's position (4-byte aligned for the block-start scan) */
    uint64_t pos_byte = (st->in_bitpos >> 3) & ~3ull;
    if (pos_byte > cu->cin_base && (cu->cin_len == w->cin_cap || pos_byte - cu->cin_base >= cu->cin_len / 2)) {
        size_t drop = (size_t)(pos_byte - cu->cin_base);
        if (drop > cu->cin_len)
            drop = cu->cin_len;
        cu->cin_off = cu_ring_pos(cu, drop); /* (a ring: nothing moves) */
        cu->cin_len -= drop;
        cu->cin_base += drop;
        cu->cin_dirty = 1;
    }
    err = cu_refill(cu);
    if (err != MZ_OK)
        return err;
    if (cu->cin_dirty) {
        /* the window, in one or two pieces, and 64 zero bytes behind it (the kernels may read a few bytes past the end) */
        const size_t n1 = cu->cin_len < w->ring_cap - cu->cin_off ? cu->cin_len : w->ring_cap - cu->cin_off;
        err = n1 ? mz_cuda_memcpy_h2d(w->d_cin, w->h_cin + cu->cin_off, n1, w->rstream) : 0;
        if (!err && cu->cin_len > n1) {
            err = mz_cuda_memcpy_h2d(w->d_cin + n1, w->h_cin, cu->cin_len - n1, w->rstream);
            cu->n_wrap += 1;
        }
        if (!err) err = mz_cuda_memcpy_h2d(w->d_cin + cu->cin_len, w->h_cin + w->ring_cap, 64, w->rstream);
        if (err)
            return err;
        cu->cin_dirty = 0;
    }
    return MZ_OK;
}

static inline uint8_t *cu_window(const mz_stream_cuda *cu, int which) { return which ? cu->ws->d_win2 : cu->ws->d_win; }

/* enough compressed input ahead of the decoder for a speculative round to pay off: 4 segments (64 KiB). One warp decodes
 * ~13 MB/s of output, so even the two or three zlib blocks of such a window, decoded side by side, beat the serial decoder;
 * below that the round's seven launches cost more than they save. */
static int cu_spec_worthwhile(const mz_stream_cuda *cu) {
    const cu_ws *w = cu->ws;
    const uint64_t seg = w->spec_seg_bytes ? w->spec_seg_bytes : 16384;
    return (cu->cin_base + cu->cin_len) * 8 > w->h_state->in_bitpos + 8 * 4 * seg;
}

static int cu_spec_eligible(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    const mz_cuda_inflate_state *st = w->h_state;
    return !w->pending && st->status == 0 && st->phase == 0 && st->in_bitpos >= cu->spec_resume_bit && cu_spec_worthwhile(cu) &&
           ws_spec_ensure(w);
}

/* Start one speculative round (K6) over the compressed window, asynchronously on the decode stream. Returns 1 if a
 * round is now in flight, 0 if none was started, < 0 on a CUDA failure. */
static int32_t cu_spec_launch(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    mz_cuda_inflate_state *st = w->h_state;
    const uint64_t bits_avail = (cu->cin_base + cu->cin_len) * 8 - st->in_bitpos;
    const uint64_t seg_bits = (uint64_t)w->spec_seg_bytes * 8;
    const uint64_t out_end = cu->win_base + w->win_cap;
    const uint64_t room = out_end - st->out_pos;
    int32_t err;
    uint64_t nseg = (bits_avail + seg_bits - 1) / seg_bits;
    /* do not scan far more input than the output window can take (the ratio estimate follows the stream) */
    uint64_t fit = (uint64_t)((double)room / (cu->ratio_est * 1.25 * (double)w->spec_seg_bytes)) + 1;
    if (nseg > fit)
        nseg = fit;
    if (nseg > w->spec_max_seg)
        nseg = w->spec_max_seg;
    if (nseg < 2)
        return 0;
    err = mz_cuda_inflate_spec_round(w->d_cin, cu->cin_base, cu->cin_len, cu->base_eof ? 1u : 0u, st->in_bitpos, w->spec_seg_bytes,
                                     (uint32_t)nseg, cu_window(cu, cu->dwin), cu->win_base, st->out_pos, out_end, w->d_spec, w->spec_max_seg, w->d_sum,
                                     w->rstream);
    if (err)
        return err;
    err = mz_cuda_memcpy_d2h(w->h_sum, w->d_sum, sizeof(*w->h_sum), w->rstream);
    if (err)
        return err;
    err = mz_cuda_event_record(w->rev, w->rstream);
    if (err)
        return err;
    w->pending = 1;
    w->pend_nseg = nseg;
    return 1;
}

/* Wait for the round in flight and take its result. Returns 1 if the stream advanced, 0 if the serial decoder has to
 * take the next step, < 0 on a CUDA failure. Stream errors are never decided here. */
static int32_t cu_spec_collect(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    mz_cuda_inflate_state *st = w->h_state;
    const uint64_t seg_bits = (uint64_t)w->spec_seg_bytes * 8;
    int32_t err;
    CU_TIMED(cu, t_round, err = mz_cuda_event_sync(w->rev));
    cu->n_round += 1;
    w->pending = 0;
    if (err)
        return err;
    const mz_cuda_spec_summary *sm = w->h_sum;
    if (getenv("MZ_CUDA_TRACE"))
        fprintf(stderr, "mz_strm_cuda: K6 round at bit %llu: %llu segments, %u guesses, %u proven, %llu bytes out, end bit %llu, status %d, flags %u\n",
                (unsigned long long)st->in_bitpos, (unsigned long long)w->pend_nseg, sm->candidates, sm->nchain, (unsigned long long)sm->total_out,
                (unsigned long long)sm->end_bit, sm->status, sm->flags);
    if (sm->flags || sm->nchain == 0 || (sm->end_bit <= st->in_bitpos && sm->status != 1)) {
        /* nothing proven: let the serial decoder move on; if the window holds no other block start at all
         * (stored or fixed blocks, one giant block), do not try again before it has been consumed */
        cu->spec_resume_bit = sm->candidates <= 1 ? st->in_bitpos + w->pend_nseg * seg_bits : st->in_bitpos + 1;
        return 0;
    }
    const uint64_t used_bytes = (sm->end_bit - st->in_bitpos + 7) >> 3;
    if (used_bytes > 4096)
        cu->ratio_est = (double)sm->total_out / (double)used_bytes < 1.0 ? 1.0 : (double)sm->total_out / (double)used_bytes;
    st->in_bitpos = sm->end_bit;
    st->out_pos += sm->total_out;
    st->blocks += sm->blocks;
    st->status = sm->status;
    st->why = 0;
    st->phase = 0;
    err = mz_cuda_memcpy_h2d(w->d_state, st, sizeof(*st), w->rstream);
    if (err)
        return err;
    if (st->status == 0)
        cu->total_in = cu->hdr_size + (int64_t)(st->in_bitpos >> 3);
    return 1;
}

/* Fold the CRCs of delivered pieces into the running value, oldest first: those whose kernels have finished, or (wait) all of
 * them / (wait && one) just the oldest. */
static int32_t cu_crc_fold(mz_stream_cuda *cu, int wait, int one) {
    cu_ws *w = cu->ws;
    while (w->c_head < w->c_tail) {
        const uint32_t slot = (uint32_t)(w->c_head % CU_CRC_RING);
        if (wait) {
            int32_t err = mz_cuda_event_sync(w->cev[slot]);
            if (err)
                return err;
        } else {
            const int32_t q = mz_cuda_event_query(w->cev[slot]);
            if (q < 0)
                return q;
            if (q == 0)
                break;
        }
        cu->crc = mz_cuda_crc32_combine(cu->crc, w->h_cres[2 * slot + 1], w->clen[slot]); /* crc(v, A) (+) crc(0, B) -> crc(v, A || B) */
        w->c_head++;
        if (one)
            break;
    }
    return MZ_OK;
}

/* the output window about to be written again must not be under a CRC kernel any more: the decode stream waits (on the device,
 * not the caller) for the newest piece's CRC */
static int32_t cu_crc_fence(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    if (w->c_tail == 0 || w->c_tail == w->c_head)
        return MZ_OK;
    return mz_cuda_stream_wait_event(w->rstream, w->cev[(w->c_tail - 1) % CU_CRC_RING]);
}

/* enqueue (on the delivery stream) the download of the next undelivered bytes into h_dec + base; advances deliv_pos */
static int32_t cu_fetch_piece(mz_stream_cuda *cu, size_t base, size_t cap) {
    cu_ws *w = cu->ws;
    const mz_cuda_inflate_state *st = w->h_state;
    int32_t err;
    if (cu->lwin != cu->dwin && cu->deliv_pos >= cu->lwin_end)
        cu->lwin = cu->dwin; /* the old window is empty: it may be decoded into again */
    const int old = cu->lwin != cu->dwin;
    uint64_t n = (old ? cu->lwin_end : st->out_pos) - cu->deliv_pos;
    if (n > cap)
        n = cap;
    const uint8_t *src = cu_window(cu, cu->lwin) + (cu->deliv_pos - (old ? cu->lwin_base : cu->win_base));
    err = mz_cuda_memcpy_d2h(w->h_dec + base, src, n, w->dstream);
    if (err)
        return err;
    if (cu->wrap == 2 && n) { /* the piece's CRC-32, asynchronously on the third stream */
        if (w->c_tail - w->c_head == CU_CRC_RING) {
            err = cu_crc_fold(cu, 1, 1);
            if (err)
                return err;
        }
        const uint32_t slot = (uint32_t)(w->c_tail % CU_CRC_RING);
        const uint32_t nseg = (uint32_t)((n + CU_CRC_SEG - 1) / CU_CRC_SEG);
        uint32_t *res = w->d_cres + (size_t)slot * cu_crc_slot_words(w->batch);
        err = mz_cuda_crc32_segments(src, n, CU_CRC_SEG, NULL, NULL, nseg, res, NULL, w->cstream);
        if (!err) err = mz_cuda_crc32_fold(res, nseg, CU_CRC_SEG, n, res + nseg, w->cstream);
        if (!err) err = mz_cuda_memcpy_d2h(w->h_cres + 2 * slot, res + nseg, 8, w->cstream);
        if (!err) err = mz_cuda_event_record(w->cev[slot], w->cstream);
        if (err)
            return err;
        w->clen[slot] = n;
        w->c_tail++;
    }
    cu->pre_len = (size_t)n;
    cu->deliv_pos += n;
    return MZ_OK;
}

/* Make ws->h_dec[0..dec_len) hold fresh output, or finish the stream. Decoded bytes stay in the device window until
 * they are delivered, at most one host buffer (`batch`) per call; while they are being delivered the next K6 round
 * is already running on the decode stream. */
static int32_t cu_decode_more(mz_stream_cuda *cu) {
    cu_ws *w = cu->ws;
    mz_cuda_inflate_state *st = w->h_state;
    int32_t err;
    if (!cu->hdr_parsed) {
        err = cu_refill(cu);
        if (err != MZ_OK)
            return err;
        err = cu_parse_header(cu);
        if (err != MZ_OK)
            return err;
        cu->cin_dirty = 1;
        if (!w->large && cu->cin_len + (size_t)cu->hdr_size >= w->cin_cap && !cu->base_eof)
            ws_read_upgrade(cu);
    }
    for (;;) {
        /* 1. deliver what is already decoded. h_dec is two halves: the piece the caller is copying out of one half has its
         * successor already crossing PCIe into the other (enqueued before this function returned last time). */
        if (cu->deliv_pos < st->out_pos || cu->pre_len) {
            /* keep the GPU busy meanwhile: if the decoder stands at a block boundary and the output window still has
             * room behind the undelivered bytes, start the next round now */
            if (w->d_spec && w->d_win2 && !w->pending && st->status == 0 && st->phase == 0 && cu->lwin == cu->dwin &&
                cu->win_base + w->win_cap - st->out_pos < w->win_cap / 4) {
                /* no room for another round behind the undelivered bytes, and the other window is idle: carry the last
                 * 32 KiB of history over and decode into it; the delivery drains this window meanwhile */
                const uint64_t have = st->out_pos - cu->win_base, keep = have < 32768 ? have : 32768;
                err = cu_crc_fence(cu); /* (the other window's last pieces may still be under their CRC kernels) */
                if (!err) err = mz_cuda_memcpy_d2d(cu_window(cu, cu->dwin ^ 1), cu_window(cu, cu->dwin) + (have - keep), keep, w->rstream);
                if (err)
                    return err;
                if (cu->trace)
                    fprintf(stderr, "mz_strm_cuda: output window %d full at byte %llu with %llu bytes to deliver: decoding on in window %d\n", cu->dwin,
                            (unsigned long long)st->out_pos, (unsigned long long)(st->out_pos - cu->deliv_pos), cu->dwin ^ 1);
                cu->lwin_base = cu->win_base;
                cu->lwin_end = st->out_pos;
                cu->dwin ^= 1;
                cu->win_base = st->out_pos - keep;
            }
            if (w->d_spec && !w->pending && st->status == 0 && st->phase == 0 &&
                cu->win_base + w->win_cap - st->out_pos >= w->win_cap / 4) {
                err = cu_prepare_input(cu);
                if (err != MZ_OK)
                    return err;
                if (cu_spec_eligible(cu)) {
                    err = cu_spec_launch(cu);
                    if (err < 0)
                        return err;
                }
            }
            const size_t half = w->batch / 2;
            if (!cu->pre_len) { /* nothing in flight: fetch the next piece now */
                cu->dec_base = 0;
                err = cu_fetch_piece(cu, cu->dec_base, half);
                if (err)
                    return err;
            } else {
                cu->dec_base = cu->dec_base ? 0 : half; /* the piece in flight landed in the other half */
            }
            CU_TIMED(cu, t_piece, err = mz_cuda_stream_sync(w->dstream));
            if (err)
                return err;
            const size_t n = cu->pre_len;
            cu->pre_len = 0;
            if (cu->wrap == 2) {
                err = cu_crc_fold(cu, 0, 0);
                if (err)
                    return err;
            }
            if (cu->wrap == 1)
                cu_adler_update(cu, w->h_dec + cu->dec_base, n);
            cu->dec_pos = 0;
            cu->dec_len = n;
            /* and send the piece after it on its way before the caller starts copying this one */
            if (cu->deliv_pos < st->out_pos) {
                err = cu_fetch_piece(cu, cu->dec_base ? 0 : half, half);
                if (err)
                    return err;
            }
            return MZ_OK;
        }
        /* 2. a round in flight: its result decides what comes next */
        if (w->pending) {
            if (w->ring_cap > w->cin_cap && cu->ahead_force >= 0) {
                err = cu_read_ahead(cu);
                if (err < 0)
                    return err;
            }
            err = cu_spec_collect(cu);
            if (err < 0)
                return err;
            if (err == 1)
                continue;
        }
        /* 3. everything delivered: terminal states */
        if (st->status < 0)
            return st->status; /* MZ_DATA_ERROR / MZ_BUF_ERROR, zlib-compatible */
        if (st->status == 1)
            return cu_finish_stream(cu);
        /* 4. decode more */
        err = cu_prepare_input(cu);
        if (err != MZ_OK)
            return err;
        /* slide the output window when little room is left: keep 32 KiB of history at the front */
        uint64_t out_pos = st->out_pos;
        uint64_t need = w->d_spec ? w->win_cap / 2 : 65536;
        if (out_pos - cu->win_base + need > w->win_cap) {
            uint64_t keep = out_pos - cu->win_base < 32768 ? out_pos - cu->win_base : 32768;
            /* cudaMemcpy of overlapping ranges is undefined: with a tiny window (MZ_CUDA_BATCH_KB <= 64) source and
             * destination can overlap, then move front to back in pieces no longer than the gap between them */
            const uint64_t gap = out_pos - cu->win_base - keep;
            err = cu_crc_fence(cu);
            if (err)
                return err;
            for (uint64_t o = 0; gap > 0 && o < keep;) {
                uint64_t k = keep - o;
                if (gap < keep && k > gap)
                    k = gap;
                err = mz_cuda_memcpy_d2d(cu_window(cu, cu->dwin) + o, cu_window(cu, cu->dwin) + gap + o, k, w->rstream);
                if (err)
                    return err;
                o += k;
            }
            cu->win_base = out_pos - keep;
        }
        if (cu_spec_eligible(cu)) {
            err = cu_spec_launch(cu);
            if (err < 0)
                return err;
            if (err == 1)
                continue; /* collected at step 2 */
        }
        w->h_job->d_in = w->d_cin;
        w->h_job->in_base = cu->cin_base;
        w->h_job->in_avail = cu->cin_len;
        w->h_job->d_out = cu_window(cu, cu->dwin);
        w->h_job->out_base = cu->win_base;
        /* at most one host buffer (`batch` bytes) of fresh output per launch */
        w->h_job->out_cap = (out_pos - cu->win_base) + w->batch < w->win_cap ? (out_pos - cu->win_base) + w->batch : w->win_cap;
        w->h_job->in_final = cu->base_eof ? 1u : 0u;
        /* streams that K6 can serve: hand back at the next block boundary so a round can start there */
        w->h_job->flags = w->d_spec && cu_spec_worthwhile(cu) ? MZ_CUDA_INFLATE_STOP_AT_BLOCK : 0u;
        err = mz_cuda_memcpy_h2d(w->d_job, w->h_job, sizeof(*w->h_job), w->rstream);
        if (err)
            return err;
        err = mz_cuda_inflate_streams(w->d_job, w->d_state, 1, w->rstream);
        if (err)
            return err;
        if (getenv("MZ_CUDA_TRACE"))
            fprintf(stderr, "mz_strm_cuda: K5 launch at bit %llu (window %zu bytes, large %d)\n", (unsigned long long)st->in_bitpos, cu->cin_len, w->large);
        err = mz_cuda_memcpy_d2h(st, w->d_state, sizeof(*st), w->rstream);
        if (err)
            return err;
        CU_TIMED(cu, t_serial, err = mz_cuda_stream_sync(w->rstream));
        cu->n_serial += 1;
        if (err)
            return err;
        if (st->status == 0)
            cu->total_in = cu->hdr_size + (int64_t)(st->in_bitpos >> 3);
        if (st->out_pos > out_pos || st->status != 0)
            continue; /* deliver / finish at the top of the loop */
        if (st->why == 1 && cu->base_eof && w->h_job->in_final)
            return MZ_BUF_ERROR; /* decoder wants input that does not exist */
        /* otherwise loop: more input was needed (refill), the window had to slide, or an empty block ended */
    }
}
#endif

/* mz_strm_zlib.c:116-193: bytes produced, 0 at end of stream, negative zlib-compatible code on error */
int32_t mz_stream_cuda_read(void *stream, void *buf, int32_t size) {
#ifdef MZ_ZIP_NO_DECOMPRESSION
    (void)stream; (void)buf; (void)size;
    return MZ_SUPPORT_ERROR;
#else
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    uint8_t *out = (uint8_t *)buf;
    int32_t done = 0;
    if (size < 0)
        return MZ_PARAM_ERROR;
    if (cu->error != 0)
        return cu->error; /* sticky, like zlib->error at :186-189 */
    if (!cu->ws) {
        cu->ws = ws_acquire(2);
        if (!cu->ws) {
            cu->error = MZ_MEM_ERROR;
            return MZ_MEM_ERROR;
        }
    }
    while (done < size) {
        if (cu->dec_pos < cu->dec_len) {
            size_t k = cu->dec_len - cu->dec_pos;
            if (k > (size_t)(size - done))
                k = (size_t)(size - done);
            CU_TIMED(cu, t_copy, cu_copy_out(out + done, cu->ws->h_dec + cu->dec_base + cu->dec_pos, k));
            if (cu->verify_copy && memcmp(out + done, cu->ws->h_dec + cu->dec_base + cu->dec_pos, k) != 0) { /* MZ_CUDA_VERIFY_COPY: debug aid */
                size_t bad = 0;
                while (bad < k && out[done + bad] == cu->ws->h_dec[cu->dec_base + cu->dec_pos + bad])
                    bad++;
                fprintf(stderr, "mz_strm_cuda: VERIFY_COPY mismatch: %zu bytes at output %lld, first bad byte +%zu (dec_base %zu dec_pos %zu dec_len %zu)\n", k,
                        (long long)(cu->total_out + done), bad, cu->dec_base, cu->dec_pos, cu->dec_len);
                memcpy(out + done, cu->ws->h_dec + cu->dec_base + cu->dec_pos, k);
            }
            cu->dec_pos += k;
            done += (int32_t)k;
            continue;
        }
        if (cu->ended)
            break;
        int32_t err = cu_decode_more(cu);
        if (err != MZ_OK) {
            cu->error = err;
            if (cu->dec_pos < cu->dec_len)
                continue; /* deliver what decoded cleanly first; the error surfaces on the next call */
            break;
        }
    }
    if (done == 0 && cu->error != 0)
        return cu->error;
    /* zlib reaches Z_STREAM_END in the call that hands out the last byte, so TOTAL_IN is final and the trailer is checked
     * by then (mz_zip_entry_read_close compares TOTAL_IN with the compressed size right after reading exactly the
     * uncompressed size, mz_zip.c:2100-2128). Do the same: when everything decoded has been delivered and the decoder
     * stands at the end of the stream, finish now instead of on an extra read() call. A bad trailer surfaces on the
     * next call, like every other error that follows cleanly decoded bytes. */
    if (cu->error == 0 && !cu->ended && cu->ws && cu->hdr_parsed && cu->dec_pos == cu->dec_len && !cu->ws->pending &&
        cu->ws->h_state->status == 1 && cu->deliv_pos == cu->ws->h_state->out_pos && cu->pre_len == 0) {
        int32_t ferr = cu_finish_stream(cu);
        if (ferr != MZ_OK)
            cu->error = ferr;
    }
    cu->total_out += done;
    return done;
#endif
}

/* mz_strm_zlib.c:266-278 */
int64_t mz_stream_cuda_tell(void *stream) {
    (void)stream;
    return MZ_TELL_ERROR;
}

int32_t mz_stream_cuda_seek(void *stream, int64_t offset, int32_t origin) {
    (void)stream; (void)offset; (void)origin;
    return MZ_SEEK_ERROR;
}

/* mz_strm_zlib.c:280-305: flush everything pending to base, keep totals readable, MZ_CLOSE_ERROR if an
 * error was latched; like the reference, a failing final flush does not change the return value */
int32_t mz_stream_cuda_close(void *stream) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    if (cu->initialized == 1 && (cu->mode & MZ_OPEN_MODE_WRITE)) {
#ifdef MZ_ZIP_NO_COMPRESSION
        return MZ_SUPPORT_ERROR;
#else
        if (!cu->ws)
            cu->ws = ws_acquire(1);
        if (!cu->ws) {
            cu->error = MZ_MEM_ERROR;
        } else if (cu->error == 0) {
            int32_t err = cu_write_header(cu);
            if (err == MZ_OK) /* what is left (possibly nothing) is the final batch */
                err = cu_push(cu, cu->ws->slot[cu->ws->cur].h_in, cu->in_len, 1);
            cu->in_len = 0;
            if (err == MZ_OK)
                err = cu_drain(cu);
            if (err == MZ_OK && cu->wrap == 2) {
                uint32_t isz = (uint32_t)cu->total_in; /* ISIZE is mod 2^32 */
                uint8_t t[8] = {(uint8_t)cu->crc, (uint8_t)(cu->crc >> 8), (uint8_t)(cu->crc >> 16), (uint8_t)(cu->crc >> 24),
                                (uint8_t)isz,     (uint8_t)(isz >> 8),     (uint8_t)(isz >> 16),     (uint8_t)(isz >> 24)};
                err = cu_emit(cu, t, 8);
            } else if (err == MZ_OK && cu->wrap == 1) {
                uint32_t ad = (cu->adler_b << 16) | cu->adler_a;
                uint8_t t[4] = {(uint8_t)(ad >> 24), (uint8_t)(ad >> 16), (uint8_t)(ad >> 8), (uint8_t)ad};
                err = cu_emit(cu, t, 4);
            }
            if (err != MZ_OK && err != MZ_WRITE_ERROR)
                cu->error = err;
        }
#endif
    } else if (cu->initialized == 1 && (cu->mode & MZ_OPEN_MODE_READ)) {
#ifdef MZ_ZIP_NO_DECOMPRESSION
        return MZ_SUPPORT_ERROR;
#endif
        if (cu->trace)
            fprintf(stderr, "mz_strm_cuda: read side, caller's thread (ms): base reads %.1f (+ %.1f for %llu bytes read ahead under rounds in flight; %llu window uploads wrapped), waiting for speculative rounds %.1f (%llu), "
                            "for serial K5 steps %.1f (%llu), for output pieces %.1f, copying to the caller %.1f; %lld bytes out\n",
                    cu->t_base / 1e6, cu->t_ahead / 1e6, (unsigned long long)cu->n_ahead, (unsigned long long)cu->n_wrap, cu->t_round / 1e6, (unsigned long long)cu->n_round, cu->t_serial / 1e6,
                    (unsigned long long)cu->n_serial, cu->t_piece / 1e6, cu->t_copy / 1e6, (long long)cu->total_out);
    }
    if (cu->ws) {
        ws_release(cu->ws);
        cu->ws = NULL;
    }
    cu->initialized = 0;
    if (cu->error != 0)
        return MZ_CLOSE_ERROR;
    return MZ_OK;
}

/* mz_strm_zlib.c:307-310 */
int32_t mz_stream_cuda_error(void *stream) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    return cu->error;
}

/* mz_strm_zlib.c:312-334 */
int32_t mz_stream_cuda_get_prop_int64(void *stream, int32_t prop, int64_t *value) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    switch (prop) {
    case MZ_STREAM_PROP_TOTAL_IN:
        *value = cu->total_in;
        break;
    case MZ_STREAM_PROP_TOTAL_IN_MAX:
        *value = cu->max_total_in;
        break;
    case MZ_STREAM_PROP_TOTAL_OUT:
        *value = cu->total_out;
        break;
    case MZ_STREAM_PROP_HEADER_SIZE:
        *value = 0;
        break;
    case MZ_STREAM_PROP_COMPRESS_WINDOW:
        *value = cu->window_bits;
        break;
    default:
        return MZ_EXIST_ERROR;
    }
    return MZ_OK;
}

/* mz_strm_zlib.c:336-355 */
int32_t mz_stream_cuda_set_prop_int64(void *stream, int32_t prop, int64_t value) {
    mz_stream_cuda *cu = (mz_stream_cuda *)stream;
    switch (prop) {
    case MZ_STREAM_PROP_COMPRESS_LEVEL:
        if (value == MZ_COMPRESS_LEVEL_DEFAULT)
            cu->level = -1;
        else
            cu->level = (int16_t)value;
        break;
    case MZ_STREAM_PROP_TOTAL_IN_MAX:
        cu->max_total_in = value;
        break;
    case MZ_STREAM_PROP_COMPRESS_WINDOW:
        cu->window_bits = (int32_t)value;
        break;
    default:
        return MZ_EXIST_ERROR;
    }
    return MZ_OK;
}

/* mz_strm_zlib.c:357-365: level default, raw window (zip entries) */
void *mz_stream_cuda_create(void) {
    mz_stream_cuda *cu = (mz_stream_cuda *)calloc(1, sizeof(mz_stream_cuda));
    if (cu) {
        cu->stream.vtbl = &mz_stream_cuda_vtbl;
        cu->level = -1;
        cu->window_bits = -15;
    }
    return cu;
}

/* mz_strm_zlib.c:367-374 */
void mz_stream_cuda_delete(void **stream) {
    mz_stream_cuda *cu = NULL;
    if (!stream)
        return;
    cu = (mz_stream_cuda *)*stream;
    if (cu) {
        if (cu->ws)
            ws_release(cu->ws);
        free(cu);
    }
    *stream = NULL;
}

/* mz_strm_zlib.c:376-378 */
void *mz_stream_cuda_get_interface(void) {
    return (void *)&mz_stream_cuda_vtbl;
}

/* ---- gzip members in device memory (include/mz_cuda_batch.h) ----------------------------------------------------------------
 * The vtbl's framing without its host staging: the member and the plain bytes both stay in device memory. Compress runs K2+K3, K14
 * place and K4 per round straight into the caller's buffer, then K1 and the K14 trailer; decompress runs K5 and K6 over the whole
 * member with the caller's buffer as the one output window, then K1 over the output. */
static inline double cu_ms(uint64_t t0) { return (double)(now_ns() - t0) / 1e6; }

/* one device allocation carved into n pieces, each 256-byte aligned; NULL on failure */
static uint8_t *cu_carve(const size_t *sz, void **out[], int n) {
    size_t total = 0;
    for (int i = 0; i < n; i++)
        total += (sz[i] + 255) & ~(size_t)255;
    uint8_t *p = (uint8_t *)mz_cuda_malloc(total ? total : 256);
    if (!p)
        return NULL;
    size_t o = 0;
    for (int i = 0; i < n; i++) {
        *out[i] = p + o;
        o += (sz[i] + 255) & ~(size_t)255;
    }
    return p;
}

int32_t mz_cuda_gzip_compress_device(const void *d_in, uint64_t len, int16_t level, void *d_out, uint64_t cap, uint64_t *out_len,
                                     mz_cuda_gzip_stats *stats, void *stream) {
    mz_cuda_gzip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    if (!out_len || (!d_in && len))
        return MZ_PARAM_ERROR;
    *out_len = 0;
    if (level == MZ_COMPRESS_LEVEL_DEFAULT)
        level = 6;
    if (level < 0 || level > 9)
        return MZ_PARAM_ERROR;
    if (mz_cuda_init() != MZ_OK) {
        fprintf(stderr, "mz_strm_cuda: no usable sm_90 GPU (%s); there is no CPU fallback\n", mz_cuda_last_error());
        return MZ_SUPPORT_ERROR;
    }
    const uint64_t nch = len ? (len + CU_CHUNK - 1) / CU_CHUNK : 1, last = len - (nch - 1) * CU_CHUNK;
    const uint64_t stride = mz_cuda_deflate_slot_bound(CU_CHUNK);
    if (!d_out) { /* sizing: header, the slot bound of every chunk, trailer */
        *out_len = 10 + (nch - 1) * stride + mz_cuda_deflate_slot_bound((uint32_t)last) + 8;
        return MZ_OK;
    }
    /* rounds: the knob of mz_zip_cuda_write_device; a round's stream bytes must fit K14 place's 32-bit scan (32768 chunks) */
    uint64_t R = ((uint64_t)env_size("MZ_CUDA_ZIP_ROUND_MB", 1024, 1) << 20) / CU_CHUNK;
    if (R < 1)
        R = 1;
    if (R > 32768)
        R = 32768;
    if (R > nch)
        R = nch;
    /* 1. scratch and the chunk table (offsets from d_in, so that every chunk sees the 32 KiB in front of it, across rounds too) */
    uint64_t t0 = now_ns();
    uint64_t *c_off = NULL, *S = NULL, *dst = NULL, *total = NULL;
    uint32_t *c_len = NULL, *olen = NULL, *glen = NULL, *residue = NULL, *crc2 = NULL, *part = NULL;
    uint8_t *c_flags = NULL, *slots = NULL;
    const size_t n = (size_t)nch;
    const size_t sz[12] = {n * 8, n * 4, n, n * 4, n * 4, (n + 1) * 8, n * 8, n * 4, 8, 8, ((size_t)R / MZ_CUDA_ZIP_WR_TILE + 1) * 4, (size_t)R * stride};
    void **pp[12] = {(void **)&c_off, (void **)&c_len, (void **)&c_flags, (void **)&olen, (void **)&glen, (void **)&S, (void **)&dst,
                     (void **)&residue, (void **)&crc2, (void **)&total, (void **)&part, (void **)&slots};
    uint8_t *work = cu_carve(sz, pp, 12);
    uint8_t *h_tab = (uint8_t *)malloc(n * 13);
    void *ev[4] = {NULL, NULL, NULL, NULL};
    int32_t err = work && h_tab ? MZ_OK : MZ_MEM_ERROR;
    for (int i = 0; i < 4 && !err; i++)
        if (!(ev[i] = mz_cuda_event_create()))
            err = MZ_MEM_ERROR;
    if (!err) {
        uint64_t *o = (uint64_t *)h_tab;
        uint32_t *l = (uint32_t *)(h_tab + n * 8);
        uint8_t *f = h_tab + n * 12;
        for (size_t c = 0; c < n; c++) {
            o[c] = (uint64_t)c * CU_CHUNK;
            l[c] = (uint32_t)(c + 1 < n ? CU_CHUNK : last);
            f[c] = (uint8_t)(MZ_CUDA_FLAG_DICT | (c + 1 == n ? MZ_CUDA_FLAG_FINAL : 0u));
        }
        err = mz_cuda_memcpy_h2d(c_off, o, n * 8, stream);
        if (!err) err = mz_cuda_memcpy_h2d(c_len, l, n * 4, stream);
        if (!err) err = mz_cuda_memcpy_h2d(c_flags, f, n, stream);
        if (!err) err = mz_cuda_memset(S, 0, 8, stream);
        if (!err) err = mz_cuda_memset(crc2, 0, 8, stream); /* the CRC of an empty input */
    }
    st.setup_ms = cu_ms(t0);
    /* 2. header (the bytes below cap), rounds, CRC-32 and trailer; one readback at the end */
    if (!err) {
        uint8_t h[10];
        cu_gzip_header(level, h);
        err = mz_cuda_event_record(ev[0], stream);
        if (!err && cap) err = mz_cuda_memcpy_h2d(d_out, h, cap < 10 ? (size_t)cap : 10, stream);
        if (!err) err = mz_cuda_event_record(ev[1], stream);
    }
    for (uint64_t c0 = 0; !err && c0 < nch; c0 += R) {
        const uint32_t m = (uint32_t)(nch - c0 < R ? nch - c0 : R);
        err = mz_cuda_deflate_chunks(d_in, 0, 0, c_off + c0, c_len + c0, c_flags + c0, m, 0, level, slots, stride, olen + c0, stream);
        if (!err) err = mz_cuda_gzip_place(olen, c0, m, S, dst, glen, 10, cap, part, stream);
        if (!err) err = mz_cuda_gather(slots, stride, glen + c0, m, dst + c0, d_out, stream);
        st.rounds++;
    }
    if (!err) err = mz_cuda_event_record(ev[2], stream);
    if (!err && len) err = mz_cuda_crc32_segments(d_in, len, CU_CHUNK, NULL, NULL, (uint32_t)nch, residue, NULL, stream);
    if (!err && len) err = mz_cuda_crc32_fold(residue, (uint32_t)nch, CU_CHUNK, len, crc2, stream);
    if (!err) err = mz_cuda_gzip_trailer(S + nch, crc2 + 1, len, 10, d_out, cap, total, stream);
    if (!err) err = mz_cuda_event_record(ev[3], stream);
    uint64_t exact = 0;
    if (!err) err = mz_cuda_memcpy_d2h(&exact, total, 8, stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    if (!err) {
        st.header_ms = mz_cuda_event_elapsed_ms(ev[0], ev[1]);
        st.work_ms = mz_cuda_event_elapsed_ms(ev[1], ev[2]);
        st.crc_ms = mz_cuda_event_elapsed_ms(ev[2], ev[3]);
        st.bytes_in = len;
        st.bytes_out = exact;
        *out_len = exact;
        if (exact > cap)
            err = MZ_BUF_ERROR;
    }
    mz_cuda_stream_sync(stream); /* (after a failure: nothing of this call is still running when its scratch goes) */
    for (int i = 0; i < 4; i++)
        mz_cuda_event_destroy(ev[i]);
    free(h_tab);
    mz_cuda_free(work);
    if (stats)
        *stats = st;
    return err;
}

int32_t mz_cuda_gzip_decompress_device(const void *d_in, uint64_t len, void *d_out, uint64_t cap, mz_cuda_gzip_result *res,
                                       mz_cuda_gzip_stats *stats, void *stream) {
    mz_cuda_gzip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    if (!res || (!d_in && len) || (!d_out && cap))
        return MZ_PARAM_ERROR;
    memset(res, 0, sizeof(*res));
    if (mz_cuda_init() != MZ_OK) {
        fprintf(stderr, "mz_strm_cuda: no usable sm_90 GPU (%s); there is no CPU fallback\n", mz_cuda_last_error());
        return MZ_SUPPORT_ERROR;
    }
    /* 1. the header: 4 KiB, then more while FEXTRA / FNAME / FCOMMENT run past what was read */
    uint64_t t0 = now_ns();
    size_t hdr = 0, nh = len < 4096 ? (size_t)len : 4096;
    uint8_t *h = NULL;
    int32_t err;
    for (;;) {
        uint8_t *h2 = (uint8_t *)realloc(h, nh ? nh : 1);
        if (!h2) {
            free(h);
            return MZ_MEM_ERROR;
        }
        h = h2;
        err = nh ? mz_cuda_memcpy_d2h(h, d_in, nh, stream) : MZ_OK;
        if (!err) err = mz_cuda_stream_sync(stream);
        if (!err) err = cu_gzip_parse(h, nh, &hdr);
        if (err != MZ_BUF_ERROR || nh == len)
            break;
        nh = len - nh < nh ? (size_t)len : 2 * nh;
    }
    free(h);
    st.header_ms = cu_ms(t0);
    if (err) {
        if (stats)
            *stats = st;
        return err;
    }
    res->header_len = hdr;
    /* 2. scratch; the raw stream (and whatever follows it) copied once, 4-byte aligned with 64 zero bytes behind it */
    t0 = now_ns();
    const uint64_t avail = len - hdr;
    const size_t seg = cu_spec_seg();
    uint32_t max_seg = seg ? (uint32_t)(avail / seg) + 1 : 0;
    if (max_seg > 12288) /* K6c keeps 16 bytes of shared memory per segment */
        max_seg = 12288;
    const uint64_t ncrc = (cap + CU_CHUNK - 1) / CU_CHUNK;
    uint8_t *stage = NULL;
    void *spec = NULL;
    mz_cuda_inflate_job *d_job = NULL;
    mz_cuda_inflate_state *d_state = NULL;
    mz_cuda_spec_summary *d_sum = NULL;
    uint32_t *residue = NULL;
    const size_t sz[6] = {(size_t)avail + 64, seg ? (size_t)mz_cuda_inflate_spec_workspace_bytes(max_seg) : 0, sizeof(*d_job), sizeof(*d_state),
                          sizeof(*d_sum), (size_t)(ncrc + 2) * 4};
    void **pp[6] = {(void **)&stage, &spec, (void **)&d_job, (void **)&d_state, (void **)&d_sum, (void **)&residue};
    uint8_t *work = cu_carve(sz, pp, 6);
    err = work ? MZ_OK : MZ_MEM_ERROR;
    if (!err && avail) err = mz_cuda_memcpy_d2d(stage, (const uint8_t *)d_in + hdr, avail, stream);
    if (!err) err = mz_cuda_memset(stage + avail, 0, 64, stream);
    mz_cuda_inflate_state s;
    memset(&s, 0, sizeof(s));
    if (!err) err = mz_cuda_memcpy_h2d(d_state, &s, sizeof(s), stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    st.setup_ms = cu_ms(t0);
    /* 3. decode: the vtbl's schedule (cu_decode_more) with the caller's buffer as the only output window */
    t0 = now_ns();
    uint64_t resume = 0;
    double ratio = 4.0;
    while (!err && s.status == 0) {
        const int worthwhile = seg && avail * 8 > s.in_bitpos + 8 * 4 * (uint64_t)seg; /* cu_spec_worthwhile */
        if (worthwhile && s.phase == 0 && s.in_bitpos >= resume) {
            const uint64_t seg_bits = (uint64_t)seg * 8;
            uint64_t nseg = (avail * 8 - s.in_bitpos + seg_bits - 1) / seg_bits;
            const uint64_t fit = (uint64_t)((double)(cap - s.out_pos) / (ratio * 1.25 * (double)seg)) + 1;
            if (nseg > fit)
                nseg = fit;
            if (nseg > max_seg)
                nseg = max_seg;
            if (nseg >= 2) {
                mz_cuda_spec_summary sm;
                err = mz_cuda_inflate_spec_round(stage, 0, avail, 1, s.in_bitpos, seg, (uint32_t)nseg, d_out, 0, s.out_pos, cap, spec, max_seg, d_sum, stream);
                if (!err) err = mz_cuda_memcpy_d2h(&sm, d_sum, sizeof(sm), stream);
                if (!err) err = mz_cuda_stream_sync(stream);
                st.k6_rounds++;
                if (err)
                    break;
                if (sm.flags || sm.nchain == 0 || (sm.end_bit <= s.in_bitpos && sm.status != 1)) {
                    resume = sm.candidates <= 1 ? s.in_bitpos + nseg * seg_bits : s.in_bitpos + 1; /* (cu_spec_collect) */
                } else {
                    const uint64_t used = (sm.end_bit - s.in_bitpos + 7) >> 3;
                    if (used > 4096)
                        ratio = (double)sm.total_out / (double)used < 1.0 ? 1.0 : (double)sm.total_out / (double)used;
                    s.in_bitpos = sm.end_bit;
                    s.out_pos += sm.total_out;
                    s.blocks += sm.blocks;
                    s.status = sm.status;
                    s.why = 0;
                    s.phase = 0;
                    err = mz_cuda_memcpy_h2d(d_state, &s, sizeof(s), stream);
                    continue;
                }
            }
        }
        mz_cuda_inflate_job job;
        job.d_in = stage;
        job.in_base = 0;
        job.in_avail = avail;
        job.d_out = d_out;
        job.out_base = 0;
        job.out_cap = cap;
        job.in_final = 1;
        job.flags = worthwhile ? MZ_CUDA_INFLATE_STOP_AT_BLOCK : 0u;
        err = mz_cuda_memcpy_h2d(d_job, &job, sizeof(job), stream);
        if (!err) err = mz_cuda_inflate_streams(d_job, d_state, 1, stream);
        if (!err) err = mz_cuda_memcpy_d2h(&s, d_state, sizeof(s), stream);
        if (!err) err = mz_cuda_stream_sync(stream);
        st.k5_launches++;
        if (!err && s.status == 0 && s.why == 2) {
            res->out_full = 1;
            err = MZ_BUF_ERROR;
        } else if (!err && s.status == 0 && s.why == 1) {
            err = MZ_BUF_ERROR; /* the decoder wants input that does not exist */
        }
    }
    if (!err && s.status < 0)
        err = s.status; /* MZ_DATA_ERROR / MZ_BUF_ERROR, zlib-compatible */
    res->out_len = s.out_pos;
    st.work_ms = cu_ms(t0);
    /* 4. the trailer: CRC-32 of the output (K1 in call scratch) and ISIZE */
    t0 = now_ns();
    if (!err) {
        const uint64_t raw = (s.in_bitpos + 7) >> 3, nseg = (s.out_pos + CU_CHUNK - 1) / CU_CHUNK;
        uint32_t crc2[2] = {0, 0};
        uint8_t t[8];
        if (nseg) err = mz_cuda_crc32_segments(d_out, s.out_pos, CU_CHUNK, NULL, NULL, (uint32_t)nseg, residue, NULL, stream);
        if (!err && nseg) err = mz_cuda_crc32_fold(residue, (uint32_t)nseg, CU_CHUNK, s.out_pos, residue + nseg, stream);
        if (!err && nseg) err = mz_cuda_memcpy_d2h(crc2, residue + nseg, 8, stream);
        if (!err && raw + 8 <= avail) err = mz_cuda_memcpy_d2h(t, stage + raw, 8, stream);
        if (!err) err = mz_cuda_stream_sync(stream);
        if (!err) {
            res->crc = crc2[1];
            if (raw + 8 > avail) { /* the trailer is cut short: TOTAL_IN counts what there is */
                res->in_used = len;
                err = MZ_BUF_ERROR;
            } else {
                const uint32_t tcrc = t[0] | (t[1] << 8) | (t[2] << 16) | ((uint32_t)t[3] << 24);
                const uint32_t isz = t[4] | (t[5] << 8) | (t[6] << 16) | ((uint32_t)t[7] << 24);
                res->in_used = hdr + raw + 8;
                if (tcrc != res->crc || isz != (uint32_t)s.out_pos)
                    err = MZ_DATA_ERROR;
            }
        }
    }
    st.crc_ms = cu_ms(t0);
    mz_cuda_stream_sync(stream);
    mz_cuda_free(work);
    st.bytes_in = res->in_used;
    st.bytes_out = res->out_len;
    if (stats)
        *stats = st;
    return err;
}
