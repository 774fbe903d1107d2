// multiverso-b200 :: C ABI of the sm_90a data-plane library (libmvb200.so).
//
// Every entry point takes raw device pointers + a cudaStream_t (as void*) so the
// Python layer can drive it with torch tensors (tensor.data_ptr(), current stream)
// through ctypes, and a C++ host program can link it directly. All functions
// return 0 on success or a cudaError_t / negative library error; the message is
// available from mvb_last_error().
#pragma once
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVB_MAX_RANKS 8
#define MVB_PAD_CHANNELS 64            /* signal-pad channels per rank           */
#define MVB_PAD_WORDS (MVB_PAD_CHANNELS * MVB_MAX_RANKS)
#define MVB_EPOCH_FIN (1ull << 62)      /* ready-slot value of a worker that finished training */

/* element types */
enum { MVB_F32 = 0, MVB_F64 = 1, MVB_I32 = 2, MVB_I64 = 3, MVB_I8 = 4 };
/* updaters (reference: -updater_type default|sgd|momentum_sgd|adagrad|dcasgd|dcasgda, plus rowwise_adagrad, adam
 * and ftrl).
 * rowwise_adagrad is AdaGrad with one accumulator per (worker, table row): h += mean_j (g_j / lr)^2 over the
 * row's C columns, d_j -= rho * rsqrt(h + 1e-6) * g_j / lr. Its state slab is indexed by local row, not by
 * element, so the entry points that update whole rows take the row length (MvbDenseAdd.num_col,
 * mvb_push_dense_rowwise); mvb_updater_apply and mvb_push_dense_stateful have none and return -2 for it.
 * adam is Adam with per-element moments m, v and one step count t per table row, all shared by every worker. One
 * worker's delta row is one step: t += 1 (it stops at 2^24), then per element g = delta / lr,
 * m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2, d -= rho / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps),
 * with b1 = momentum, b2 = 0.999 and eps = 1e-8 (torch.optim.Adam's step). Its state geometry: m is state0 and v
 * state1, indexed by element (state_stride >= the shard's elements), and t of local row r is state1[state_stride
 * + r], after v's slab; a shard of R rows x C needs 2 round4(R C) + round4(R) elements. Like rowwise_adagrad it
 * needs the row length (mvb_push_dense_adam for the one-sided push) and mvb_updater_apply and
 * mvb_push_dense_stateful return -2 for it.
 * ftrl is FTRL-Proximal (McMahan et al. 2013) with per-element z and n, shared by every worker. With
 * g = delta / lr, alpha = rho, lambda1 = lambda, lambda2 = momentum and beta = 1, one worker's delta is one step per
 * element with g != 0: sigma = g^2 / (alpha (sqrt(n + g^2) + sqrt(n))), z += g - sigma d, n += g^2,
 * d = |z| <= lambda1 ? 0 : (sign(z) lambda1 - z) / ((beta + sqrt(n)) / alpha + lambda2). An element with g == 0
 * keeps d, z and n. Its state geometry is momentum_sgd's with two slabs: z is state0 and n state1, both indexed by
 * element (state_stride >= the shard's elements; a shard of R rows x C needs 2 round4(R C) elements). It is an
 * element-wise updater: mvb_add_dense_fused, mvb_updater_apply, mvb_push_dense_stateful, mvb_add_rows_owner and
 * mvb_rowbox_apply serve it, and mvb_push_dense_rowwise and mvb_push_dense_adam return -2 for it.
 * Integer tables keep the plain add.
 * Code 6 is left unassigned: it is the "unknown updater" of the dispatch tests. */
enum {
  MVB_UPD_DEFAULT = 0,
  MVB_UPD_SGD = 1,
  MVB_UPD_MOMENTUM = 2,
  MVB_UPD_ADAGRAD = 3,
  MVB_UPD_DCASGD = 4,
  MVB_UPD_DCASGDA = 5,
  MVB_UPD_ROWWISE_ADAGRAD = 7,
  MVB_UPD_ADAM = 8,
  MVB_UPD_FTRL = 9
};

/* Same 20-byte layout as the reference AddOption (updater.h:13-69):
 * {worker_id, momentum, learning_rate, rho, lambda}. */
typedef struct MvbAddOpt {
  int worker_id;
  float momentum;
  float lr;
  float rho;
  float lambda;
} MvbAddOpt;

const char* mvb_last_error(void);
int mvb_device_count(void);
int mvb_set_device(int dev);
int mvb_device_info(int dev, int* sms, int* cc_major, int* cc_minor, int64_t* total_mem);

/* ---- symmetric memory (cudaMalloc + cudaIpc) ------------------------------ */
int mvb_symm_alloc(int64_t bytes, void** out_ptr);
int mvb_symm_free(void* ptr);
int mvb_ipc_get_handle(void* ptr, void* handle64 /* 64 bytes */);
int mvb_ipc_open_handle(const void* handle64, void** out_ptr);
int mvb_ipc_close_handle(void* ptr);
int mvb_enable_peer_access(int peer_dev);
int mvb_can_access_peer(int dev, int peer, int* out);
int mvb_memset_async(void* ptr, int value, int64_t bytes, void* stream);
int mvb_memcpy_async(void* dst, const void* src, int64_t bytes, void* stream);
int mvb_stream_sync(void* stream);
int mvb_host_alloc_pinned(int64_t bytes, void** out);
int mvb_host_free_pinned(void* p);
/* plain device memory, streams, events: for hosts without their own CUDA runtime (csrc/device_rt) */
int mvb_device_malloc(int64_t bytes, void** out);
int mvb_device_free(void* p);
int mvb_device_sync(void);
int mvb_stream_create(void** out);
int mvb_stream_destroy(void* stream);
int mvb_event_create(void** out, int timing);
int mvb_event_record(void* event, void* stream);
int mvb_event_sync(void* event);
int mvb_event_elapsed_ms(void* start, void* stop, float* ms);
int mvb_event_destroy(void* event);

/* ---- signal pads / device barrier (K11) ------------------------------------
 * pads[r] = rank r's pad (uint64[MVB_PAD_WORDS]); slot(channel, src) on rank r is
 * written by rank `src`. Epochs are monotonically increasing per channel. */
int mvb_signal(void* const* pads, int me, int world, int channel, uint64_t epoch, void* stream);
int mvb_wait(void* const* pads, int me, int world, int channel, uint64_t epoch,
             uint32_t src_mask, int* err_flag, double timeout_s, void* stream);
int mvb_barrier(void* const* pads, int me, int world, int channel, uint64_t epoch,
                int* err_flag, double timeout_s, void* stream);

/* ---- dense Add / Get (K1, K2) ----------------------------------------------
 * mvb_add_dense_fused: owner-side reduce-scatter + updater. The owner pulls its
 * slice [shard_off, shard_off+shard_len) from each of `nworkers` staging buffers
 * (delta_ptrs[w], full-table sized, peer-mapped) and applies the updater once per
 * worker in worker order, in registers, writing the shard (and state) once.
 * If pads != NULL the kernel first publishes (channel ch_ready) that this rank's
 * staging buffer is complete and waits for all workers in worker_mask, and on
 * completion publishes ch_done (consumed by mvb_get_dense).  */
typedef struct MvbDenseAdd {
  int dtype;              /* MVB_F32 | MVB_F64 | MVB_I32 */
  int updater;            /* MVB_UPD_*                   */
  void* shard;            /* local shard                 */
  void* state0;           /* updater state slab(s)       */
  void* state1;
  int64_t shard_len;      /* elements                    */
  int64_t shard_off;      /* element offset in staging   */
  int64_t state_stride;   /* elements between per-worker state slabs */
  int nworkers;
  uint32_t worker_mask;   /* which workers contribute    */
  const void* delta_ptrs[MVB_MAX_RANKS]; /* indexed by worker id */
  const void* delta_multicast;  /* optional NVLS multicast mapping of the staging buffers:
                                   default/sgd fp32 adds then reduce in the switch */
  MvbAddOpt opts[MVB_MAX_RANKS];         /* per worker          */
  /* fused Add -> Get (optional): push the updated shard into every rank's full-table replica */
  void* replica_ptrs[MVB_MAX_RANKS];     /* indexed by rank, NULL = off */
  void* replica_multicast;               /* NVLS multicast view of the replicas or NULL */
  float scale;            /* delta pre-scale (1 = none)  */
  float clip;             /* |delta| clip, 0 = off       */
  /* fused signalling (optional) */
  void* const* pads;      /* host array[world] of pad pointers or NULL */
  int me, world;
  int ch_ready, ch_done;
  uint64_t epoch;
  int worker_rank[MVB_MAX_RANKS]; /* worker id -> rank (for flag slots) */
  int is_worker;          /* this rank publishes ch_ready             */
  int* err_flag;          /* device int, set on watchdog timeout      */
  int* fin_flag;          /* device int, set to 1 when every worker has finished */
  unsigned int* done_counter; /* device uint, zero-initialised         */
  double timeout_s;
  /* per-worker AddOptions through symmetric memory (optional): opt_box[r] = rank r's option box
     (2 x MVB_MAX_RANKS MvbAddOpt, peer mapped).  The calling worker publishes opts[my_worker] in every
     owner's box before its ready flag; owners apply worker w's delta with worker w's published option.
     NULL boxes: opts[] are used as given (single process / identical options).                       */
  void* opt_box[MVB_MAX_RANKS];
  int my_worker;          /* this rank's worker id (-1: not a worker)  */
  /* row length of the table; read by row-state updaters only (rowwise_adagrad, adam), which need num_col >= 1,
     shard_len % num_col == 0 and state_stride >= shard_len / num_col (rowwise_adagrad: its slabs hold one
     element per local row) or state_stride >= shard_len (adam: element slabs, then the step counts), else
     MVB_BAD_ROW_MAP before any CUDA call. */
  int64_t num_col;
} MvbDenseAdd;
int mvb_add_dense_fused(const MvbDenseAdd* a, void* stream);

/* Local (single-source) updater apply: the stand-alone K9 kernel used by the
 * NCCL comparator path and by row-wise / whole adds with one worker. Element-wise updaters only, ftrl included
 * (-2 for rowwise_adagrad and adam, which need rows). */
int mvb_updater_apply(int dtype, int updater, void* data, const void* delta, void* state0,
                      void* state1, int64_t n, const MvbAddOpt* opt, float scale, void* stream);

/* mvb_get_dense: all-gather by pull. shard_ptrs[s] = server s's shard (peer-mapped),
 * shard_offs[s]/shard_lens[s] in elements, out = local full-size buffer. If pads
 * != NULL waits for ch_done >= epoch from every server rank first. */
typedef struct MvbDenseGet {
  int dtype;
  void* out;
  int nservers;
  const void* shard_ptrs[MVB_MAX_RANKS];
  int64_t shard_offs[MVB_MAX_RANKS];
  int64_t shard_lens[MVB_MAX_RANKS];
  void* const* pads;
  int me, world;
  int ch_done;
  uint64_t epoch;
  int server_rank[MVB_MAX_RANKS];
  int* err_flag;
  double timeout_s;
} MvbDenseGet;
int mvb_get_dense(const MvbDenseGet* g, void* stream);

/* One-sided async push: red.add of (sign * delta[shard range]) into every owner's
 * shard through the peer mapping. Stateless updaters only (default: +, sgd: -).
 * Both one-sided pushes return -3 for nservers outside [1, MVB_MAX_RANKS], before any CUDA call. */
int mvb_push_dense_red(int dtype, const void* delta, int nservers, void* const* shard_ptrs,
                       const int64_t* shard_offs, const int64_t* shard_lens, float sign,
                       void* stream);

/* One-sided async push for STATEFUL updaters: remote read-modify-write of the owners' shard +
 * state slabs (state must be peer-mapped). Per-worker state is exact; data is Hogwild, and so is the shared state
 * of momentum_sgd and ftrl (exact for one pusher). f32 / f64 and the momentum, AdaGrad, DC-ASGD, DC-ASGD-A and ftrl
 * updaters only (-1 / -2 otherwise). */
int mvb_push_dense_stateful(int dtype, int updater, const void* delta, int nservers,
                            void* const* shard_ptrs, void* const* state0_ptrs, void* const* state1_ptrs,
                            const int64_t* shard_offs, const int64_t* shard_lens,
                            const int64_t* state_strides, const MvbAddOpt* opt, int me, void* stream);
/* The same push for row-state updaters (rowwise_adagrad): one warp per row of num_col elements reduces the
 * worker's delta row, read-modify-writes the worker's accumulator of that row at the owner (state_ptrs[s] +
 * opt->worker_id * state_strides[s] + local row) and red.adds the step into the owner's row. Returns -3 for
 * nservers outside [1, MVB_MAX_RANKS], -1 for element types other than f32 / f64, -2 for updaters without row
 * state and MVB_BAD_ROW_MAP when num_col < 1, a shard_lens[s] is not a multiple of num_col or a
 * state_strides[s] is below shard_lens[s] / num_col; all before any CUDA call. */
int mvb_push_dense_rowwise(int dtype, int updater, const void* delta, int nservers, void* const* shard_ptrs,
                           void* const* state_ptrs, const int64_t* shard_offs, const int64_t* shard_lens,
                           const int64_t* state_strides, int64_t num_col, const MvbAddOpt* opt, int me,
                           void* stream);
/* The same push for adam: per row of num_col elements, the owner's step count of the row (state1_ptrs[s] +
 * state_strides[s] + local row) is counted atomically, so concurrent pushers each count their step; the owner's
 * m (state0_ptrs[s]) and v (state1_ptrs[s]) elements are read-modify-written (Hogwild across concurrent pushers,
 * exact for one) and the step is red.added into the owner's row. A row of C elements runs on the power of two
 * lanes >= C up to a warp. Returns -3 for nservers outside [1, MVB_MAX_RANKS], -1 for element types other than
 * f32 / f64, -2 for updaters other than adam and MVB_BAD_ROW_MAP when num_col < 1, a shard_lens[s] is not a
 * multiple of num_col or a state_strides[s] is below shard_lens[s]; all before any CUDA call. */
int mvb_push_dense_adam(int dtype, int updater, const void* delta, int nservers, void* const* shard_ptrs,
                        void* const* state0_ptrs, void* const* state1_ptrs, const int64_t* shard_offs,
                        const int64_t* shard_lens, const int64_t* state_strides, int64_t num_col,
                        const MvbAddOpt* opt, int me, void* stream);

/* ---- row-sparse Get / Add (K3, K4, K10) ------------------------------------ */
/* Server min(r / rows_per_server, nservers - 1) holds row r, at local index r - server * rows_per_server.
 * Every entry point that takes a row map, directly or inside another descriptor, needs
 * 1 <= nservers <= MVB_MAX_RANKS and rows_per_server >= 1, and checks it before any CUDA call. A map that
 * fails returns MVB_BAD_ROW_MAP, except from the entry points with an older code of their own:
 * mvb_get_gemm_fused -33, mvb_topk_cosine and mvb_full_softmax -41, mvb_embedding_bag_* -50 and
 * mvb_sgns_train_win -21. The mvb_keys_* entry points check their MvbKeyMap in the same way. */
enum { MVB_BAD_ROW_MAP = -70 };
typedef struct MvbRowMap {
  int64_t num_row, num_col;
  int nservers;
  int64_t rows_per_server;            /* reference rule: num_row / nservers      */
  void* shard_ptrs[MVB_MAX_RANKS];    /* server s shard base (rows [s*rps, ...)) */
} MvbRowMap;
int mvb_get_rows(int dtype, const MvbRowMap* m, const int64_t* row_ids, int64_t k, void* out,
                 int64_t out_ld, void* stream);
int mvb_add_rows_red(int dtype, const MvbRowMap* m, const int64_t* row_ids, int64_t k,
                     const void* vals, int64_t vals_ld, float sign, void* stream);
/* fused AddDeltaParameter: red.add of (cur - old) * scale per row (fp32, num_col % 4 == 0, ld % 4 == 0,
 * cur and old 16-byte aligned, else -9); the same kernel as mvb_rows_push_delta */
int mvb_add_rows_delta(const MvbRowMap* m, const int64_t* row_ids, int64_t k, const float* cur,
                       const float* old, int64_t ld, float scale, void* stream);
/* Stateful row add applied by the OWNER on its local shard for rows in its range:
 * ids/vals may be another rank's (peer-mapped) staging.  A repeated row is updated once per
 * occurrence, in list order, when its occurrences are adjacent (sort the request stably by id);
 * occurrences that are not adjacent race. rowwise_adagrad indexes its state slab by local row
 * (state_stride >= row_hi - row_lo). adam indexes m and v by element and keeps the step counts after v's slab
 * (state_stride >= (row_hi - row_lo) * num_col, else MVB_BAD_ROW_MAP before any CUDA call); a repeated row
 * counts one step per occurrence. ftrl indexes z and n by element like momentum_sgd; a repeated row is one step
 * per occurrence. */
int mvb_add_rows_owner(int dtype, int updater, void* shard, void* state0, void* state1,
                       int64_t row_lo, int64_t row_hi, int64_t num_col, int64_t state_stride,
                       const int64_t* row_ids, int64_t k, const void* vals, int64_t vals_ld,
                       const MvbAddOpt* opt, void* stream);
int mvb_row_nonzero_mask(int dtype, const void* data, int64_t rows, int64_t cols, int64_t ld,
                         uint8_t* mask, void* stream);
/* stale-row bitmap (T4/T5 delta-pull): mark rows stale for all workers / query+clear */
int mvb_stale_mark(uint8_t* stale /*[workers][rows]*/, int64_t rows, int nworkers,
                   const int64_t* row_ids, int64_t k /* k<0: all rows */, void* stream);
int mvb_stale_take(uint8_t* stale_w /*[rows] for one worker*/, int64_t rows,
                   const int64_t* row_ids, int64_t k, uint8_t* out_mask, void* stream);
/* ascending positions of the non-zero bytes of a mask; *count on the device */
int mvb_mask_compact(const uint8_t* mask, int64_t n, int64_t* out_ids, int64_t* count, void* stream);

/* ---- KV hash table (K5) ----------------------------------------------------- */
/* open addressing, keys int64 (empty = INT64_MIN), values 8 bytes (f64 or i64) or 4
 * bytes (f32 / i32). Owner of key = mod(key, nservers). */
typedef struct MvbKV {
  int vtype;                       /* MVB_F32|MVB_F64|MVB_I32|MVB_I64 */
  int nservers;
  int64_t capacity;                /* slots per shard (power of two)  */
  void* keys[MVB_MAX_RANKS];       /* int64[capacity] per server      */
  void* vals[MVB_MAX_RANKS];
} MvbKV;
int mvb_kv_init(void* keys, int64_t capacity, void* stream);
/* growth: live keys of a shard; re-insertion of a shard into a larger (initialised) local table */
int mvb_kv_count(const void* keys, int64_t capacity, int64_t* out_count, void* stream);
int mvb_kv_rehash(int vtype, const void* old_keys, const void* old_vals, int64_t old_cap, void* new_keys,
                  void* new_vals, int64_t new_cap, int* err_flag, void* stream);
/* mvb_kv_add and mvb_kv_get return -3 for nservers outside [1, MVB_MAX_RANKS] and -4 for a capacity that is not
 * a power of two >= 1 (mvb_kv_rehash: -4 for such a new_cap), before any CUDA call. INT64_MIN is not a key:
 * mvb_kv_add skips it and sets *err_flag = 5003, mvb_kv_get returns 0 for it. A key with no free slot on its
 * probe chain sets *err_flag = 5001 (5002 in mvb_kv_rehash). */
int mvb_kv_add(const MvbKV* kv, const int64_t* keys, const void* vals, int64_t n, int* err_flag,
               void* stream);
int mvb_kv_get(const MvbKV* kv, const int64_t* keys, void* out_vals, int64_t n, void* stream);
int mvb_kv_dump(int vtype, const void* keys, const void* vals, int64_t capacity,
                int64_t* out_keys, void* out_vals, int64_t* out_count, void* stream);

/* ---- hash index of a HashMatrixTable (hash_rows.cu) ---------------------------------------------------- */
/* Rows keyed by any int64 except INT64_MIN. Server s = mod(key, nservers) owns the key; it has `slots` (P, a
 * power of two) slots, probed linearly from mix64(key) & (P - 1). Slot j of server s is row s P + j of an fp32
 * MatrixTable of nservers P + 1 rows (row pitch % 4 == 0); the last row is the zero row, never given to a key.
 * A server holds at most floor(7 P / 8) keys. keys / ready / count are symmetric (peer-mapped) allocations. */
enum { MVB_HASH_INIT_CONST = 0, MVB_HASH_INIT_UNIFORM = 1 };
enum { MVB_HASH_FULL = 1, MVB_HASH_TIMEOUT = 2, MVB_HASH_BAD_KEY = 3 };
typedef struct MvbHashRows {
  int nservers;
  int64_t slots;                   /* P per server                                                          */
  void* keys[MVB_MAX_RANKS];       /* int64[P] per server, INT64_MIN = empty                                */
  void* ready[MVB_MAX_RANKS];      /* uint32[P] per server: 1 once the slot's row holds its initial value,
                                      2 for a key refused at the limit (it keeps the slot, never a row)     */
  void* count[MVB_MAX_RANKS];      /* uint64 per server: live keys (ready == 1)                             */
  MvbRowMap map;                   /* the rows                                                              */
  int init;                        /* MVB_HASH_INIT_CONST: init_value; UNIFORM: lo + u (hi - lo), u from the key */
  float init_value, lo, hi;
  uint64_t seed;
  /* access clock (optional): a lookup that inserts stamps each key it finds or inserts with
     last_seen[j] = max(last_seen[j], *clock); lookups that do not insert stamp nothing                    */
  void* last_seen[MVB_MAX_RANKS];  /* int64[P] per server, symmetric, or NULL: not tracked (clock unused)   */
  const int64_t* clock;            /* device int64 of the calling rank; needed when last_seen is set        */
  /* count-based admission (optional; admit_after < 2, as in a zeroed descriptor, is off): an inserting lookup
     gives a missing key a slot only once the key's count-min estimate at its owner is >= admit_after        */
  void* sketch[MVB_MAX_RANKS];     /* uint32[4 width] per server, symmetric: row r's counters at r width    */
  void* total[MVB_MAX_RANKS];      /* uint64 per server, symmetric: occurrences counted since the last aging */
  void* age;                       /* device uint32[MVB_MAX_RANKS] of the calling rank: mvb_hash_rows_age's
                                      scratch                                                               */
  int64_t width;                   /* W counters per sketch row, a power of two in [2, 2^31]; aging at W / 2 */
  int admit_after;                 /* n                                                                     */
} MvbHashRows;
typedef struct MvbHashLookup {
  const MvbHashRows* tables;       /* device [T] index descriptors                                          */
  const int64_t* keys;             /* [n]                                                                   */
  int64_t n;
  const int64_t* seg_end;          /* device [G]: key i belongs to the first segment g with i < seg_end[g];
                                      NULL: every key belongs to table 0                                    */
  const int* seg_table;            /* device [G]: the descriptor of segment g, or -1: the key is a row id,
                                      copied unchanged                                                       */
  int G;
  int insert;                      /* 1: a missing key claims a slot; 0: it reads the zero row              */
  const int64_t* insert_ok;        /* device int64 or NULL: when it holds 0, insert is treated as 0 (the
                                      caller's device-side check of the segment layout failed)              */
  int64_t* rows;                   /* [n] out                                                               */
  int64_t* status;                 /* device int64, 0 on entry; the first error as kind << 40 | table << 8 | server */
  double timeout_s;                /* watchdog of the wait for a slot another thread is initialising        */
  int admit;                       /* 1: some descriptor of the call has admission on: a count pass runs
                                      before the translation; 0: it is not launched                         */
} MvbHashLookup;
/* empty keys, zero ready flags and counter of one server's index */
int mvb_hash_rows_init(void* keys, void* ready, void* count, int64_t slots, void* stream);
/* Admission. With a->admit set and the lookup inserting (insert and *insert_ok != 0), a count pass runs first:
 * every occurrence of a key of a descriptor with admission on that holds no slot at its owner (no key in its probe
 * chain: ready, being initialised or refused keys hold one) adds 1 to its 4 counters
 * sketch[s][r W + ((hash64(key + (r + 1) 0x9E3779B97F4A7C15) >> 32) & (W - 1))], r = 0..3, and to total[s]
 * (system-scope atomics, peers included). The translation then gives such a key a slot only when its estimate, the
 * minimum of its 4 counters, is >= admit_after; otherwise it reads the zero row, sets no status and takes nothing.
 * All occurrences of a call are counted before any is admitted, so on one rank every occurrence of a key in a call
 * gets the same row. Counts of other ranks landing during the translation can admit a key in the middle of a call:
 * an occurrence may then read the zero row in the call in which another occurrence got the slot. */
int mvb_hash_rows_lookup(const MvbHashLookup* a, void* stream);
/* Aging step of an index with admission (run after each inserting lookup): every server whose total is >= W / 2
 * has its total and all its counters shifted right by the smallest k that takes the total below W / 2. One CAS on
 * the total elects the one caller that shifts a server, and each counter is shifted by a CAS loop, so a count
 * landing concurrently is never lost (it is shifted or kept whole). Returns, before any CUDA call, -3 / -4 as
 * mvb_hash_rows_mark, -7 for admit_after < 2, -8 for a width not a power of two in [2, 2^31], -9 for a NULL age,
 * sketch[s] or total[s] (s < nservers). */
int mvb_hash_rows_age(const MvbHashRows* h, void* stream);
/* *out = live keys over all servers of the (host) descriptor */
int mvb_hash_rows_count(const MvbHashRows* h, int64_t* out, void* stream);
/* (key, row) of every live slot (ready == 1) of server `server`, in no particular order; *out_count on the device */
int mvb_hash_rows_dump(const MvbHashRows* h, int server, int64_t* out_keys, int64_t* out_rows, int64_t* out_count,
                       void* stream);
/* Eviction. Both calls need every lookup of the index to have completed on every rank (run them between barriers).
 * mvb_hash_rows_mark: a translation without insert of keys[0, n) that sets ready[j] = 3 ("marked") at the owner of
 * every live key found (peer stores included). Missing keys and INT64_MIN are ignored.
 * mvb_hash_rows_evict: rebuilds server `server`'s index in place (run by the rank holding it). It removes the marked
 * and refused slots and, unless older_than is INT64_MIN, the live keys with last_seen < older_than. The survivors
 * are placed by the in-place rehash: the index is cut into clusters (maximal runs of non-empty slots, wrapping
 * P - 1 -> 0), each walked from its first slot; a victim is cleared, a survivor moves to the first empty slot
 * probing from its home, or stays. A survivor carries its row (num_col floats), its updater state rows and
 * last_seen. The state is nst = (state0 != NULL) + (state1 != NULL) arrays of n_slabs fp32 slabs state_stride
 * elements apart, slot j owning elements [j state_row, (j + 1) state_row) of each slab. Every slot left empty
 * holds zero state and last_seen 0; its row is left as it was. An index without an empty slot first loses its
 * lowest victim slot by a sequential backward-shift deletion (one warp), then is walked as one cluster. The zero row
 * is never touched. counts: device int64[2] out, {live keys removed, survivors moved}; the server's count drops by
 * counts[0]. work: device int64[slots / 2 + 2] scratch.
 * Returns, before any CUDA call: -3 for nservers outside [1, MVB_MAX_RANKS], -1 for a server outside
 * [0, nservers), -4 for slots not a power of two in [2, 2^31], MVB_BAD_ROW_MAP for a map that fails the row map
 * rule, disagrees with nservers, has rows_per_server < slots or num_col not a positive multiple of 4, -5 for
 * older_than != INT64_MIN without last_seen[server], -6 for a state description with n_slabs < 1, state_row < 1
 * or n_slabs > 1 and state_stride < slots * state_row. mvb_hash_rows_mark returns -3 and -4 alike.
 * mvb_hash_rows_evict_ex also moves and clears a third state slab with its own row length: slot j owns elements
 * [j state2_row, (j + 1) state2_row) of state2 (adam's step counts: state2 = v's array + state_stride,
 * state2_row = 1). It returns -6 for state2 != NULL with state2_row < 1; with state2 NULL it is
 * mvb_hash_rows_evict. */
int mvb_hash_rows_mark(const MvbHashRows* h, const int64_t* keys, int64_t n, void* stream);
int mvb_hash_rows_evict(const MvbHashRows* h, int server, int64_t older_than, void* state0, void* state1,
                        int n_slabs, int64_t state_stride, int64_t state_row, int64_t* counts, int64_t* work,
                        void* stream);
int mvb_hash_rows_evict_ex(const MvbHashRows* h, int server, int64_t older_than, void* state0, void* state1,
                           int n_slabs, int64_t state_stride, int64_t state_row, int64_t* counts, int64_t* work,
                           void* stream, void* state2, int64_t state2_row);

/* ---- all-reduce (K6) --------------------------------------------------------- */
/* One-shot P2P: every rank reads all peers' symmetric buffers and reduces locally
 * in fixed rank order (deterministic, identical on all ranks). Two-shot: reduce own
 * slice, then write it to every peer. In-kernel signalling on channels ch..ch+1. */
typedef struct MvbAllreduce {
  int dtype;
  int64_t n;
  void* bufs[MVB_MAX_RANKS];    /* symmetric staging, peer-mapped */
  void* out;                    /* local result, any element alignment (may alias bufs[me] for two-shot) */
  void* const* pads;
  int me, world;
  int ch;
  uint64_t epoch;
  int* err_flag;
  unsigned int* done_counter;
  double timeout_s;
} MvbAllreduce;
int mvb_allreduce_oneshot(const MvbAllreduce* a, void* stream);
int mvb_allreduce_twoshot(const MvbAllreduce* a, void* stream);
/* latency path: stage-in from `src`, handshake on channel a->ch (ready only) and one-shot reduction in
 * ONE launch; bufs[r] + slot_off_bytes is the epoch's half of a double-buffered staging area */
int mvb_allreduce_fused(const MvbAllreduce* a, const void* src, int64_t slot_off_bytes, void* stream);
/* NVLS: in-switch reduction through the multicast mapping of the staging buffers (fp32) */
int mvb_allreduce_nvls(const MvbAllreduce* a, void* multicast_ptr, void* stream);

/* ---- WordEmbedding (K7) -------------------------------------------------------- */
typedef struct MvbSgns {
  const int* tokens;         /* word ids, <0 = sentence break            */
  int64_t n_tokens;
  float* w_in;               /* input embeddings  [rows x ld]             */
  float* w_out;              /* output embeddings [rows x ld]             */
  float* g2_in;              /* AdaGrad G^2 (or NULL)                     */
  float* g2_out;
  int dim;
  int64_t ld;
  int window;
  int negative;              /* K (0 when hs)                             */
  int cbow;                  /* 0 skip-gram, 1 cbow                       */
  int hs;                    /* hierarchical softmax                      */
  int use_adagrad;
  float lr;
  /* negative sampling: alias table over vocab (prob,alias), or an explicit pool */
  const float* alias_prob;
  const int* alias_idx;
  int vocab;
  const int* neg_pool;
  int neg_pool_size;
  /* hierarchical softmax: per word path [codelen<=MVB_MAX_CODE] */
  const int* hs_points;      /* [vocab x max_code] inner-node row ids      */
  const int8_t* hs_codes;    /* [vocab x max_code]                         */
  const int* hs_len;         /* [vocab]                                    */
  int hs_max_code;
  /* optional global-id -> local-slot maps (block mode); NULL = identity   */
  const int* map_in;
  const int* map_out;
  uint64_t seed;
  float* loss_sum;           /* optional: += sum of -log sigma(..)         */
  unsigned long long* pair_count;  /* optional: += trained (input,target) samples */
  int hogwild;               /* one device, skip-gram + NS: 0 = deterministic waves, 1 = the Hogwild
                                window-batched kernel (one centre per warp)                          */
  /* optional per-WORD step scales in (0,1] (deterministic and window kernels): caps the summed step of
     the Zipf-head rows that collect more concurrent stale updates than plain SGD tolerates;
     NULL = 1 everywhere                                                                              */
  const float* scale_in;
  const float* scale_out;
  const int* neg_pool_size_ptr;  /* optional: pool size read on the DEVICE (mvb_we_prepare counts[2]);
                                    deterministic and window kernels, overrides neg_pool_size.  An input
                                    that routes elsewhere (K >= 8, CBOW, HS, AdaGrad, register-kernel
                                    shapes) makes mvb_sgns_train return -23 before any CUDA call       */
  /* direct mode (nservers > 1, window kernel only): train IN the row-sharded tables over NVLink -- rows
     are loaded from and reduced into their owners' shards (owner = id / rows_per_server, last server takes the
     remainder) through the peer mappings; no block cache, no maps (Hogwild across GPUs)                 */
  int nservers;
  int64_t rows_per_server;
  void* w_in_peers[MVB_MAX_RANKS];
  void* w_out_peers[MVB_MAX_RANKS];
} MvbSgns;
int mvb_sgns_train(const MvbSgns* a, void* stream);
int mvb_sgns_train_win(const MvbSgns* a, void* stream);   /* window-batched TMA pipeline      */
int mvb_sgns_train_det(const MvbSgns* a, void* stream);   /* deterministic waves (default)    */
int mvb_sgns_last_launches(void);   /* kernel launches of the last mvb_sgns_train call */
int mvb_sgns_win_inflight(int dim, int negative, int window);  /* centre positions in flight; 0 outside
                                                                  1 <= negative <= 7                     */
/* ---- key-addressed shards for application-defined tables (keys.cu): the device-side extension point ---- */
typedef struct MvbKeyMap {
  int64_t size;                        /* keys 0 .. size-1                                   */
  int64_t per_server;                  /* size / nservers, the last server takes the remainder */
  int nservers;
  int width;                           /* fp32 values per key (SparseTable 1, FTRLTable 2)    */
  void* shard_ptrs[MVB_MAX_RANKS];     /* server s: [keys of s x width] fp32, peer mapped      */
  void* touched_ptrs[MVB_MAX_RANKS];   /* server s: touched bitmap uint32[ceil(keys of s / 32)] */
} MvbKeyMap;
/* all three return -8 for a width outside [1, 16] before any CUDA call */
int mvb_keys_add(const MvbKeyMap* m, const int64_t* keys, const float* vals, int64_t n, float sign, void* stream);
int mvb_keys_get(const MvbKeyMap* m, const int64_t* keys, float* out, int64_t n, void* stream);
int mvb_keys_collect(const MvbKeyMap* m, int64_t* out_keys, float* out_vals, int64_t* count, int64_t cap,
                     void* stream);

/* ---- staleness instrumentation: per-shard version counters (symmetric memory), bumped by every Add,
   recorded by every Get; staleness of an Add = other workers' Adds applied since this worker's last Get */
int mvb_stale_on_add(void* const* version_ptrs, int nservers, unsigned long long* last_get,
                     unsigned int* adds_since, unsigned long long* hist, int nbins, void* stream);
int mvb_stale_on_get(void* const* version_ptrs, int nservers, unsigned long long* last_get,
                     unsigned int* adds_since, void* stream);

/* ---- row mailboxes (rowbox.cu): device-side row Add with owner-side apply ------------- */
typedef struct MvbRowBox {
  MvbRowMap map;             /* the table's shards (fp32, num_col % 4 == 0, every rank worker + server)   */
  int me;                    /* my rank == worker id == server id                                     */
  int64_t cap;               /* entries per (owner, source) slot: the rows of the largest shard         */
  int64_t slot_bytes;        /* mvb_rowbox_slot_bytes(cap, num_col)                                    */
  void* box[MVB_MAX_RANKS];  /* rank r's mailbox slab: nservers x mvb_rowbox_slots() slots, peer mapped */
  void* ack[MVB_MAX_RANKS];  /* rank r's ack array uint64[nservers], peer mapped                       */
  int* seg;                  /* device scratch int[nservers + 1]                                       */
  unsigned int* done;        /* device scratch uint[2], zero-initialised                               */
  uint64_t* applied;         /* device uint64[nservers], zero-initialised: epochs applied per source   */
  int* go;                   /* device scratch int[nservers]                                           */
  int* err_flag;
  double timeout_s;
} MvbRowBox;
/* A push's ids (the first *n_ptr, or n_max) are ascending; a repeated id is applied once per entry, in list order;
 * ids outside [0, num_row) are ignored; at most `cap` entries may fall to one owner (more set err_flag to 3100 + owner
 * and the excess is dropped), so a list with repeats longer than `cap` goes in several pushes. */
int64_t mvb_rowbox_slot_bytes(int64_t cap, int64_t num_col);
int mvb_rowbox_slots(void);            /* slots per (owner, source) pair (double-buffered: 2) */
int mvb_rowbox_push_delta(const MvbRowBox* b, const int* ids, const int* n_ptr, int64_t n_max,
                          const float* cur, const float* old, int64_t ld, float scale, uint64_t epoch,
                          const MvbAddOpt* opt, int ctas_per_sm, void* stream);
int mvb_rowbox_push_vals(const MvbRowBox* b, const int* ids, const int* n_ptr, int64_t n_max,
                         const float* vals, int64_t ld, float scale, uint64_t epoch, const MvbAddOpt* opt,
                         int ctas_per_sm, void* stream);
int mvb_rowbox_poll(const MvbRowBox* b, int src, int wait, void* stream);
/* state_stride: elements per source slab; rowwise_adagrad indexes its slab by local row; adam's m and v are
 * element slabs, its step counts follow v's slab (st1 + state_stride + local row); ftrl's z (st0) and n (st1) are
 * element slabs */
int mvb_rowbox_apply(const MvbRowBox* b, int updater, float* shard, float* st0, float* st1,
                     int64_t state_stride, int64_t row_lo, int src, int ctas_per_sm, void* stream);

/* WordEmbedding block protocol on the device (we_block.cu): PrepareData without a host round trip,
   row pull / delta push in ctas_per_sm (>= 1) register-only CTAs per SM.  All counts live in device memory. */
typedef struct MvbWePrep {
  const int* tokens;         /* block of word ids, <0 = sentence break                          */
  int64_t n_tokens;
  int vocab;
  int negative;              /* K: negative x |input| pool draws (0 = no pool)                 */
  const float* alias_prob;   /* unigram^0.75 alias table                                      */
  const int* alias_idx;
  uint64_t seed;
  uint32_t* bm_in;           /* scratch bitmaps [ceil(vocab/32)]                                */
  uint32_t* bm_out;
  int* chunk_sums;           /* scratch [ceil(vocab/32768)]                                     */
  int* map_in;               /* out: word id -> slot in the input cache (-1 = absent) [vocab]   */
  int* map_out;
  int* ids_in;               /* out: slot -> word id [cap_in]                                   */
  int* ids_out;              /*                      [cap_out]                                  */
  int* neg_pool;             /* out: the block's negative pool [pool_cap]                       */
  int64_t pool_cap;
  int* counts;               /* out (device): [0] = n_in, [1] = n_out, [2] = n_pool             */
  int64_t cap_in, cap_out;
} MvbWePrep;
int mvb_we_prepare(const MvbWePrep* p, void* stream);
int mvb_we_prepare_launches(int negative);      /* kernels + memset/memcpy nodes it enqueues */
int mvb_rows_pull(const MvbRowMap* m, int esz, const int* ids, const int* n_ptr, int64_t n_max,
                  void* dst_a, void* dst_b, int64_t dst_ld, int ctas_per_sm, void* stream);
int mvb_rows_push_delta(const MvbRowMap* m, const int* ids, const int* n_ptr, int64_t n_max,
                        const float* cur, const float* old, int64_t ld, float scale, int ctas_per_sm,
                        void* stream);
int mvb_build_alias_table(const double* weights_host, int n, float* prob_host, int* alias_host);

/* ---- LogisticRegression (K8) ---------------------------------------------------- */
/* sparse CSR minibatch: objective 0 linear(squared) 1 sigmoid 2 softmax(dense only) */
typedef struct MvbLrSparse {
  const int64_t* row_ptr;    /* [n+1]                      */
  const int64_t* keys;       /* [nnz] feature ids          */
  const float* vals;         /* [nnz] (NULL => 1.0)        */
  const float* labels;       /* [n]                        */
  const float* sample_w;     /* [n] or NULL                */
  int64_t n;
  int objective;
  const float* w;            /* dense weight vector (pulled table) [dim*out] */
  int64_t dim;               /* input_size incl. bias      */
  int out;                   /* output classes (1 for binary) */
  float* grad;               /* [dim*out] accumulated += g*x / n  (atomic)  */
  float* loss_sum;           /* scalar                      */
  int* correct;              /* scalar: # correct predictions */
  float* pred;               /* optional [n*out]            */
  float* err;                /* scratch [n*out]: (p - y) * weight / n */
  int compute_grad;          /* 0 = predict only            */
} MvbLrSparse;
int mvb_lr_sparse_fwd_bwd(const MvbLrSparse* a, void* stream);
typedef struct MvbLrDense {
  const float* x;            /* [n x dim] row-major (bias column included) */
  const float* labels;       /* [n] class index or target                   */
  int64_t n, dim;
  int out;
  int objective;
  const float* w;            /* [out x dim]                                 */
  float* grad;               /* [out x dim]  = (1/n) sum (p-y) x^T          */
  float* loss_sum;
  int* correct;
  float* pred;               /* optional [n x out]                          */
  float* err;                /* scratch [n x out]                           */
  int compute_grad;
} MvbLrDense;
int mvb_lr_dense_fwd_bwd(const MvbLrDense* a, void* stream);
/* wide dense path (> 64 classes / GEMM-sized minibatches): logits and gradient run on the tcgen05 kernel
   (mvb_get_gemm_fused); this is the softmax / sigmoid / linear epilogue between the two products: loss,
   accuracy, predictions and the error matrix E^T = ((P - Y) / n)^T as [out x n_pad] (zero padded).     */
int mvb_lr_wide_epilogue(const float* logits, const float* labels, int64_t n, int out, int objective,
                         float* err_t, int64_t n_pad, float* pred, float* loss_sum, int* correct, void* stream);
int mvb_transpose_pad_f32(const float* in, int64_t rows, int64_t cols, int64_t ld_in, float* out,
                          int64_t ld_out, void* stream);
int mvb_axpy_f32(float* y, const float* x, int64_t n, float alpha, void* stream);
/* FTRL-proximal: weights from (z,n); gradient emits (dz,dn) (reference objective.cpp:260-336) */
int mvb_ftrl_weights(const float* z, const float* n, float* w, int64_t len, float alpha, float beta,
                     float l1, float l2, void* stream);
int mvb_ftrl_update(float* z, float* n, const float* w, const float* g, int64_t len, float alpha,
                    void* stream);
/* FTRL through the PS: dz = -(g - sigma w), dn = -g^2 with sigma = (sqrt(n + g^2) - sqrt(n)) / alpha */
int mvb_ftrl_delta(const float* n, const float* w, const float* g, float* dz, float* dn, int64_t len,
                   float alpha, void* stream);
/* regulariser add: 1 = L1 sign(w)*c, 2 = L2 w*c */
int mvb_regularize(float* grad, const float* w, int64_t len, int type, float coef, void* stream);

/* ---- fused Get + GEMM (tcgen05 / TMEM / TMA) -------------------------------------- */
/* Y[M x N] = X[M x K] * W[N x K]^T where W's rows are sharded over servers (row-range
 * partition, peer-mapped); optionally also materialises W into w_cache (the Get). */
typedef struct MvbGetGemm {
  const float* x;            /* [M x K] fp32 row-major, local     */
  float* y;                  /* [M x N] fp32                      */
  float* w_cache;            /* reserved (must be NULL)           */
  int64_t M, N, K;
  MvbRowMap wmap;            /* N rows x K cols over servers      */
  int local_server;          /* index of the shard in local HBM, -1 if none */
} MvbGetGemm;
int mvb_get_gemm_fused(const MvbGetGemm* g, void* stream);
int mvb_get_gemm_supported(void);
int mvb_get_gemm_last_config(void);  /* ctas*1000 + grid of the last launch */

/* ---- fused cosine top-k over a row-sharded MatrixTable (TMA + tf32 wgmma, top-k epilogue) ---- */
/* For each query row: the k rows of [0, n_rows) with the largest cosine over the first dim columns,
 * sorted by score descending, ties by the smaller id; zero rows score 0; missing slots get id -1 and
 * score -inf. tf32 selects k + 8 candidates, their cosines are recomputed in fp64 from the rows. W is
 * read from its owners' shards like mvb_get_gemm_fused (no collective). MVB_TOPK_MAX: k + 8 sorted
 * candidates per query next to the candidate buffer in the 227 KB of shared memory. */
#define MVB_TOPK_MAX 64
typedef struct MvbTopkCos {
  const float* q;            /* [M x ldq] fp32, ldq % 4 == 0, columns >= dim unused    */
  int64_t M, ldq;            /* M <= 65535 per call                                    */
  int64_t dim, n_rows;       /* columns compared (<= wmap.num_col); rows searched      */
  MvbRowMap wmap;            /* the table's shards, row pitch wmap.num_col (% 4 == 0)  */
  int k;                     /* 1 <= k <= MVB_TOPK_MAX                                 */
  float* scores;             /* [M x k] out                                            */
  int64_t* ids;              /* [M x k] out                                            */
  void* scratch;             /* device, mvb_topk_cos_scratch_bytes(M, k, n_rows) bytes */
  int64_t scratch_bytes;
} MvbTopkCos;
int64_t mvb_topk_cos_scratch_bytes(int64_t M, int k, int64_t n_rows);
int mvb_topk_cosine(const MvbTopkCos* a, void* stream);

/* Full softmax of an output layer whose classes are the rows [0, n_rows) of the table (topk_cos.cu, the
 * same one-pass search with the dot product z = q . w as the score): for each query row
 *   lse  = log sum_n exp(z_n)   (tf32 logits, fp32 accumulation, folded in a fixed tile / range order)
 *   loss = lse - z_label        (label logit in fp64; not clamped)
 * and / or the k rows with the largest z, sorted by score descending, ties by the smaller id (the fp64 dot
 * products of k + 8 tf32 candidates, rounded to fp32; missing slots id -1, score -inf). The [M x n_rows]
 * logits are never written. lse NULL: top-k only (k >= 1). labels and loss go together and need lse.
 * The caller validates labels (in [0, n_rows)). Errors: -40 k, -41 row map, -42 pitches, -43 dim,
 * -44 n_rows (1 <= n_rows <= num_row), -45 M or scratch, -46 outputs. */
typedef struct MvbFullSoftmax {
  const float* q;            /* [M x ldq] fp32, ldq % 4 == 0, columns >= dim unused             */
  int64_t M, ldq;            /* M <= 65535 per call                                             */
  int64_t dim, n_rows;       /* columns used (<= wmap.num_col); classes                         */
  MvbRowMap wmap;            /* the table's shards, row pitch wmap.num_col (% 4 == 0)           */
  int k;                     /* 0 <= k <= MVB_TOPK_MAX                                          */
  const int64_t* labels;     /* [M] or NULL                                                     */
  float* lse;                /* [M] out or NULL                                                 */
  float* loss;               /* [M] out, with labels                                            */
  float* scores;             /* [M x k] out, k > 0                                              */
  int64_t* ids;              /* [M x k] out, k > 0                                              */
  void* scratch;             /* device, mvb_full_softmax_scratch_bytes(M, k, n_rows) bytes      */
  int64_t scratch_bytes;
} MvbFullSoftmax;
int64_t mvb_full_softmax_scratch_bytes(int64_t M, int k, int64_t n_rows);
int mvb_full_softmax(const MvbFullSoftmax* a, void* stream);

/* Backward of the full softmax over all num_row rows of the table (full_softmax_bwd.cu): with the forward's lse,
 * the upstream gradient g of loss = lse - z_label and G_bn = g_b (exp(z_bn - lse_b) - [labels_b = n]),
 *   dq = G W            ([M x dim] at pitch lddq, or NULL: not computed)
 *   dw = scale G^T Q    ([num_row x dim] at pitch lddw, every row written whole, or NULL: not computed)
 * recomputing the tf32 logits tile by tile; the [M x num_row] logits are never written. dw is bitwise the same for
 * every sharding of the table; dq agrees across shardings within the tf32 bound. M == 0 zeroes dw. The caller
 * validates labels (in [0, num_row)). Errors, all before any CUDA call: MVB_BAD_ROW_MAP, -42 pitches (ldq, num_col),
 * -43 dim, -44 num_row, -45 M or scratch, -46 outputs or inputs missing, -47 output pitches below dim. */
typedef struct MvbFullSoftmaxBwd {
  const float* q;            /* [M x ldq] fp32, ldq % 4 == 0, columns >= dim unused             */
  int64_t M, ldq;
  int64_t dim;               /* columns used (<= wmap.num_col)                                  */
  MvbRowMap wmap;            /* the table's shards, row pitch wmap.num_col (% 4 == 0)           */
  const int64_t* labels;     /* [M]                                                             */
  const float* lse;          /* [M] the forward's log-partition                                 */
  const float* g;            /* [M] dL/dloss                                                    */
  float* dq;                 /* [M x lddq] out or NULL                                          */
  int64_t lddq;
  float* dw;                 /* [num_row x lddw] out or NULL, columns >= dim untouched          */
  int64_t lddw;
  float scale;               /* dw multiplier                                                   */
  void* scratch;             /* device, mvb_full_softmax_bwd_scratch_bytes(M, dim, num_row, dq != NULL, dw != NULL) */
  int64_t scratch_bytes;
} MvbFullSoftmaxBwd;
int64_t mvb_full_softmax_bwd_scratch_bytes(int64_t M, int64_t dim, int64_t n_rows, int with_dq, int with_dw);
int mvb_full_softmax_bwd(const MvbFullSoftmaxBwd* a, void* stream);

/* ---- embedding bag over a row-sharded fp32 MatrixTable (emb_bag.cu) ---------------------------- */
/* Bag b holds the lookups [offsets[b], offsets[b + 1]) (the last bag ends at L); its output row is the sum
 * (mean: the sum over the bag length) of psw_j * W[ids_j, :dim]; an empty bag gives zeros. Rows are read
 * from their owners' shards through wmap, as mvb_get_rows does. Results are bitwise reproducible and the
 * same for every sharding of the table. The caller validates ids (in [0, num_row)) and offsets. */
enum { MVB_EMB_PUSH = 0, MVB_EMB_COMPACT = 1 };
typedef struct MvbEmbBag {
  MvbRowMap wmap;            /* fp32 shards, row pitch wmap.num_col (% 4 == 0)                         */
  int64_t dim;               /* columns used, 1 <= dim <= wmap.num_col; padding columns are never read  */
  const int64_t* ids;        /* [L]; backward: sorted ascending, equal ids in ascending position        */
  int64_t L;
  const int64_t* offsets;    /* [B]: offsets[0] == 0, non-decreasing, <= L                              */
  int64_t B;
  const float* psw;          /* [L] per-sample weights by lookup position, or NULL                      */
  int mean;                  /* 0 sum, 1 mean                                                           */
  float* out;                /* forward: [B x ldo], ldo % 4 == 0, 16-byte aligned                       */
  int64_t ldo;
  const float* dout;         /* backward, psw grad: [B x ldd], ldd % 4 == 0, >= round4(dim) columns     */
  int64_t ldd;
  const int64_t* perm;       /* backward: lookup position of each sorted id                             */
  int epilogue;              /* MVB_EMB_PUSH: red.add of scale * g into the owner's row (default / sgd);
                                MVB_EMB_COMPACT: grads[u] = scale * g, uniq[u] = id, ids ascending      */
  float scale;
  float* grads;              /* compact: [U x ldg] (ldg % 4 == 0); NULL: only write *n_unique           */
  int64_t ldg;
  int64_t* uniq;             /* compact: [U]                                                            */
  int64_t* n_unique;         /* backward: device int64, the number of unique ids U, or NULL             */
  float* dpsw;               /* psw grad: [L]                                                           */
  void* scratch;             /* backward: mvb_embedding_bag_scratch_bytes(L, dim) bytes of device memory */
  int64_t scratch_bytes;
  int64_t push_rows;         /* backward: > 0: lookups of rows >= push_rows contribute nothing (no epilogue,
                                not in n_unique); <= 0: every row. Those rows sort last, so no other row's
                                rank or chunk boundary moves                                             */
} MvbEmbBag;
int mvb_embedding_bag_fwd(const MvbEmbBag* a, void* stream);
int64_t mvb_embedding_bag_scratch_bytes(int64_t L, int64_t dim);
/* sum of psw_j * s_bag * dout[bag(j)] per run of equal ids, in ascending position (s_bag = 1, or 1 / bag
 * length for mean), then the epilogue once per unique id */
int mvb_embedding_bag_bwd(const MvbEmbBag* a, void* stream);
/* dpsw[j] = s_bag * <dout[bag(j)], W[ids_j, :dim]> (ids in lookup order) */
int mvb_embedding_bag_psw_grad(const MvbEmbBag* a, void* stream);

/* ---- embedding-bag collection: F features over T row-sharded fp32 tables (emb_bag_coll.cu) -------- */
/* Jagged input: ids holds feature 0's lookups for bags 0..B-1, then feature 1's, ...; offsets[g] (g = f B + b)
 * is the exclusive scan of the [F x B] lengths. Feature f writes columns [col, col + round4(dim)) of out[b].
 * Each feature's bags are summed exactly as mvb_embedding_bag_fwd sums them over its table. The backward sorts
 * keys key_base[table] + id, so each table is one contiguous segment of the sorted order, cut into its own
 * chunks: a table's gradient depends only on its own lookups. The table and feature descriptors live in device
 * memory; they are built once and read by every call. The caller validates lengths and ids. */
enum { MVB_EMB_NO_PUSH = 2 };  /* a collection table whose gradient is not pushed */
typedef struct MvbEmbTable {
  MvbRowMap wmap;            /* fp32 shards, row pitch wmap.num_col (% 4 == 0), rows_per_server >= 1       */
  int64_t dim;               /* columns used, 1 <= dim <= min(512, wmap.num_col)                          */
  int64_t key_base;          /* backward key of row id: key_base + id (exclusive scan of the num_row)     */
  int mean;                  /* 0 sum, 1 mean                                                            */
  int epilogue;              /* MVB_EMB_PUSH, MVB_EMB_COMPACT or MVB_EMB_NO_PUSH                         */
  float scale;               /* the pushed value is scale * g                                            */
  int64_t ldg;               /* compact: row pitch of the table's gradient, % 4 == 0, >= round4(dim)     */
  int64_t push_rows;         /* > 0: lookups of rows >= push_rows contribute nothing to the backward (as in
                                MvbEmbBag); <= 0: every row                                              */
} MvbEmbTable;
typedef struct MvbEmbFeature {
  int table;                 /* index into the table descriptors                                         */
  int64_t col;               /* first column of the feature in out / dout, % 4 == 0                      */
} MvbEmbFeature;
typedef struct MvbEmbColl {
  const MvbEmbTable* tables;      /* device [T]                                                          */
  const MvbEmbFeature* features;  /* device [F]                                                          */
  const int* class_feats;         /* device [F]: the features grouped by register class (1..4 float4 per lane,
                                     round4(dim) <= 128, 256, 384, 512)                                   */
  int class_off[5];               /* class k holds class_feats[class_off[k - 1] .. class_off[k]), k = 1..4 */
  int T, F;
  int64_t B;                      /* bags per feature                                                    */
  const int64_t* ids;             /* [L] row ids, feature-major                                          */
  int64_t L;
  const int64_t* offsets;         /* [F B]                                                               */
  const float* psw;               /* [L] or NULL                                                         */
  float* out;                     /* forward: [B x ldo], ldo % 4 == 0, 16-byte aligned                   */
  int64_t ldo;
  const float* dout;              /* backward, psw grad: [B x ldd], ldd % 4 == 0, 16-byte aligned        */
  int64_t ldd;
  int64_t* keys;                  /* [L], written by mvb_emb_coll_keys                                   */
  const int64_t* skeys;           /* [L] keys sorted ascending, equal keys in ascending position         */
  const int64_t* perm;            /* [L] lookup position of each sorted key                              */
  int64_t* info;                  /* device int64 [4 T + 2]: per table {U, first unique, grads offset,
                                     uniq offset}, then the total floats of grads and entries of uniq      */
  float* grads;                   /* compact tables: table t's [U x ldg] gradient at grads + grads offset */
  int64_t* uniq;                  /* compact tables: table t's [U] row ids at uniq + uniq offset         */
  float* dpsw;                    /* psw grad: [L]                                                       */
  void* scratch;                  /* mvb_emb_coll_scratch_bytes(L, T, max dim) bytes of device memory    */
  int64_t scratch_bytes;
} MvbEmbColl;
int mvb_emb_coll_fwd(const MvbEmbColl* a, void* stream);
int64_t mvb_emb_coll_scratch_bytes(int64_t L, int T, int64_t max_dim);
/* backward, in order: keys (then sort them), count (unique ids per table into info), bwd (the epilogues) */
int mvb_emb_coll_keys(const MvbEmbColl* a, void* stream);
int mvb_emb_coll_count(const MvbEmbColl* a, void* stream);
int mvb_emb_coll_bwd(const MvbEmbColl* a, void* stream);
int mvb_emb_coll_psw_grad(const MvbEmbColl* a, void* stream);

/* ---- sampled softmax over a row-sharded fp32 MatrixTable (sampled_softmax.cu) ---------------------------- */
/* Example b has the true logit t_b = x_b . w_{y_b} - log(S q(y_b)) and the sampled logits
 * s_bj = logits[b, j] - logq_c[j], -inf where cand[j] == y_b; loss_b = logsumexp(t_b, s_b.) - t_b. The row
 * gathers and the products logits = X W_S^T, dX = E W_S, dW_S = E^T X are mvb_get_rows and mvb_get_gemm_fused. */
typedef struct MvbSampledSoftmax {
  const float* alias_prob;   /* [n] alias table of q (mvb_build_alias_table)                               */
  const int* alias_idx;      /* [n]                                                                        */
  const float* logq;         /* [n] log q(k)                                                               */
  int64_t n;                 /* rows of the table, < 2^31                                                  */
  uint64_t seed, step;       /* draw j of a call is a pure function of (seed, step, j)                     */
  int64_t S, S_pad;          /* draws per call; S_pad = round4(S), the row pitch of logits                 */
  float log_s;               /* log S in fp32                                                              */
  int64_t* cand;             /* sample: [S] drawn row ids                                                  */
  float* logq_c;             /* sample: [S] log_s + logq[cand]                                             */
  const float* x;            /* [B x d] hidden, 16-byte aligned                                            */
  const float* w_y;          /* [B x d] the label rows                                                     */
  int64_t B, B_pad, d;       /* d % 4 == 0; B_pad = round4(B), the row pitch of e_t                        */
  const int64_t* labels;     /* [B] in [0, n) (validated by the caller)                                    */
  float* logits;             /* [B x S_pad]: X W_S^T in the forward; the backward overwrites it with E      */
  float* loss;               /* forward: [B]                                                               */
  float* lse;                /* forward: [B] logsumexp of the row                                          */
  float* t_true;             /* forward: [B] the true logit                                                */
  const float* g;            /* backward: [B] gradient of the loss                                         */
  float* e_t;                /* backward: [S_pad x B_pad] E^T, zero on padding rows and columns            */
  float* e_true;             /* backward: [B] g_b (exp(t_b - lse_b) - 1)                                   */
} MvbSampledSoftmax;
int mvb_ss_sample(const MvbSampledSoftmax* a, void* stream);
int mvb_ss_fwd_epilogue(const MvbSampledSoftmax* a, void* stream);
int mvb_ss_bwd_epilogue(const MvbSampledSoftmax* a, void* stream);

/* ---- hierarchical softmax over a row-sharded fp32 MatrixTable (hier_softmax.cu) ------------------------------- */
/* Row p of the table is inner node p of a tree whose leaves are the n_classes labels. Example b with label y walks
 * the path points[y, 0..L) (root first, L = lens[y]) with branch codes codes[y, 0..L):
 *   z_i = hidden_b . w_{p_i},  loss_b = sum_i softplus(-(1 - 2 c_i) z_i),  g_i = sigmoid(z_i) - (1 - c_i),
 *   u_b = sum_i g_i w_{p_i}   (so dloss_b / dhidden_b = u_b)
 * One warp per example, rows read from their owners' shards as mvb_get_rows reads them. Every sum has a fixed order
 * and no atomics: loss, g and u are bitwise reproducible and the same for every sharding. Widths above
 * MVB_HSM_MAX_DIM are refused (-80). The caller validates labels (in [0, n_classes)) and that the tree's inner
 * nodes are < wmap.num_row. Errors, all before any CUDA call: MVB_BAD_ROW_MAP; -80 dim (4 <= dim <= MVB_HSM_MAX_DIM,
 * % 4 == 0, <= wmap.num_col) or a row pitch not % 4; -81 n_classes < 2, n_classes - 1 > wmap.num_row, or ldp outside
 * [1, MVB_HSM_MAX_PATH]; -82 B < 0 or a pitch (ldh, ldu) below dim or not % 4; -83 a missing input, ids or g without
 * offsets, or hidden, u or a shard not 16-byte aligned. B == 0 launches nothing. */
#define MVB_HSM_MAX_DIM 1024
#define MVB_HSM_MAX_PATH 64
typedef struct MvbHsm {
  MvbRowMap wmap;            /* fp32 shards, row pitch wmap.num_col (% 4 == 0); row p is inner node p          */
  int64_t dim;               /* columns used                                                                 */
  const float* hidden;       /* [B x ldh], 16-byte aligned                                                   */
  int64_t B, ldh;
  const int64_t* labels;     /* [B] in [0, n_classes)                                                        */
  int64_t n_classes;         /* leaves; the tree has n_classes - 1 inner nodes                               */
  const int* points;         /* [n_classes x ldp] inner-node ids of each label's path, root first            */
  const signed char* codes;  /* [n_classes x ldp] branch codes, 0 or 1                                       */
  const int* lens;           /* [n_classes] path lengths, 1 <= lens[y] <= ldp                                */
  int64_t ldp;
  const int64_t* offsets;    /* [B] exclusive scan of lens[labels]: example b's steps start at offsets[b];
                                needed with ids or g                                                         */
  float* loss;               /* [B] out, or NULL                                                             */
  int64_t* ids;              /* [sum of lens[labels]] out: the path node of every step, or NULL              */
  float* g;                  /* [sum of lens[labels]] out: dloss / dz of every step, or NULL                 */
  float* u;                  /* [B x ldu] out, 16-byte aligned, columns >= dim untouched, or NULL            */
  int64_t ldu;
} MvbHsm;
int mvb_hsm_fwd(const MvbHsm* a, void* stream);

/* ---- factorization machine over a row-sharded fp32 MatrixTable (fm.cu) ------------------------------------------ */
/* Row r holds the k = dim - 1 factors v_r = W[r, 0:k] and the linear weight W[r, k]. Bag b holds the lookups
 * [offsets[b], offsets[b + 1]) (the last bag ends at L) with ids i_j and values x_j:
 *   S_b = sum_j x_j W[i_j, :dim],  q_b = sum_j x_j^2 |v_{i_j}|^2,  y_b = S_b[k] + (|S_b[0:k]|^2 - q_b) / 2
 * (an empty bag gives 0). S_b is summed exactly as mvb_embedding_bag_fwd sums the bag with per-sample weights x.
 * The backward pushes, once per unique row r, scale * sum over the lookups j of r of dy_b x_j (S'_b - x_j v'_r),
 * S'_b being S_b with column k set to 1 and v'_r being v_r with 0 in column k, through the epilogues of
 * MvbEmbBag. Results are bitwise reproducible and the same for every sharding; rows are read from their owners'
 * shards as mvb_get_rows reads them. The caller validates ids (in [0, num_row)) and offsets. Errors, all before any
 * CUDA call: MVB_BAD_ROW_MAP; -90 dim outside [2, MVB_FM_MAX_DIM] or above wmap.num_col, a row pitch not % 4, or a
 * shard not 16-byte aligned; -91 B < 0, L < 0, or offsets / ids missing; -92 (fwd) y missing with B > 0, or sp set with a bad
 * pitch or alignment; -93 (bwd, L > 0) dy, sp, perm or scratch missing, sp's pitch or alignment bad, or scratch too
 * small; -94 (bwd) an unknown epilogue or a compact gradient without uniq, with a bad pitch or alignment. B == 0
 * (fwd) and L == 0 (bwd) launch nothing. */
#define MVB_FM_MAX_DIM 1024
typedef struct MvbFm {
  MvbRowMap wmap;            /* fp32 shards, row pitch wmap.num_col (% 4 == 0), 16-byte aligned             */
  int64_t dim;               /* C = k + 1 columns used, 2 <= C <= min(MVB_FM_MAX_DIM, wmap.num_col)          */
  const int64_t* ids;        /* [L]; backward: sorted ascending, equal ids in ascending position             */
  int64_t L;
  const int64_t* offsets;    /* [B]: offsets[0] == 0, non-decreasing, <= L                                   */
  int64_t B;
  const float* values;       /* [L] x by lookup position, or NULL (every x is 1)                             */
  float* y;                  /* forward: [B] out                                                             */
  float* sp;                 /* [B x lds] S': forward out (NULL: not written), backward in; 16-byte aligned   */
  int64_t lds;               /* % 4 == 0, >= round4(dim); columns in [dim, round4(dim)) are written 0         */
  const float* dy;           /* backward: [B] dL/dy                                                          */
  const int64_t* perm;       /* backward: lookup position of each sorted id                                  */
  int epilogue;              /* MVB_EMB_PUSH (red.add into the owner's row) or MVB_EMB_COMPACT               */
  float scale;
  float* grads;              /* compact: [U x ldg] (ldg % 4 == 0), 16-byte aligned; NULL: only write *n_unique */
  int64_t ldg;
  int64_t* uniq;             /* compact: [U] ascending                                                       */
  int64_t* n_unique;         /* backward: device int64, the number of unique ids U, or NULL                  */
  void* scratch;             /* backward: mvb_embedding_bag_scratch_bytes(L, dim) bytes of device memory      */
  int64_t scratch_bytes;
  int64_t push_rows;         /* backward: > 0: rows >= push_rows get no epilogue and are not counted (as in
                                MvbEmbBag); <= 0: every row                                                  */
} MvbFm;
int mvb_fm_fwd(const MvbFm* a, void* stream);
int mvb_fm_bwd(const MvbFm* a, void* stream);

/* ---- field-aware factorization machine over a row-sharded fp32 MatrixTable (ffm.cu) ---------------------------- */
/* F fields of k factors, D = F k. Row r holds V_r[f] = W[r, f k : (f + 1) k] (f < F) and the linear weight
 * w_r = W[r, D]; columns past D are never used. Bag b holds the lookups [offsets[b], offsets[b + 1]) (the last bag
 * ends at L) with ids i_j, fields f_j and values x_j:
 *   y_b = sum_j x_j w_{i_j} + sum_{j < l} x_j x_l <V_{i_j}[f_l], V_{i_l}[f_j]>   (an empty bag gives 0)
 * With h set, the forward also writes, for every lookup j of bag b, H_j = dy_b / d(row values at j):
 *   H_j[f k + c] = x_j sum_{l != j in the bag, f_l = f} x_l V_{i_l}[f_j][c] (l in position order),  H_j[D] = x_j,
 * and 0 in the columns [D + 1, ldh). The row gradient of sum_b g_b y_b is then sum_{j: i_j = r} g_{b(j)} H_j: the
 * embedding-bag backward (MvbEmbBag) over one bag per lookup with per-sample weights g_{b(j)} and dout = H.
 * y_b = sum_j x_j w_{i_j} + (1/2) sum_j <H_j[0:D], W[i_j, 0:D]>, with each thread's terms in a fixed order and a
 * fixed-tree reduction: y and H are bitwise reproducible, the same for every sharding and for any max_len, and y is
 * the same with and without h. Rows are read from their owners' shards as mvb_get_rows reads them. The caller
 * validates ids (in [0, num_row)), fields (in [0, F)) and offsets. Errors, all before any CUDA call:
 * MVB_BAD_ROW_MAP; -95 k < 4, k not % 4, F < 1 or D + 1 > MVB_FFM_MAX_DIM; -96 wmap.num_col < D + 1 or not % 4,
 * or a shard not 16-byte aligned; -97 B < 0 or L < 0; -98 offsets / y missing with B > 0, or ids / fields missing
 * with L > 0; -99 h set with ldh not % 4, ldh < round4(D + 1), or h not 16-byte aligned. B == 0 launches nothing. */
#define MVB_FFM_MAX_DIM 1024
typedef struct MvbFfm {
  MvbRowMap wmap;            /* fp32 shards, row pitch wmap.num_col (% 4 == 0, >= D + 1), 16-byte aligned     */
  int64_t F;                 /* fields, >= 1                                                                 */
  int64_t k;                 /* factors per field, % 4 == 0, >= 4; F k + 1 <= MVB_FFM_MAX_DIM                 */
  const int64_t* ids;        /* [L] rows                                                                     */
  const int* fields;         /* [L] field of every lookup, in [0, F)                                         */
  const float* values;       /* [L] x by lookup position, or NULL (every x is 1)                             */
  const int64_t* offsets;    /* [B]: offsets[0] == 0, non-decreasing, <= L                                   */
  int64_t L;
  int64_t B;
  int64_t max_len;           /* the longest bag, or <= 0: unknown. Only sizes the shared-memory tile           */
  float* y;                  /* [B] out                                                                      */
  float* h;                  /* [L x ldh] out (16-byte aligned), or NULL: not written                         */
  int64_t ldh;               /* % 4 == 0, >= round4(D + 1)                                                   */
} MvbFfm;
int mvb_ffm_fwd(const MvbFfm* a, void* stream);

/* ---- random walks on a CSR graph: DeepWalk and node2vec (walk.cu) ----------------------------------------------- */
/* Node v's out-list is indices[indptr[v], indptr[v + 1]), sorted ascending (repeated entries are multi-edges); cum,
 * when set, holds the weights' prefix sums within each list (mvb_csr_cumsum). Walk i is walk number g = first_walk + i:
 * row i of out holds starts[i] and the nodes it visits, -1 in every slot after the walk ends (L nodes, or a node
 * without out-arcs), up to the pitch. Every random number is a pure function of (seed, g, step, attempt)
 * (multiverso_b200/ops/random_walk.py states the formula), so the walks do not depend on the launch or on how the
 * starts are split between calls. With node_count set, the number of nodes written is added to it. The caller
 * validates starts (in [0, num_nodes)). Errors, all before any CUDA call: -100 indptr / indices / starts / out
 * missing, or a pointer not aligned to its element; -101 num_nodes < 0 or >= 2^31 - 1, or n < 0 or >= 2^31;
 * -102 length < 1 or >= 2^31; -103 pitch < length; -104 p or q not finite and > 0, or 1/p or 1/q not finite and
 * > 0 in fp32; -105 first_walk < 0 or first_walk + n > INT64_MAX. n == 0 launches nothing. */
typedef struct MvbRandomWalk {
  const int64_t* indptr;     /* [num_nodes + 1]                                                             */
  const int* indices;        /* [E], each list sorted ascending                                             */
  const double* cum;         /* [E] per-list prefix sums of positive weights, or NULL: unweighted            */
  int64_t num_nodes;
  const int* starts;         /* [n] first node of every walk                                                */
  int64_t n;
  int64_t length;            /* L >= 1 nodes per walk at most                                              */
  int64_t pitch;             /* row pitch of out in ints, >= L                                              */
  double p;                  /* return parameter                                                           */
  double q;                  /* in-out parameter; p = q = 1: first-order (DeepWalk)                         */
  uint64_t seed;
  int64_t first_walk;        /* walk number of row 0                                                       */
  int* out;                  /* [n x pitch]                                                                */
  int64_t* node_count;       /* device int64 += nodes written, or NULL                                      */
} MvbRandomWalk;
int mvb_random_walk(const MvbRandomWalk* a, void* stream);
/* cum[j] = w[indptr[v]] + ... + w[j] for j in v's list, summed in list order in fp64. Errors: -100 a pointer missing
 * or not 8-byte aligned; -101 num_nodes < 0 or >= 2^31 - 1. */
int mvb_csr_cumsum(const int64_t* indptr, const double* w, int64_t num_nodes, double* cum, void* stream);

#ifdef __cplusplus
}
#endif
