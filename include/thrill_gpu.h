/*******************************************************************************
 * include/thrill_gpu.h — C ABI of libthrill_gpu.so
 *
 * The drop-in boundary for Thrill's Sort / ReduceByKey hot path on H100 (sm_90a).
 * Thrill (thrill/thrill @ 12c5b59b) has no FFI of its own — operators are header templates — so every
 * entry point below cites the reference interface it REPLACES (paths relative to the reference root);
 * INTEGRATION.md shows the host-side DOpNode classes (thrill_b200/host/) that bind them.
 *
 * Conventions: plain pointers and sizes, no C++ types, no exceptions.  Every function returns TG_OK (0)
 * or a negative tg_status; tg_last_error(ctx) gives a message.  The host shim turns non-zero into
 * die() → tlx::DieException, the reference's only error path (api/dia_base.cpp:143-150).
 * One tg_ctx per worker thread / GPU / CUDA stream / NCCL rank (api/context.hpp:243-245: one worker =
 * one DIA shard).  Functions are asynchronous on the ctx stream unless stated; they are not re-entrant
 * per ctx.  Collective entry points (tg_sort, tg_reduce_by_key with nranks > 1) must be entered by all
 * ranks in the same order — the rule Thrill has for GetNewMixStream (api/context.hpp:308-316).
 * Device buffers passed in must be 16-byte aligned.  There is NO CPU fallback anywhere behind this ABI.
 *
 * Limits (TG_ERR_TOO_LARGE, checked before any work): every entry point that takes a device item count (tg_radix_sort_local,
 * tg_classify_scatter, tg_sort_select (per shard), tg_hash_aggregate, tg_hash_partition, tg_range_partition, tg_sort, tg_reduce_by_key,
 * tg_reduce_to_index and their _file / _dev forms) takes at most 2^30 - 1 items per call and worker (n_local), and a worker receives at most 2^30 - 1
 * items in an exchange: the partition passes count in 30-bit fields.  ReduceToIndex gives each worker fewer than 2^31
 * indices of the result.  Merge (tg_merge and its forms) takes at most 2^30 - 1 items in a worker's k inputs together, and gives
 * each worker at most 2^30 - 1 items of the result; it merges 2..16 inputs of 8- or 16-byte items.  InnerJoin (tg_inner_join
 * and its _file form) takes at most 2^30 - 1 items per worker and side, before and after its exchange, and gives each worker at
 * most 2^30 - 1 items of the result.  GroupByKey and GroupToIndex (tg_group_by_key, tg_group_to_index and their _file forms)
 * take at most 2^30 - 1 items per worker, before and after their exchange, and tg_mod_partition at most 2^30 - 1 items per call.
 * PrefixSum, ExPrefixSum and ZipWithIndex (tg_prefix_sum, tg_zip_with_index, their _file and _select forms, tg_scan_local_total)
 * take at most 2^30 - 1 items per worker and give each worker as many items as it holds.  Sum, Min, Max and AllReduce (tg_all_reduce
 * and its _file and _select forms) take at most 2^30 - 1 items per worker.  The collective operators return TG_ERR_TOO_LARGE on every rank or on none.
 ******************************************************************************/
#ifndef THRILL_GPU_H
#define THRILL_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tg_ctx tg_ctx;

typedef enum {
    TG_OK = 0,
    TG_ERR_CUDA = -1,          /* a CUDA runtime call failed */
    TG_ERR_NCCL = -2,          /* an NCCL call failed */
    TG_ERR_ARG = -3,           /* bad argument / unsupported descriptor */
    TG_ERR_TOO_LARGE = -4,     /* over a per-call limit (see Limits above) */
    TG_ERR_NO_DEVICE = -5,     /* no sm_90 device: the product path fails loudly, never falls back */
    TG_ERR_OOM = -6
} tg_status;

/* ---- descriptors: the closed set of (type, functor) pairs the GPU path accepts ----------------------
 * Reference operators take arbitrary C++ lambdas (api/dia.hpp:1753-1816 Sort(cmp), :929-1170
 * ReduceByKey(key_ex, red_fn)).  The host shim recognises the supported functor types and fills these. */
enum { TG_KEY_UINT_LE = 0,     /* unsigned little-endian integer key of 1..8 bytes inside 8- or 16-byte items: std::less<T> */
       TG_KEY_BYTES_BE = 1 };  /* byte-string key compared lexicographically (TeraSort Record,
                                  examples/terasort/terasort.cpp:35-37): <= 16 bytes in 16-byte items, <= 12 bytes in
                                  records (item_bytes % 4 == 0, e.g. 100) */
typedef struct {
    uint32_t item_bytes;       /* serialized item size (data/serialization.hpp:34-49): 8, 16 or 100 */
    uint32_t key_offset;
    uint32_t key_bytes;
    uint32_t key_kind;         /* TG_KEY_* */
    uint32_t descending;       /* std::greater<T> */
    uint32_t stable;           /* SortStable (api/sort.hpp:873-937); the GPU path is always stable */
} tg_key_desc;

enum { TG_OP_SUM_F64 = 0, TG_OP_SUM_U64 = 1, TG_OP_MIN_U64 = 2, TG_OP_MAX_U64 = 3,
       TG_OP_MIN_F64 = 4, TG_OP_MAX_F64 = 5, TG_OP_FIRST = 6 };
typedef struct {
    uint32_t item_bytes;       /* 16: pair<uint64_t key, 8-byte value> serialized member-wise
                                  (data/serialization.hpp:67-84), the ReducePair TableItem
                                  (api/reduce_by_key.hpp:410-449, core/reduce_functional.hpp:156-209) */
    uint32_t op;               /* TG_OP_*: the recognised ReduceFunction (std::plus<double>, ...) */
} tg_kv_desc;

/* one data::Block of a data::File as the host sees it after PinWait (data/block.hpp:52-145):
 * `data` = ByteBlock::data() + begin, `bytes` = end - begin */
typedef struct {
    const void* data;
    size_t bytes;
} tg_block;
typedef struct {
    void* data;
    size_t bytes;
} tg_block_mut;

/* ---- context ---------------------------------------------------------------------------------------- */
int tg_version(void);
int tg_device_count(void);                          /* sm_90 GPUs visible to this process (0: none, no CPU fallback) */
const char* tg_strerror(int status);
const char* tg_last_error(const tg_ctx* ctx);

/* 128-byte NCCL unique id for the job (rank 0 creates it, the host control plane — Thrill's
 * net::FlowControlChannel broadcast, net/flow_control_channel.hpp:404 — distributes it). */
int tg_get_unique_id(void* out128);
/* Replaces per-worker setup in api/context.cpp:1179 (Context ctor) for the GPU operators: binds `device`
 * (= Context::local_worker_id()), creates the stream and, if nranks > 1, the NCCL communicator that stands
 * in for data::MixStream (data/mix_stream.cpp:52-113).  unique_id may be NULL when nranks == 1. */
int tg_init(int device, int rank, int nranks, const void* unique_id128, tg_ctx** out_ctx);
int tg_shutdown(tg_ctx* ctx);
int tg_rank(const tg_ctx* ctx);
int tg_nranks(const tg_ctx* ctx);
void* tg_stream(const tg_ctx* ctx);                 /* cudaStream_t of the ctx */
int tg_sync(tg_ctx* ctx);                           /* cudaStreamSynchronize */
int tg_barrier(tg_ctx* ctx);                        /* ncclAllReduce of one int + sync: ctx.net.Barrier() */

/* device memory owned by the ctx (BlockPool analogue for HBM, data/block_pool.hpp:40) */
int tg_alloc(tg_ctx* ctx, size_t bytes, void** out_dptr);
int tg_free(tg_ctx* ctx, void* dptr);
/* device timing on the ctx stream (CUDA events) */
int tg_timer_start(tg_ctx* ctx);
int tg_timer_stop(tg_ctx* ctx, float* out_ms);      /* synchronises */
/* kernels launched by this ctx since tg_init (bench.py's gpu_launches) */
uint64_t tg_launch_count(const tg_ctx* ctx);
/* how many local sorts on this ctx abandoned the prefix sort (top digits + finishing pass) for the plain LSD passes
 * because a run of equal key prefixes was too long (heavy duplicates); see tg_radix_sort_local */
uint64_t tg_prefix_sort_fallbacks(const tg_ctx* ctx);
/* records of popular keys that the aggregations on this ctx folded in their counting read, cumulative (such records are read once
 * and never moved: bench.py needs the count for the algorithmic bytes of the hash passes) */
uint64_t tg_hot_records(const tg_ctx* ctx);
/* per-kernel-class device timing (CUDA events around every launch of the class while enabled):
 * bench.py's live roofline measurement.  tg_profile_get synchronises and returns the summed duration
 * and the number of launches of `kernel_class` since tg_profile_enable(ctx, 1). */
enum { TG_K_RADIX_HIST = 0, TG_K_PARTITION = 1, TG_K_MERGE = 2, TG_K_PREAGG = 3, TG_K_AGGREGATE = 4,
       TG_K_COMPACT = 5, TG_K_OTHER = 6, TG_K_FIXUP = 7, TG_K_SEGCOUNT = 8,
       TG_K_EXCHANGE = 9 /* the NCCL Alltoallv (not a kernel of ours: timed like one) */,
       TG_K_JOIN = 10 /* InnerJoin's co-rank count, offset scan and emit kernels */,
       TG_K_SCAN = 11 /* PrefixSum's tile reduce, tile prefix and scan kernels; ZipWithIndex's kernel; the actions' tile reduce
                         and fold */, TG_K_NUM = 12 };
int tg_profile_enable(tg_ctx* ctx, int on);
int tg_profile_get(tg_ctx* ctx, int kernel_class, float* out_total_ms, uint64_t* out_launches);
/* the individual launch durations of `kernel_class` in launch order (up to `capacity`); *out_n = how many there are */
int tg_profile_list(tg_ctx* ctx, int kernel_class, float* out_ms, size_t capacity, size_t* out_n);
/* page-locked host memory (what the BlockPool arenas should be for full PCIe bandwidth; the host shim
 * can equally cudaHostRegister its existing ByteBlocks) */
int tg_host_alloc(tg_ctx* ctx, size_t bytes, void** out_hptr);
int tg_host_free(tg_ctx* ctx, void* hptr);

/* ---- File <-> flat device buffer codec (SURVEY.md §8b; data/file.hpp:56-283) -------------------------
 * A File of fixed-size POD items is the concatenation of its Blocks' [begin,end) with zero framing
 * (data/serialization.hpp:34-49; items may straddle Blocks).  Upload gathers Blocks into consecutive
 * device bytes (replaces File::GetReader + BlockReader::Next per item, data/block_reader.hpp:87-139);
 * download scatters consecutive device bytes into caller-allocated ByteBlocks (replaces
 * BlockWriter::Put per item, data/block_writer.hpp:208-335).  Host memory is the caller's. */
int tg_upload(tg_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int tg_download(tg_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
int tg_upload_blocks(tg_ctx* ctx, void* dst_dev, const tg_block* blocks, size_t nblocks, size_t* out_bytes);
int tg_download_blocks(tg_ctx* ctx, const void* src_dev, const tg_block_mut* blocks, size_t nblocks);
/* The Block geometry BlockWriter would produce for `num_items` fixed-size items (block sizes start at
 * start_block_size, double while 2*bs < max_block_size: data/block_writer.hpp:61-67,405-420); fills
 * {bytes, first_item, num_items} per block so the host shim can build data::Block(begin=0,end,first_item,
 * num_items).  Pure host arithmetic.  Returns the number of blocks (or needed count if > capacity). */
typedef struct { uint64_t bytes, first_item, num_items; } tg_block_geom;
size_t tg_file_geometry(uint64_t num_items, uint32_t item_bytes, uint64_t start_block_size,
                        uint64_t max_block_size, tg_block_geom* out, size_t capacity);

/* ---- kernel-level entry points (parity tests, ncu captures) ------------------------------------------ */

/* Stable local sort of n items in place (result in d_items); d_tmp >= n*item_bytes scratch.  Replaces
 * SortNode::SortAndWriteToFile's sort_algorithm_(begin,end,cmp) = std::sort (api/sort.hpp:696-742,
 * :789-796) and the common::RadixSort functor hook (common/radix_sort.hpp:147-162).  Radix sort on the
 * non-constant key bytes: partition passes on the K most significant ones + one finishing pass on the runs
 * of equal prefixes, or plain LSD passes where that does not apply (DESIGN.md §4). */
int tg_radix_sort_local(tg_ctx* ctx, const tg_key_desc* desc, void* d_items, void* d_tmp, size_t n);

/* Sample count and host-side splitter selection: common/reservoir_sampling.hpp:270-275 (eps = 0.1,
 * api/sort.hpp:298) and FindAndSendSplitters (api/sort.hpp:337-378, LessSampleIndex :419-422).
 * samples: nsamples x (item_bytes + 8) packed (item, u64 global index) = SampleIndexPair on the wire;
 * sorted in place; writes p-1 splitters in the same packing.  Pure host arithmetic. */
uint64_t tg_sample_size(uint64_t local_items);
int tg_select_splitters(const tg_key_desc* desc, void* samples, uint64_t nsamples, uint32_t p,
                        void* out_splitters);

/* Draw the local sample on the device: min(n, tg_sample_size(n)) items at indices rng % n (the
 * OnPreOpFile path, api/sort.hpp:151-175), packed (item, global_index_base + index) into host memory. */
int tg_draw_samples(tg_ctx* ctx, const tg_key_desc* desc, const void* d_items, size_t n,
                    uint64_t global_index_base, uint64_t rng_seed, void* out_samples_host, uint64_t* out_nsamples);

/* Splitter classify + histogram + scatter.  Replaces SortNode::TransmitItems (api/sort.hpp:434-535):
 * tree descent over the p-1 splitters, ties to a splitter broken by global index
 * (EqualSampleGreaterIndex :424-426, :487-502); item i of d_in has global index global_index_base + i.
 * d_out receives the items grouped by destination worker in stable order; out_counts[p] (host) the
 * per-destination counts (what BlockWriter::Put into data_writers[b] accumulated, :507-508). */
int tg_classify_scatter(tg_ctx* ctx, const tg_key_desc* desc, const void* d_in, size_t n,
                        uint64_t global_index_base, const void* splitters_host, uint32_t p,
                        void* d_out, uint64_t* out_counts);

/* The classification of the multi-worker Sort for p simulated workers on one device (2 <= p <= 16, any ctx): shard w (n_shards[w]
 * items at d_shards[w], global indices after those of the shards before it) is worker w.  It runs the operator's device code
 * except the all-gather: worker w draws its sample with the operator's seed into the slot the all-gather fills, the splitters and
 * their top-byte lookup table are selected on the device as worker w does, and the classification pass of the exchange stores
 * shard w's items grouped by destination (stable) into d_out[w] instead of the peers' windows.  Writes out_splitters: (p-1) x
 * (item_bytes + 8) packed as by tg_select_splitters (the sampled item, its global index; zeros when there are no items at all),
 * out_counts[src * p + dst], and if out_merge_bounds is not NULL, the bucket boundaries the merge pipeline (TG_SORT_PIPELINE=merge)
 * computes on the stable sort of each shard: out_merge_bounds[w * (p-1) + j].  Shards are read, never modified.  8- or 16-byte
 * items with any descriptor tg_sort takes for them (records are classified as 16-byte BYTES_BE tuples); otherwise TG_ERR_ARG;
 * a shard of 2^30 or more items is TG_ERR_TOO_LARGE. */
int tg_sort_select(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_shards, const size_t* n_shards, uint32_t p,
                   uint64_t rng_seed, void* out_splitters, void* const* d_out, uint64_t* out_counts, uint64_t* out_merge_bounds);

/* k-way merge of sorted runs laid back to back in d_runs (run r has run_items[r] items).  Replaces
 * core::MultiwayMergeTree::Next over tlx::LoserTree (core/multiway_merge.hpp:30-116,
 * extlib/tlx/tlx/container/loser_tree.hpp:54-292) as driven by SortNode::PushData (api/sort.hpp:216-271).
 * Ties are resolved by run index (the stable variant, :265-292), which is a valid unstable outcome too. */
int tg_kway_merge(tg_ctx* ctx, const tg_key_desc* desc, const void* d_runs, const uint64_t* run_items,
                  uint32_t k, void* d_out, void* d_tmp);

/* Open-addressing hash aggregate of n (key,value) items into distinct keys.  Replaces
 * ReducePrePhase::Insert / ReduceByHashPostPhase::Insert -> ReduceProbingHashTable::Insert
 * (core/reduce_probing_hash_table.hpp:190-268) + FlushAll (:484-488).  The key 0 (== Key(), the
 * reference's empty-slot sentinel, :195-218) is supported through a side accumulator.
 * d_out must hold min(n, capacity_hint) items; *out_distinct (host) = number of distinct keys.
 * Output order is table order (unspecified, as in the reference). */
int tg_hash_aggregate(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n,
                      void* d_out, uint64_t* out_distinct);

/* Hash partition: destination worker of key = Hash128to64(0, key) % p (common/hash.hpp:64-73,
 * core/reduce_functional.hpp:60-72 with std::hash<uint64_t> = identity), items grouped by destination in
 * d_out, counts in out_counts[p] (host).  Replaces ReducePrePhaseEmitter::Emit into
 * writer_[partition_id] (core/reduce_pre_phase.hpp:57-61). */
int tg_hash_partition(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n, uint32_t p,
                      void* d_out, uint64_t* out_counts);

/* Range partition of ReduceToIndex (what its exchange classifies by): destination of a 16-byte item with u64 index k is
 * k < size ? k * p / size : p - 1 (core/reduce_functional.hpp:112-125; worker d's range starts at ceil(d * size / p)).  Stable:
 * d_out receives the items grouped by destination in input order, out_counts[p] (host) the counts.  1 <= p <= 256; a size with
 * (size - 1) * p >= 2^64 is TG_ERR_ARG. */
int tg_range_partition(tg_ctx* ctx, const void* d_in, size_t n, uint64_t size, uint32_t p,
                       void* d_out, uint64_t* out_counts);

/* The arithmetic of one exchange, pure host code (what every rank derives from the all-gathered p x p count matrix; exported so
 * that the N > 1 host logic is testable without GPUs): counts[src * p + dst] = items rank src holds for rank dst.  For rank `me`:
 * send_cnt[d], recv_cnt[s], recv_before[d] = items of the ranks below `me` in rank d's window (where this rank's share starts),
 * *n_recv = items this rank receives, *worst = the largest receive size of ANY rank (window growth and TG_ERR_TOO_LARGE are
 * decided on it, identically everywhere).  Replaces the per-(src,dst) block headers of the MixStream (data/multiplexer_header.hpp:36-72). */
int tg_exchange_plan(uint32_t p, uint32_t me, const uint32_t* counts, uint64_t* send_cnt, uint64_t* recv_cnt,
                     uint64_t* recv_before, uint64_t* n_recv, uint64_t* worst);

/* ---- operator-level entry points -------------------------------------------------------------------- */

/* Whole SortNode::MainOp + PushData (api/sort.hpp:537-663, :216-271) on device-resident items:
 * ExPrefixSumTotal (:541) -> samples -> splitters -> classify/scatter -> NCCL Alltoallv (replaces the
 * MixStream exchange :615-641: here the classification pass stores into the peers' exchange windows) -> local radix sort
 * of what was received.  d_in holds n_local items (it is clobbered); *out_dptr points to *out_n items inside a ctx-owned
 * workspace, the exchange window or d_in itself: valid until the next operator call on this ctx, never to be freed by the
 * caller (tg_free rejects it), to be copied (or detached with tg_output_detach after a *_file / *_dev call) before it is
 * fed to another operator.  At most 16 ranks.  Collective: sizes are agreed on by all ranks. */
int tg_sort(tg_ctx* ctx, const tg_key_desc* desc, void* d_in, size_t n_local, uint64_t rng_seed,
            void** out_dptr, size_t* out_n);

/* Whole ReduceNode (api/reduce_by_key.hpp:100-211): local pre-aggregation (pre phase), hash partition,
 * NCCL Alltoallv (replaces MixStream, :109-114), final aggregation (post phase).  Collective. */
int tg_reduce_by_key(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n_local,
                     void** out_dptr, size_t* out_n);

/* DIA<pair<size_t, V>>::ReduceToIndex(key = .first, reduce function on .second, result_size, neutral_element)
 * (api/reduce_to_index.hpp:60-237; the PageRank step, examples/page_rank/page_rank.hpp:125-135): pre phase = local
 * aggregation, range partition k -> k * p / result_size (core/reduce_functional.hpp:83-149, common/math.hpp:83-120),
 * NCCL Alltoallv, dense post phase (core/reduce_by_index_post_phase.hpp:43-330).  Rank r receives the contiguous index
 * range [ceil(r*size/p), ceil((r+1)*size/p)) as a dense array of 16-byte items in *out_dptr: item i = (i, fold of the values
 * whose index is i), or *neutral_item16 where no item has that index.  *out_begin = first index of the range.  An index
 * >= result_size is TG_ERR_ARG (the reference asserts).  Collective. */
int tg_reduce_to_index(tg_ctx* ctx, const tg_kv_desc* desc, const void* d_in, size_t n_local, uint64_t result_size,
                       const void* neutral_item16, void** out_dptr, size_t* out_n, uint64_t* out_begin);
/* ... with a host File as input; the dense result is fetched with tg_fetch_output */
int tg_reduce_to_index_file(tg_ctx* ctx, const tg_kv_desc* desc, const tg_block* in_blocks, size_t n_in_blocks,
                            uint64_t result_size, const void* neutral_item16, size_t* out_items, uint64_t* out_begin);

/* The same two operators with HOST Files on both sides (the drop-in call: GpuSortNode::Execute /
 * GpuReduceNode::StopPreOp in thrill_b200/host/): gathers the input Blocks to the device, runs the
 * operator, reports the output size; tg_fetch_output then scatters the result into caller-allocated
 * ByteBlocks and releases it. */
int tg_sort_file(tg_ctx* ctx, const tg_key_desc* desc, const tg_block* in_blocks, size_t n_in_blocks,
                 uint64_t rng_seed, size_t* out_items);
int tg_reduce_file(tg_ctx* ctx, const tg_kv_desc* desc, const tg_block* in_blocks, size_t n_in_blocks,
                   size_t* out_items);
int tg_fetch_output(tg_ctx* ctx, const tg_block_mut* out_blocks, size_t n_out_blocks);

/* ---- device-resident Files: GPU node -> GPU node without the PCIe round trip (SURVEY.md §8f-2) ----------------------
 * The reference hands a node's result to its children as a data::File (DIANode::PushFile -> child->OnPreOpFile,
 * api/dia_node.hpp:156-180; api/sort.hpp:151-175 takes it whole).  When the child is another GPU node the File need not
 * exist on the host at all: the parent keeps its result as a device File: flat items in HBM, the same layout as the
 * concatenated Blocks, and the child's operator reads it there.  A host File is materialised only when a child that is
 * not a GPU node asks for it (tg_dev_file_fetch: the lazy D2H of a PinnedBlock, data/block.hpp:116). */
typedef struct {
    void* dptr;                /* HBM buffer owned by the handle (tg_dev_file_free) */
    uint64_t items;
    uint32_t item_bytes;
    uint32_t reserved;
} tg_dev_file;
/* take the result of the last *_file / *_dev operator as a device File instead of fetching it (tg_fetch_output) */
int tg_output_detach(tg_ctx* ctx, tg_dev_file* out);
int tg_dev_file_fetch(tg_ctx* ctx, const tg_dev_file* f, const tg_block_mut* out_blocks, size_t n_out_blocks);
int tg_dev_file_free(tg_ctx* ctx, tg_dev_file* f);
/* the operators with a device File as input (the handle is left intact: a DIA may have several children) */
int tg_sort_dev(tg_ctx* ctx, const tg_key_desc* desc, const tg_dev_file* in, uint64_t rng_seed, size_t* out_items);
int tg_reduce_dev(tg_ctx* ctx, const tg_kv_desc* desc, const tg_dev_file* in, size_t* out_items);
int tg_reduce_to_index_dev(tg_ctx* ctx, const tg_kv_desc* desc, const tg_dev_file* in, uint64_t result_size,
                           const void* neutral_item16, size_t* out_items, uint64_t* out_begin);
/* bytes this ctx has moved over PCIe through the File codec since tg_init (tests: a GPU -> GPU chain moves none in between) */
int tg_transfer_bytes(const tg_ctx* ctx, uint64_t* out_h2d, uint64_t* out_d2h);

/* ---- Merge: k globally sorted DIAs into one (DIA::Merge / api::Merge, api/merge.hpp:75-721) --------------------------------
 * Each input is sorted by the descriptor across the workers (worker w's shard is sorted and precedes worker w+1's).  The result is
 * the sorted sequence of all N items in the order (key, input index, global position within the input) — one of the outcomes the
 * reference allows (it leaves equal items of different inputs in unspecified order) — split so that worker d holds the global
 * ranks [ceil(d*N/p), ceil((d+1)*N/p)).  The reference balances by a randomised multi-sequence selection (MainOp, :465-700); here the
 * selection is exact: the key of the item at each boundary rank is found one key byte per round on the device (one ncclAllReduce
 * of 255 counts per boundary per round), then the per-input counts below / equal to it fix the pieces (tg_merge_plan).  The local
 * merge of the k runs is a tree of stable 2-way merge-path passes (ceil(log2 k) passes; it replaces the multiway merge tree of
 * PushData, :160-190).  8- or 16-byte items with any key descriptor tg_sort takes for them; desc->stable
 * is ignored (the result is always deterministic); records, k < 2 and k > 16 are TG_ERR_ARG.  Inputs are read, never modified.
 * Output of unsorted inputs is unspecified (a permutation of the items), as in the reference. */
/* on device buffers; *out_dptr as for tg_sort (ctx-owned, valid until the next operator call).  Collective. */
int tg_merge(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_inputs, const size_t* n_inputs, uint32_t k,
             void** out_dptr, size_t* out_n);
/* the drop-in call (GpuMergeNode::Execute): input j is a device File (dev != NULL) or a host File (its Blocks); the result is
 * fetched with tg_fetch_output or taken with tg_output_detach.  Device Files are left intact. */
typedef struct {
    const tg_dev_file* dev;
    const tg_block* blocks;
    size_t nblocks;
} tg_merge_input;
int tg_merge_file(tg_ctx* ctx, const tg_key_desc* desc, const tg_merge_input* inputs, uint32_t k, size_t* out_items);
/* kernel level (parity tests): the selection of the p-worker operator for p simulated workers on one device, with the sum over
 * the simulated workers' runs in place of the all-reduce.  d_runs[w*k + j] = worker w's shard of input j; writes
 * out_bounds[(w*k + j)*(p+1) + d] = the first position of run (w, j) that goes to worker d (d = 0..p). */
int tg_merge_select(tg_ctx* ctx, const tg_key_desc* desc, const void* const* d_runs, const size_t* n_runs, uint32_t p,
                    uint32_t k, uint64_t* out_bounds);
/* The split arithmetic of Merge, pure host code (every worker derives the same plan; exported so that the p > 1 logic is
 * testable without GPUs).  For runs r = w*k + j and d = 0..p, at index r*(p+1) + d: less / equal = items of run r below / equal
 * to K_d, the key of the item at merged rank targets[d].  bounds = less + clamp(targets[d] - sum(less) - sum(equal of the runs
 * before (j, w) in input-major order), 0, equal).  TG_ERR_ARG if the counts are inconsistent: targets decreasing, targets[d]
 * outside [sum(less), sum(less + equal)], or bounds of a run decreasing in d. */
int tg_merge_plan(uint32_t p, uint32_t k, const uint64_t* targets, const uint64_t* less, const uint64_t* equal,
                  uint64_t* out_bounds);

/* ---- InnerJoin: DIA<pair<u64, V1>> ⋈ DIA<pair<u64, V2>> on .first (api::InnerJoin, api/inner_join.hpp:700-830) ---------------------
 * Both inputs are 16-byte items (uint64_t key, 8-byte value: any type, copied as bits).  Every pair (l, r) with l.first == r.first
 * gives one output item, by join_fn:
 *   TG_JOIN_KEY_VALUES  std::tuple<uint64_t, V1, V2> = (key, l.second, r.second), 24 bytes: serialized member by member in get<0..2>
 *                       order (data/serialization.hpp:89-178), so the device layout is (key, v1, v2)
 *   TG_JOIN_VALUES      std::pair<V1, V2> = (l.second, r.second), 16 bytes
 * Placement: worker Hash128to64(0, key) % p owns a key (as in ReduceByKey).  The reference's JoinNode (:61-481) exchanges both
 * sides by that hash, sorts each side locally and joins by a sort-merge on the host; here each side goes through one exchange
 * (the partition pass storing into the owners' windows), a stable local radix sort by the key, then a co-rank count (merge path
 * over left and right), an exclusive scan of the match counts and a load-balanced emit kernel (each CTA a range of the output).
 * Order within a worker: ascending key, then the left item's global position, then the right item's (global position = position
 * in the concatenation of the workers' shards).  This is one of the outcomes the reference allows; it leaves equal keys unordered
 * and, with location detection, may place keys elsewhere, so comparisons with it are on the multiset.  Key 0 is an ordinary key.
 * Inputs are read, never modified; an empty side gives an empty result.  item_bytes other than 16 or an unknown join_fn is
 * TG_ERR_ARG.  The largest output count of any worker is agreed on (all-reduce) before output memory is allocated, so an output of
 * 2^30 or more items on any worker is TG_ERR_TOO_LARGE on every rank.  Host round trips: with p > 1 three (the two count matrices
 * of the exchanges and the output-size all-reduce), with p = 1 one (the output size).  Collective. */
enum { TG_JOIN_KEY_VALUES = 0, TG_JOIN_VALUES = 1 };
typedef struct {
    uint32_t item_bytes;       /* 16, both inputs */
    uint32_t join_fn;          /* TG_JOIN_* */
} tg_join_desc;
/* device buffers; *out_dptr as for tg_sort (ctx-owned, valid until the next operator call).  Collective. */
int tg_inner_join(tg_ctx* ctx, const tg_join_desc* desc, const void* d_left, size_t n_left, const void* d_right, size_t n_right,
                  void** out_dptr, size_t* out_n);
/* the drop-in call (GpuJoinNode::Execute): each side a host File (Blocks) or a device File (read in place, left intact); the
 * result is fetched with tg_fetch_output or taken with tg_output_detach (item_bytes 24 or 16) */
int tg_inner_join_file(tg_ctx* ctx, const tg_join_desc* desc, const tg_merge_input* left, const tg_merge_input* right,
                       size_t* out_items);

/* ---- GroupByKey / GroupToIndex: a DIA<pair<u64, V>> grouped by .first (DIA::GroupByKey, api/group_by_key.hpp:46-428;
 * DIA::GroupToIndex, api/group_to_index.hpp:36-290) ---------------------------------------------------------------------------
 * The reference's nodes work in two halves: MainOp exchanges every item to the owner of its key and sorts each worker's share by
 * the key (group_by_key.hpp:348-376, group_to_index.hpp:234-254); PushData walks the sorted items and calls the user's group
 * function once per group (group_by_key.hpp:204-331, group_to_index.hpp:116-215).  These entry points replace the first half;
 * the group function, with its arbitrary output type, stays on the host (GpuGroupNode in thrill_b200/host/).  The result of a
 * worker is its share of the 16-byte items (uint64_t key, 8-byte value: any type, copied as bits) sorted by the key, and stable:
 * equal keys keep their global input order (global position = position in the concatenation of the workers' shards).  The
 * reference sorts with std::sort and leaves that order open; this is one of the orders it allows.
 * Placement:
 *   GroupByKey    worker key % p owns a key: hash_function(key) % p (group_by_key.hpp:149-159) with the default hash
 *                 std::hash<uint64_t>, the identity in libstdc++ (:419-428).  (Not ReduceByKey's Hash128to64.)
 *   GroupToIndex  worker k * p / result_size owns index k (CalculatePartition, group_to_index.hpp:98-105): worker r answers for
 *                 [*out_begin, *out_end) = Range(0, result_size).Partition(r, p) = [ceil(r * size / p), ceil((r+1) * size / p)),
 *                 ReduceToIndex's ranges.  An index >= result_size (an assert in the reference) is TG_ERR_ARG on every rank: such
 *                 items go to the last worker, whose verdict an all-reduce hands to the others.  A result_size with
 *                 (result_size - 1) * p >= 2^64 is TG_ERR_ARG.
 * The input is read, never modified; 2^30 or more items on a worker, before or after the exchange, is TG_ERR_TOO_LARGE on every
 * rank (the exchange's count matrix decides it).  Host round trips: GroupByKey none with p = 1, one with p > 1 (the count matrix);
 * GroupToIndex one with p = 1 (the index check), two with p > 1 (the count matrix and the all-reduce of the index check).
 * Collective. */
/* on device buffers; *out_dptr as for tg_sort (ctx-owned, valid until the next operator call) */
int tg_group_by_key(tg_ctx* ctx, const void* d_in, size_t n_local, void** out_dptr, size_t* out_n);
int tg_group_to_index(tg_ctx* ctx, const void* d_in, size_t n_local, uint64_t result_size, void** out_dptr, size_t* out_n,
                      uint64_t* out_begin, uint64_t* out_end);
/* the drop-in calls (GpuGroupNode::Execute): the input is a host File (Blocks) or a device File (read in place, left intact); the
 * result (16-byte items) is fetched with tg_fetch_output or taken with tg_output_detach */
int tg_group_by_key_file(tg_ctx* ctx, const tg_merge_input* in, size_t* out_items);
int tg_group_to_index_file(tg_ctx* ctx, const tg_merge_input* in, uint64_t result_size, size_t* out_items,
                           uint64_t* out_begin, uint64_t* out_end);
/* kernel level (tests of the placement on one GPU): GroupByKey's partition, destination of a 16-byte item = key % p.  Stable:
 * d_out receives the items grouped by destination in input order, out_counts[p] (host) the counts.  1 <= p <= 256. */
int tg_mod_partition(tg_ctx* ctx, const void* d_in, size_t n, uint32_t p, void* d_out, uint64_t* out_counts);

/* ---- PrefixSum / ExPrefixSum / ZipWithIndex: scans by global position (DIA::PrefixSum, DIA::ExPrefixSum, api/dia.hpp:1850,
 * :1867, PrefixSumNode api/prefix_sum.hpp:28-128; DIA::ZipWithIndex, ZipWithIndexNode api/zip_with_index.hpp:40-110) -----------
 * Every worker keeps its items, in order: one output per input item, no rebalancing (prefix_sum.hpp:92-110,
 * zip_with_index.hpp:96-110).  The stock PrefixSumNode folds each worker's local total from the value-initialised item T(), not
 * from the initial element: S_w = ((T() + x_0) + x_1) ... (prefix_sum.hpp:43, :56-59, :72-77), an empty worker contributes T().
 * Worker r's carry is net.ExPrefixSum(S_r, +, initial) (:85-90), with thread workers on one host (net/flow_control_channel.hpp:
 * 236-290) carry_0 = initial and carry_r = initial + (S_0 + ... + S_{r-1}), the inner fold left to right.  Then
 *   inclusive  out_i = carry + x_0 + ... + x_i          exclusive  out_0 = carry, out_i = carry + x_0 + ... + x_{i-1}
 * The descriptor set (the host shim recognises the sum function, thrill_b200/host/):
 *   item_bytes 8   uint64_t with TG_OP_SUM_U64 (std::plus, wraps modulo 2^64), TG_OP_MIN_U64, TG_OP_MAX_U64 (thrill_gpu::MinU64 /
 *                  MaxU64; with MinU64, T() = 0 absorbs everything, so every output of a worker r >= 1 is 0); double with
 *                  TG_OP_SUM_F64 (std::plus<double>; local totals start from +0.0)
 *   item_bytes 16  std::pair<uint64_t, V> (V any 8-byte value) with thrill_gpu::ScanSecond<F>: a + b = (b.first, F(a.second,
 *                  b.second)), op = F's TG_OP_* as above.  So out_i.first is x_i.first (inclusive) or x_{i-1}.first (exclusive;
 *                  carry.first for i = 0, which is the .first of worker r-1's last item, 0 if that worker is empty, and
 *                  initial.first on worker 0)
 * Anything else (TG_OP_MIN_F64, TG_OP_MAX_F64, TG_OP_FIRST, other item sizes) is TG_ERR_ARG.  Integer results are exact; double
 * sums are bracketed by tiles (reduce-then-scan), the same way on every run, so a result is always bitwise reproducible.  Let
 * exact_i be the exact sum of initial and every item folded into output i (the lower workers' items included), A_i the same
 * sum over |x|, u = 2^-53 and gamma_D = D u / (1 - D u), where D is the longest chain of additions a summand goes through:
 *   D = 2k + R + max(50, 42 + p),  k = 16 (8-byte items) or 8 (pairs),  R = ceil(tiles / 4096) of the largest worker (>= 1)
 * (146 for 8-byte items and 194 for pairs at 2^30 - 1 items on one worker).  While (1 + gamma_D) A_i < DBL_MAX, no partial sum
 * can overflow, and then |out_i - exact_i| <= gamma_D A_i + u |exact_i|; NaN where the prefix has seen a NaN or both
 * infinities, the infinity where it has seen one, and the sign of a zero (-0.0 only where every summand is -0.0) are exactly
 * the stock fold's.  Beyond that range a partial sum of the bracketing may overflow where none of the stock fold's does: with
 * x_0 = -1e308, x_4096 = x_4097 = 1e308 and +0.0 elsewhere the stock fold ends at 1e308, and the tile scan can give +inf.
 * ZipWithIndex takes 8-byte items (any value, copied as bits) and gives 16-byte pairs: index_first != 0 gives (index, item)
 * (thrill_gpu::IndexFirst), index_first == 0 gives (item, index) (thrill_gpu::IndexSecond); index = the item's global position.
 * Collective flow: p = 1 has no host round trip.  With p > 1 one ncclAllGather of a 32-byte record per worker (n_local and S_r)
 * into device memory, then one host read of the gathered sizes: n_local >= 2^30 on any worker is TG_ERR_TOO_LARGE on every rank.
 * The carry is folded on the device from the gathered totals; ZipWithIndex's base index is the sum of the lower ranks' sizes.
 * Inputs are read, never modified.  Collective. */
typedef struct {
    uint32_t item_bytes;       /* 8 or 16 */
    uint32_t op;               /* TG_OP_SUM_F64 (8-byte items only: double), TG_OP_SUM_U64, TG_OP_MIN_U64, TG_OP_MAX_U64 */
} tg_scan_desc;
/* on device buffers; initial_item: item_bytes bytes on the host (NULL: T(), all zero bytes); inclusive: PrefixSum (1) or
 * ExPrefixSum (0).  *out_dptr holds n_local items, as for tg_sort (ctx-owned, valid until the next operator call). */
int tg_prefix_sum(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                  int inclusive, void** out_dptr, size_t* out_n);
int tg_zip_with_index(tg_ctx* ctx, const void* d_in, size_t n_local, int index_first, void** out_dptr, size_t* out_n);
/* the drop-in calls (GpuPrefixSumNode / GpuZipWithIndexNode::Execute): the input is a host File (Blocks) or a device File (read in
 * place, left intact); the result is fetched with tg_fetch_output or taken with tg_output_detach */
int tg_prefix_sum_file(tg_ctx* ctx, const tg_scan_desc* desc, const tg_merge_input* in, const void* initial_item, int inclusive,
                       size_t* out_items);
int tg_zip_with_index_file(tg_ctx* ctx, const tg_merge_input* in, int index_first, size_t* out_items);
/* kernel level (p workers simulated on one GPU): the local total S of n items (what a worker contributes to the all-gather), as
 * one item of desc->item_bytes bytes into host memory */
int tg_scan_local_total(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n, void* out_total_item);
/* ... and worker `rank` of p (1 <= p <= 16): the operator's device path with totals (p items on the host, from
 * tg_scan_local_total) in place of the all-gather, carry fold included; sizes[p] (host) are the workers' item counts, of which
 * ZipWithIndex takes its base index.  Outputs as for tg_prefix_sum / tg_zip_with_index. */
int tg_prefix_sum_select(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, uint32_t rank, uint32_t p,
                         const void* totals, const void* initial_item, int inclusive, void** out_dptr, size_t* out_n);
int tg_zip_with_index_select(tg_ctx* ctx, const void* d_in, size_t n_local, uint32_t rank, uint32_t p, const uint64_t* sizes,
                             int index_first, void** out_dptr, size_t* out_n);

/* ---- Sum / Min / Max / AllReduce: a DIA reduced to one value on every worker (DIA::Sum, Min, Max, AllReduce: api/sum.hpp,
 * min.hpp, max.hpp, AllReduceNode api/all_reduce.hpp:27-85) ---------------------------------------------------------------------
 * Worker value S_r: the worker folds its items left to right starting from its FIRST item, not from an identity
 * (all_reduce.hpp:56-63): S_r = ((x_0 + x_1) + x_2) ...  With an initial value (Sum(fn, initial), Min(initial), Max(initial),
 * AllReduce(fn, initial)) worker 0 starts from it instead and folds every item into it.  A worker with no items contributes T(),
 * the value-initialised item (0, +0.0, (0, 0)), or, when there is an initial value, the initial value: the stock node's value
 * starts as the initial value on every worker, and a worker other than 0 replaces it with its first item (:39-46).  So with an
 * empty worker the Min() of positive uint64_t values is 0, the Min() of doubles is at most +0.0, and Sum(fn, initial) counts the
 * initial value once more for every empty worker other than worker 0, exactly as in the stock node.
 * Result: the left fold of the worker values in rank order, v = S_0, v = v + S_r for r = 1..p-1 (FlowControlChannel::AllReduce
 * with the thread workers of one host, net/flow_control_channel.hpp:599-638); every rank gets the same value.
 * The descriptor set (tg_scan_desc; the host shim recognises the function, thrill_b200/host/):
 *   item_bytes 8   uint64_t with TG_OP_SUM_U64 (std::plus, wraps modulo 2^64), TG_OP_MIN_U64 (thrill_gpu::MinU64,
 *                  common::minimum<uint64_t>), TG_OP_MAX_U64 (MaxU64, common::maximum<uint64_t>); double with TG_OP_SUM_F64
 *                  (std::plus<double>), TG_OP_MIN_F64 (common::minimum<double>), TG_OP_MAX_F64 (common::maximum<double>)
 *   item_bytes 16  std::pair<uint64_t, V> with thrill_gpu::ScanSecond<F>, F any function above: .first comes from the right-hand
 *                  operand, so the result's .first is the .first of the last worker's last item; if that worker is empty, the
 *                  .first of what it contributes (0, or the initial value's)
 * Anything else (TG_OP_FIRST, other item sizes) is TG_ERR_ARG.  Integer results are exact.  Min / Max on doubles are exact bit for
 * bit: std::min(a, b) = b < a ? b : a (std::max: a < b ? b : a), so a NaN as the first operand of a fold sticks (a worker's first
 * item, the initial value on worker 0, S_0 in the fold of the workers) and the result has that NaN's bits; a NaN anywhere else is
 * skipped; of equal values the earliest wins (-0.0 and +0.0: the sign of a zero minimum is the earlier zero's).  The tile
 * reduce folds positions in order with a NaN-skipping function, and the first operand goes through the stock function on its
 * own.  Double sums are bracketed by tiles and then in a fixed order (no CTA waits on another, no atomics), so a result is
 * bitwise reproducible from run to run.  Let exact be the exact sum of the initial value and every item, A the same sum over
 * |x|, u = 2^-53 and gamma_D = D u / (1 - D u), where D is the longest chain of additions a summand goes through:
 *   D = k + 31 + ceil(T / 512) + p,  k = 16 (8-byte items) or 8 (pairs),  T = the tiles of the largest worker (32 KB each)
 * (k - 1 in a thread's run, 5 lanes, 7 warps of the tile reduce; ceil(T / 512) in a thread's run of aggregates, 5 lanes, 15 warps
 * of the fold; 1 for the initial value; p - 1 for the workers).  D = 559 + p for 8-byte items at 2^30 - 1 items on a worker.
 * While (1 + gamma_D) A < DBL_MAX, |out - exact| <= gamma_D A + u |exact|; NaN where the items hold a NaN or both infinities,
 * the infinity where they hold one, and the sign of a zero (-0.0 exactly when every summand is -0.0, the T() = +0.0 of an empty
 * worker included) are the stock fold's.  A NaN's payload is left open for sums.
 * Limits: at most 2^30 - 1 items per worker; more on any worker is TG_ERR_TOO_LARGE on every rank (the sizes travel in the
 * all-gather).  Collective flow: p = 1 has one host round trip (reading the value back).  With p > 1 one ncclAllGather of a
 * 32-byte record per worker (n_local, .first, S_r) into device memory, the fold on the device, then one host read of the sizes
 * and the value.  Inputs are read, never modified.  Collective. */
/* on a device buffer; initial_item: item_bytes bytes on the host (NULL: none); out_item: item_bytes bytes on the host */
int tg_all_reduce(tg_ctx* ctx, const tg_scan_desc* desc, const void* d_in, size_t n_local, const void* initial_item,
                  void* out_item);
/* the drop-in call (GpuAllReduceNode::Execute): a host File (Blocks) or a device File (read in place, left intact) */
int tg_all_reduce_file(tg_ctx* ctx, const tg_scan_desc* desc, const tg_merge_input* in, const void* initial_item, void* out_item);
/* kernel level (1 <= p <= 16 workers simulated on one device): shard w (n_shards[w] items at d_shards[w]) is worker w, which
 * takes the initial value if w == 0.  Runs the operator's device code with each worker's record written into the slot the
 * all-gather fills, then the fold; writes the result every rank would get.  Shards are read, never modified; a shard of 2^30 or
 * more items is TG_ERR_TOO_LARGE. */
int tg_all_reduce_select(tg_ctx* ctx, const tg_scan_desc* desc, const void* const* d_shards, const size_t* n_shards, uint32_t p,
                         const void* initial_item, void* out_item);

/* ---- synthetic inputs of SURVEY.md §8(d), generated on the device (bench / tests support) ------------ */
int tg_gen_sort_uniform(tg_ctx* ctx, void* d_out, uint64_t begin, uint64_t n, uint64_t seed);
int tg_gen_reduce_uniform(tg_ctx* ctx, void* d_out, uint64_t begin, uint64_t n, uint64_t seed,
                          uint64_t universe, int exact);
/* d_cdf: universe doubles (cumulative Zipf table built on the host exactly as
 * common/zipf_distribution.hpp:119-140 and uploaded once) */
int tg_gen_sort_zipf(tg_ctx* ctx, void* d_out, uint64_t begin, uint64_t n, uint64_t seed,
                     const void* d_cdf, uint64_t universe);
int tg_gen_reduce_zipf(tg_ctx* ctx, void* d_out, uint64_t begin, uint64_t n, uint64_t seed,
                       const void* d_cdf, uint64_t universe, int exact);
int tg_gen_records(tg_ctx* ctx, void* d_out, uint64_t begin, uint64_t n, uint64_t seed);
/* order-independent 64-bit checksum of n items (sum and xor of a per-item hash) and sortedness check;
 * used by the full-size parity properties (sortedness + multiset preservation) */
int tg_checksum(tg_ctx* ctx, const void* d_items, size_t n, uint32_t item_bytes, uint64_t out_sum_xor[2]);
int tg_is_sorted(tg_ctx* ctx, const tg_key_desc* desc, const void* d_items, size_t n, uint64_t* out_violations);

#ifdef __cplusplus
}
#endif
#endif /* THRILL_GPU_H */
