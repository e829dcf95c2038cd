/*******************************************************************************
 * thrill_b200/host/thrill_gpu_nodes.hpp — the C++ host side of the drop-in.
 *
 * Two DOpNode classes with exactly the StageBuilder protocol of the reference's SortNode
 * (thrill/api/sort.hpp:64-271) and ReduceNode (thrill/api/reduce_by_key.hpp:64-211), and the front doors
 *     thrill_gpu::Sort(dia [, std::less<T>/std::greater<T>])     <->  DIA<T>::Sort      (api/sort.hpp:800)
 *     thrill_gpu::ReducePair(dia, std::plus<double> ...)          <->  DIA<T>::ReducePair(api/reduce_by_key.hpp:410)
 *     thrill_gpu::Merge(std::less<T>(), dia0, dia1, ...)          <->  api::Merge        (api/merge.hpp:673)
 *     thrill_gpu::InnerJoin(l, r, KeyFirst(), KeyFirst(), JoinValues()) <->  api::InnerJoin (api/inner_join.hpp:700)
 *     thrill_gpu::GroupByKey<Out>(dia, KeyFirst(), fn)            <->  DIA<T>::GroupByKey (api/group_by_key.hpp:419)
 *     thrill_gpu::GroupToIndex<Out>(dia, KeyFirst(), fn, size)    <->  DIA<T>::GroupToIndex (api/group_to_index.hpp:257)
 *     thrill_gpu::PrefixSum(dia, fn [, initial]) / ExPrefixSum    <->  DIA<T>::PrefixSum / ExPrefixSum (api/dia.hpp:1850, :1867)
 *     thrill_gpu::ZipWithIndex(dia, IndexFirst() | IndexSecond()) <->  DIA<T>::ZipWithIndex (api/zip_with_index.hpp:140)
 *     thrill_gpu::Sum / Min / Max / AllReduce (dia, ...) [Future]  <->  DIA<T>::Sum / Min / Max / AllReduce (api/sum.hpp, ...)
 *     thrill_gpu::Size(dia) / SizeFuture(dia)                     <->  DIA<T>::Size / SizeFuture (api/size.hpp)
 * Everything else of the pipeline (sources, LOps, other DOps, actions, the net/data layers) is the
 * UNMODIFIED reference library: this header only includes it.  The heavy lifting happens behind the C ABI
 * of include/thrill_gpu.h (libthrill_gpu.so): the nodes hand the Blocks of their input data::File to
 * tg_sort_file / tg_reduce_file and wrap the result bytes in fresh ByteBlocks of the worker's BlockPool with
 * the geometry BlockWriter would have produced (tg_file_geometry), so children see an ordinary data::File
 * (PushFile, thrill/api/dia_node.hpp:156-180).
 *
 * One Thrill worker thread = one GPU = one tg_ctx (device = Context::local_worker_id()); the NCCL id is
 * created by worker 0 and broadcast over the reference's own control plane (ctx.net.Broadcast,
 * net/flow_control_channel.hpp:424).  Only a closed set of (type, functor) pairs maps to a descriptor;
 * anything else is a compile-time error (static_assert) — there is no CPU fallback inside these nodes:
 * a user who wants the CPU path calls the stock dia.Sort() / dia.ReducePair().
 * Requires Release builds (common::g_self_verify == false, common/config.hpp:32), which is asserted.
 ******************************************************************************/
#pragma once
#ifndef THRILL_GPU_NODES_HEADER
#define THRILL_GPU_NODES_HEADER

#include <thrill/api/action_node.hpp>
#include <thrill/api/dia.hpp>
#include <thrill/api/dop_node.hpp>
#include <thrill/common/config.hpp>
#include <thrill/common/functional.hpp>
#include <thrill/data/file.hpp>
#include <tlx/meta/call_foreach_with_index.hpp>
#include <tlx/meta/vexpand.hpp>

#include <array>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/thrill_gpu.h"

namespace thrill_gpu {

using thrill::api::Context;
using thrill::api::DIA;
using thrill::api::DIAMemUse;

//! non-zero status of the C ABI -> die() (tlx::DieException), the reference's error path
inline void Check(tg_ctx* c, int status, const char* what) {
    if (status != TG_OK)
        die("thrill_gpu: " << what << " failed: " << tg_strerror(status) << ": " << tg_last_error(c));
}

//! One tg_ctx per worker THREAD, created on first use (collective: every worker must reach its first GPU node) and shut
//! down when the thread ends.  api::Run starts every worker on a thread of its own (api/context.cpp:RunLoopbackThreads /
//! RunBackendLoopback), so the ctx — stream, workspaces, exchange window, NCCL communicator — lives exactly as long as the
//! job's Context does: a second api::Run in the same process gets fresh threads and a fresh ctx, never a stale one.  On a
//! hit the cached ctx is checked against the Context (a re-used thread, api::RunLocalSameThread) and rebuilt if it differs.
struct WorkerCtxHolder {
    tg_ctx* c = nullptr;
    const Context* owner = nullptr;
    size_t rank = 0, nranks = 0;
    void Reset() { if (c) tg_shutdown(c); c = nullptr; owner = nullptr; }
    ~WorkerCtxHolder() { Reset(); }
};

inline tg_ctx * WorkerCtx(Context& ctx) {
    static thread_local WorkerCtxHolder holder;
    if (holder.c && holder.owner == &ctx && holder.rank == ctx.my_rank() && holder.nranks == ctx.num_workers())
        return holder.c;
    holder.Reset();
    die_unless(!thrill::common::g_self_verify);     // Debug builds prefix every item with a typecode
    using Id = std::array<char, 128>;
    Id id;
    id.fill(0);
    if (ctx.num_workers() > 1) {
        if (ctx.my_rank() == 0) Check(nullptr, tg_get_unique_id(id.data()), "tg_get_unique_id");
        id = ctx.net.Broadcast(id, 0);
    }
    // worker -> GPU: the worker's index on its host (api/context.hpp: local_worker_id).  The in-process test networks
    // (THRILL_NET=mock/local with several "hosts") put every host's workers into this one process: there the global rank
    // picks the GPU, and two workers are never given the same device (NCCL and the peer mapping both need distinct GPUs).
    int ndev = tg_device_count();
    if (ndev <= 0) die("thrill_gpu: no sm_90 GPU visible (there is no CPU fallback in the GPU nodes)");
    size_t device = ctx.local_worker_id();
    const char* net = getenv("THRILL_NET");
    if (ctx.num_hosts() > 1 && net && (!strcmp(net, "mock") || !strcmp(net, "local"))) device = ctx.my_rank();
    if (device >= static_cast<size_t>(ndev))
        die("thrill_gpu: worker " << ctx.my_rank() << " needs GPU " << device << " but only " << ndev << " are visible "
            "(run with THRILL_WORKERS_PER_HOST <= number of GPUs)");
    tg_ctx* c = nullptr;
    int st = tg_init(static_cast<int>(device), static_cast<int>(ctx.my_rank()),
                     static_cast<int>(ctx.num_workers()), id.data(), &c);
    Check(c, st, "tg_init");
    holder.c = c;
    holder.owner = &ctx;
    holder.rank = ctx.my_rank();
    holder.nranks = ctx.num_workers();
    return c;
}

/******************************************************************************/
// descriptors of the recognised (type, functor) pairs

template <typename ValueType, typename Compare, typename Enable = void>
struct SortDesc {
    static constexpr bool supported = false;
};
//! Items whose order is the lexicographic order of a run of key bytes (TeraSort's Record{uint8 key[10]; uint8 value[90]} with
//! operator< = std::lexicographical_compare of the keys, examples/terasort/terasort.cpp:31-42): specialise for the item type
//!   template <> struct thrill_gpu::ByteKeyTraits<Record> { static constexpr bool is_byte_key = true;
//!                                                          static constexpr uint32_t key_offset = 0, key_bytes = 10; };
//! and thrill_gpu::Sort(dia) / Sort(dia, std::less<Record>()) take the GPU path (key_bytes <= 12, sizeof(T) % 4 == 0).
template <typename ValueType>
struct ByteKeyTraits {
    static constexpr bool is_byte_key = false;
};
template <typename ValueType>
struct SortDesc<ValueType, std::less<ValueType>, typename std::enable_if<ByteKeyTraits<ValueType>::is_byte_key>::type>{
    static_assert(sizeof(ValueType) % 4 == 0 && ByteKeyTraits<ValueType>::key_bytes <= 12 &&
                  ByteKeyTraits<ValueType>::key_offset + ByteKeyTraits<ValueType>::key_bytes <= sizeof(ValueType),
                  "byte-key records: sizeof % 4 == 0 and a key of at most 12 bytes inside the item");
    static constexpr bool supported = true;
    static tg_key_desc make() {
        return tg_key_desc { static_cast<uint32_t>(sizeof(ValueType)), ByteKeyTraits<ValueType>::key_offset,
                             ByteKeyTraits<ValueType>::key_bytes, TG_KEY_BYTES_BE, 0, 0 };
    }
};
template <typename Compare>
struct SortDesc<uint64_t, Compare, typename std::enable_if<
                    std::is_same<Compare, std::less<uint64_t> >::value ||
                    std::is_same<Compare, std::greater<uint64_t> >::value>::type>{
    static constexpr bool supported = true;
    static tg_key_desc make() {
        return tg_key_desc { 8, 0, 8, TG_KEY_UINT_LE,
                             std::is_same<Compare, std::greater<uint64_t> >::value ? 1u : 0u, 0 };
    }
};
//! pair<uint64_t, 8-byte POD> ordered by .first (serialized member-wise as 16 bytes, data/serialization.hpp:67-84)
struct LessFirst {
    template <typename P>
    bool operator () (const P& a, const P& b) const { return a.first < b.first; }
};
template <typename V>
struct SortDesc<std::pair<uint64_t, V>, LessFirst,
                typename std::enable_if<sizeof(V) == 8 && std::is_pod<V>::value>::type>{
    static constexpr bool supported = true;
    static tg_key_desc make() { return tg_key_desc { 16, 0, 8, TG_KEY_UINT_LE, 0, 1 }; }
};

template <typename Value, typename ReduceFunction>
struct ReduceDesc {
    static constexpr bool supported = false;
};
template <>
struct ReduceDesc<double, std::plus<double> >{
    static constexpr bool supported = true;
    static constexpr uint32_t op = TG_OP_SUM_F64;
};
template <>
struct ReduceDesc<uint64_t, std::plus<uint64_t> >{
    static constexpr bool supported = true;
    static constexpr uint32_t op = TG_OP_SUM_U64;
};
struct MinU64 { uint64_t operator () (uint64_t a, uint64_t b) const { return b < a ? b : a; } };
struct MaxU64 { uint64_t operator () (uint64_t a, uint64_t b) const { return a < b ? b : a; } };
template <>
struct ReduceDesc<uint64_t, MinU64>{
    static constexpr bool supported = true;
    static constexpr uint32_t op = TG_OP_MIN_U64;
};
template <>
struct ReduceDesc<uint64_t, MaxU64>{
    static constexpr bool supported = true;
    static constexpr uint32_t op = TG_OP_MAX_U64;
};

//! The functors thrill_gpu::ReduceByKey recognises (DIA::ReduceByKey takes a key extractor and a reduce function over whole
//! items, api/reduce_by_key.hpp:312-363): the key is pair.first, the reduce function folds pair.second and keeps the key.
struct KeyFirst {
    template <typename P>
    const typename P::first_type& operator () (const P& p) const { return p.first; }
};
template <typename ValueFunction>
struct OnSecond {
    ValueFunction fn;
    template <typename P>
    P operator () (const P& a, const P& b) const { return P(a.first, fn(a.second, b.second)); }
};

//! The join functions thrill_gpu::InnerJoin recognises (api::InnerJoin takes any function of (left item, right item),
//! api/inner_join.hpp:700-827), on pair<uint64_t, V1> and pair<uint64_t, V2> joined on .first.  They are plain functors, so the
//! stock api::InnerJoin takes them too.
struct JoinKeyValues {
    template <typename L, typename R>
    std::tuple<uint64_t, typename L::second_type, typename R::second_type> operator () (const L& l, const R& r) const {
        return std::make_tuple(l.first, l.second, r.second);
    }
};
struct JoinValues {
    template <typename L, typename R>
    std::pair<typename L::second_type, typename R::second_type> operator () (const L& l, const R& r) const {
        return std::make_pair(l.second, r.second);
    }
};
//! out_bytes: the SERIALIZED output item size (std::tuple is written member by member, data/serialization.hpp:89-178)
template <typename JoinFunction>
struct JoinDesc { static constexpr bool supported = false; };
template <>
struct JoinDesc<JoinKeyValues>{
    static constexpr bool supported = true;
    static constexpr uint32_t fn = TG_JOIN_KEY_VALUES, out_bytes = 24;
};
template <>
struct JoinDesc<JoinValues>{
    static constexpr bool supported = true;
    static constexpr uint32_t fn = TG_JOIN_VALUES, out_bytes = 16;
};

//! The sum function thrill_gpu::PrefixSum / ExPrefixSum recognise on pair<uint64_t, V>: F (one of the ReducePair functions,
//! std::plus<double>, std::plus<uint64_t>, MinU64, MaxU64) on .second, .first taken from the right-hand operand.  Prefix doubling
//! names its suffixes with ScanSecond<MaxU64> (examples/suffix_sorting/prefix_doubling.cpp:348).  A plain functor with one
//! operator() (the stock nodes read its argument type), so the stock DIA::PrefixSum takes it too.
template <typename MemberFn> struct MemberResult;
template <typename R, typename C, typename... A>
struct MemberResult<R (C::*)(A...) const> { using type = typename std::decay<R>::type; };   // (common::minimum returns const T&)
template <typename ValueFunction>
struct ScanSecond {
    using Pair = std::pair<uint64_t, typename MemberResult<decltype(&ValueFunction::operator ())>::type>;
    ValueFunction fn;
    Pair operator () (const Pair& a, const Pair& b) const { return Pair(b.first, fn(a.second, b.second)); }
};
//! the (item type, sum function) pairs of PrefixSum / ExPrefixSum: uint64_t and double with their ReduceDesc functions, and
//! pair<uint64_t, V> with ScanSecond<F>
template <typename Value, typename SumFunction, bool = ReduceDesc<Value, SumFunction>::supported>
struct ScanOp { static constexpr bool supported = false; static constexpr uint32_t op = 0; };
template <typename Value, typename SumFunction>
struct ScanOp<Value, SumFunction, true>{
    static constexpr bool supported = true;
    static constexpr uint32_t op = ReduceDesc<Value, SumFunction>::op;
};
template <typename ValueType, typename SumFunction>
struct ScanDesc : ScanOp<ValueType, SumFunction> { static constexpr uint32_t item_bytes = 8; };
template <typename V, typename F>
struct ScanDesc<std::pair<uint64_t, V>, ScanSecond<F> >
    : ScanOp<typename std::conditional<std::is_same<V, typename ScanSecond<F>::Pair::second_type>::value, V, void>::type, F>{
    static constexpr uint32_t item_bytes = 16;
};
//! the (item type, function) pairs of Sum / Min / Max / AllReduce: those of PrefixSum, and common::minimum / common::maximum
//! (what the stock Min / Max use) on uint64_t and double, also inside ScanSecond<F> on pairs
template <typename Value, typename Function>
struct ActionOp : ScanOp<Value, Function> { };
template <uint32_t kOp>
struct ActionOpIs { static constexpr bool supported = true; static constexpr uint32_t op = kOp; };
template <>
struct ActionOp<uint64_t, thrill::common::minimum<uint64_t> >: ActionOpIs<TG_OP_MIN_U64> { };
template <>
struct ActionOp<uint64_t, thrill::common::maximum<uint64_t> >: ActionOpIs<TG_OP_MAX_U64> { };
template <>
struct ActionOp<double, thrill::common::minimum<double> >: ActionOpIs<TG_OP_MIN_F64> { };
template <>
struct ActionOp<double, thrill::common::maximum<double> >: ActionOpIs<TG_OP_MAX_F64> { };
template <typename ValueType, typename Function>
struct ActionDesc : ActionOp<ValueType, Function> { static constexpr uint32_t item_bytes = 8; };
template <typename V, typename F>
struct ActionDesc<std::pair<uint64_t, V>, ScanSecond<F> >
    : ActionOp<typename std::conditional<std::is_same<V, typename ScanSecond<F>::Pair::second_type>::value, V, void>::type, F>{
    static constexpr uint32_t item_bytes = 16;
};
//! The zip functions thrill_gpu::ZipWithIndex recognises on 8-byte items: (item, index) -> pair(index, item) or pair(item, index)
struct IndexFirst {
    template <typename T>
    std::pair<uint64_t, T> operator () (const T& item, const size_t& index) const { return std::pair<uint64_t, T>(index, item); }
};
struct IndexSecond {
    template <typename T>
    std::pair<T, uint64_t> operator () (const T& item, const size_t& index) const { return std::pair<T, uint64_t>(item, index); }
};

/******************************************************************************/
// shared File <-> C ABI plumbing

//! pin every Block of a File and describe it for the C ABI (replaces File::GetReader + per-item Next)
class PinnedFileView
{
public:
    PinnedFileView(const thrill::data::File& file, size_t local_worker_id) {
        pins_.reserve(file.num_blocks());
        blocks_.reserve(file.num_blocks());
        for (const thrill::data::Block& b : file.blocks()) {
            pins_.emplace_back(b.PinWait(local_worker_id));
            const thrill::data::PinnedBlock& pb = pins_.back();
            blocks_.push_back(tg_block { pb.data_begin(), pb.size() });
        }
    }
    const tg_block * data() const { return blocks_.data(); }
    size_t size() const { return blocks_.size(); }

private:
    std::vector<thrill::data::PinnedBlock> pins_;
    std::vector<tg_block> blocks_;
};

/******************************************************************************/
// GPU node -> GPU node hand-off without the PCIe round trip (SURVEY.md 8f-2)

//! A node result that lives in HBM (tg_dev_file); shared by the parent and the children it was handed to.
class DeviceFile
{
public:
    DeviceFile(tg_ctx* c, const tg_dev_file& f) : ctx_(c), f_(f) { }
    DeviceFile(const DeviceFile&) = delete;
    DeviceFile& operator = (const DeviceFile&) = delete;
    ~DeviceFile() { tg_dev_file_free(ctx_, &f_); }
    const tg_dev_file * get() const { return &f_; }
    size_t items() const { return f_.items; }

private:
    tg_ctx* ctx_;
    tg_dev_file f_;
};
using DeviceFilePtr = std::shared_ptr<DeviceFile>;

//! Implemented by the GPU nodes: a parent GPU node offers its device-resident result instead of a data::File.  The offer is
//! made inside the parent's PushData, i.e. between the child's StartPreOp and StopPreOp, exactly where OnPreOpFile would be
//! called (api/dia_node.hpp:156-180); a child whose function stack towards this parent is not empty declines.
class GpuNodeBase
{
public:
    virtual ~GpuNodeBase() { }
    //! parent_index: which of the child's parents makes the offer (DIANode::PushFile passes it to OnPreOpFile the same way,
    //! api/dia_node.hpp:156-177); a parent that feeds two inputs of one child offers once per edge
    virtual bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t parent_index) = 0;
};

//! materialise a device File as a host data::File (the lazy D2H, only for children that are not GPU nodes)
inline void FetchDeviceFileIntoFile(tg_ctx* c, Context& ctx, const DeviceFile& df, uint32_t item_bytes,
                                    thrill::data::File& out) {
    size_t num_items = df.items();
    size_t nblocks = tg_file_geometry(num_items, item_bytes, thrill::data::start_block_size,
                                      thrill::data::default_block_size, nullptr, 0);
    std::vector<tg_block_geom> geom(nblocks);
    tg_file_geometry(num_items, item_bytes, thrill::data::start_block_size,
                     thrill::data::default_block_size, geom.data(), geom.size());
    std::vector<thrill::data::PinnedByteBlockPtr> bytes;
    std::vector<tg_block_mut> targets;
    bytes.reserve(nblocks);
    for (const tg_block_geom& g : geom) {
        size_t cap = thrill::data::start_block_size;
        while (cap < g.bytes) cap *= 2;
        bytes.emplace_back(ctx.block_pool().AllocateByteBlock(cap, ctx.local_worker_id()));
        targets.push_back(tg_block_mut { bytes.back()->data(), static_cast<size_t>(g.bytes) });
    }
    Check(c, tg_dev_file_fetch(c, df.get(), targets.data(), targets.size()), "tg_dev_file_fetch");
    for (size_t i = 0; i < nblocks; ++i) {
        thrill::data::PinnedBlock pb(std::move(bytes[i]), 0, geom[i].bytes, geom[i].first_item,
                                     geom[i].num_items, /* typecode_verify */ false);
        out.AppendBlock(std::move(pb).MoveToBlock());
    }
}

//! true if every child of `node` is a GPU node (so no host File is needed)
template <typename Node>
bool AllChildrenAreGpuNodes(const Node& node) {
    std::vector<thrill::api::DIABase*> ch = node.children();
    if (ch.empty()) return false;
    for (thrill::api::DIABase* c : ch)
        if (dynamic_cast<GpuNodeBase*>(c) == nullptr) return false;
    return true;
}

/******************************************************************************/

template <typename ValueType>
class GpuSortNode final : public thrill::api::DOpNode<ValueType>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueType>;
    using Super::context_;

public:
    template <typename ParentDIA>
    GpuSortNode(const ParentDIA& parent, const tg_key_desc& desc)
        : Super(parent.ctx(), "GpuSort", { parent.id() }, { parent.node() }),
          desc_(desc), parent_stack_empty_(ParentDIA::stack_empty) {
        // hook the per-item PreOp exactly as SortNode does (api/sort.hpp:131-136)
        auto pre_op_fn = [this](const ValueType& input) { unsorted_writer_.Put(input); };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    void StartPreOp(size_t /* parent_index */) final { unsorted_writer_ = unsorted_file_.GetWriter(); }

    //! whole-File hand-off: the bulk path (api/sort.hpp:151-175)
    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        unsorted_file_ = file.Copy();
        return true;
    }

    //! a parent GPU node hands its result over in HBM
    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueType)) return false;
        device_input_ = file;
        return true;
    }

    void StopPreOp(size_t /* parent_index */) final { unsorted_writer_.Close(); }

    DIAMemUse ExecuteMemUse() final { return DIAMemUse::Max(); }

    //! MainOp (api/sort.hpp:537-663) + the local sort, all behind tg_sort_file / tg_sort_dev.  Collective.  The result stays
    //! in HBM; PushData hands it to GPU children as it is and writes a host File only if another kind of child needs one.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        size_t out_items = 0;
        if (device_input_) {
            Check(c, tg_sort_dev(c, &desc_, device_input_->get(), context_.rng_(), &out_items), "tg_sort_dev");
            device_input_.reset();
        }
        else {
            PinnedFileView view(unsorted_file_, context_.local_worker_id());
            Check(c, tg_sort_file(c, &desc_, view.data(), view.size(), context_.rng_(), &out_items), "tg_sort_file");
        }
        unsorted_file_.Clear();
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    DIAMemUse PushDataMemUse() final { return 0; }

    //! one sorted run per worker: always the files_.size() == 1 branch of SortNode::PushData (:224-227)
    void PushData(bool consume) final {
        if (device_result_ && AllChildrenAreGpuNodes(*this)) {
            bool all = true;
            for (const auto& ch : this->children_)
                all = dynamic_cast<GpuNodeBase*>(ch.node)->OnPreOpDeviceFile(device_result_, sizeof(ValueType), ch.parent_index) && all;
            if (all) return;
        }
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, sizeof(ValueType), sorted_file_);
            have_host_file_ = true;
        }
        this->PushFile(sorted_file_, consume);
    }

    void Dispose() final { sorted_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    tg_key_desc desc_;
    const bool parent_stack_empty_;
    thrill::data::File unsorted_file_ { context_.GetFile(this) };
    thrill::data::File::Writer unsorted_writer_;
    thrill::data::File sorted_file_ { context_.GetFile(this) };
    DeviceFilePtr device_input_, device_result_;
    bool have_host_file_ = false;
};

template <typename ValueType>
class GpuReduceNode final : public thrill::api::DOpNode<ValueType>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueType>;
    using Super::context_;

public:
    template <typename ParentDIA>
    GpuReduceNode(const ParentDIA& parent, const tg_kv_desc& desc)
        : GpuReduceNode(parent, desc, false, 0, ValueType()) { }

    //! to_index: ReduceToIndexNode (api/reduce_to_index.hpp:60-237) — dense result of result_size items, neutral_element
    //! where no item has that index; worker r holds the index range Range(0, size).Partition(r, p)
    template <typename ParentDIA>
    GpuReduceNode(const ParentDIA& parent, const tg_kv_desc& desc, bool to_index, size_t result_size,
                  const ValueType& neutral_element)
        : Super(parent.ctx(), to_index ? "GpuReduceToIndex" : "GpuReducePair", { parent.id() }, { parent.node() }),
          desc_(desc), parent_stack_empty_(ParentDIA::stack_empty),
          to_index_(to_index), result_size_(result_size), neutral_(neutral_element) {
        // ReduceNode inserts each item into the pre-phase table (api/reduce_by_key.hpp:126-133); the GPU pre
        // phase wants the whole shard, so items are collected in a File first
        auto pre_op_fn = [this](const ValueType& input) { input_writer_.Put(input); };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    DIAMemUse PreOpMemUse() final { return DIAMemUse::Max(); }

    void StartPreOp(size_t /* parent_index */) final { input_writer_ = input_file_.GetWriter(); }

    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        input_file_ = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueType)) return false;
        device_input_ = file;
        return true;
    }

    //! pre phase flush + exchange + post phase (api/reduce_by_key.hpp:157-211) behind tg_reduce_file / tg_reduce_dev.
    //! Collective.  The result stays in HBM until PushData knows who wants it.
    void StopPreOp(size_t /* parent_index */) final {
        input_writer_.Close();
        tg_ctx* c = WorkerCtx(context_);
        size_t out_items = 0;
        static_assert(sizeof(ValueType) == 16, "16-byte (key, value) items");
        uint64_t begin = 0;
        if (device_input_) {
            if (to_index_)
                Check(c, tg_reduce_to_index_dev(c, &desc_, device_input_->get(), result_size_, &neutral_, &out_items, &begin),
                      "tg_reduce_to_index_dev");
            else
                Check(c, tg_reduce_dev(c, &desc_, device_input_->get(), &out_items), "tg_reduce_dev");
            device_input_.reset();
        }
        else {
            PinnedFileView view(input_file_, context_.local_worker_id());
            if (to_index_)
                Check(c, tg_reduce_to_index_file(c, &desc_, view.data(), view.size(), result_size_, &neutral_, &out_items, &begin),
                      "tg_reduce_to_index_file");
            else
                Check(c, tg_reduce_file(c, &desc_, view.data(), view.size(), &out_items), "tg_reduce_file");
        }
        input_file_.Clear();
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    void Execute() final { }

    DIAMemUse PushDataMemUse() final { return 0; }

    void PushData(bool consume) final {
        if (device_result_ && AllChildrenAreGpuNodes(*this)) {
            bool all = true;
            for (const auto& ch : this->children_)
                all = dynamic_cast<GpuNodeBase*>(ch.node)->OnPreOpDeviceFile(device_result_, sizeof(ValueType), ch.parent_index) && all;
            if (all) return;
        }
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, sizeof(ValueType), reduced_file_);
            have_host_file_ = true;
        }
        this->PushFile(reduced_file_, consume);
    }

    void Dispose() final { reduced_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    tg_kv_desc desc_;
    const bool parent_stack_empty_;
    const bool to_index_ = false;
    const size_t result_size_ = 0;
    const ValueType neutral_ = ValueType();
    thrill::data::File input_file_ { context_.GetFile(this) };
    thrill::data::File::Writer input_writer_;
    thrill::data::File reduced_file_ { context_.GetFile(this) };
    DeviceFilePtr device_input_, device_result_;
    bool have_host_file_ = false;
};

//! DIA::Merge / api::Merge (api/merge.hpp:75-721) of kNumInputs DIAs sorted by the same comparator: the MergeNode protocol (one
//! File per parent, registered with AddChild(this, chain, index), :115-139; OnPreOpFile / StopPreOp per parent) with MainOp and
//! the multiway merge of PushData behind tg_merge_file.  Any input may arrive as a device File from a parent GPU node.
template <typename ValueType, size_t kNumInputs>
class GpuMergeNode final : public thrill::api::DOpNode<ValueType>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueType>;
    using Super::context_;

public:
    template <typename ParentDIA0, typename... ParentDIAs>
    GpuMergeNode(const tg_key_desc& desc, const ParentDIA0& parent0, const ParentDIAs& ... parents)
        : Super(parent0.ctx(), "GpuMerge", { parent0.id(), parents.id() ... }, { parent0.node(), parents.node() ... }),
          desc_(desc), parent_stack_empty_({ { ParentDIA0::stack_empty, (ParentDIAs::stack_empty)... } }) {
        for (size_t i = 0; i < kNumInputs; ++i) {
            files_[i] = context_.GetFilePtr(this);
            writers_[i] = files_[i]->GetWriter();
        }
        tlx::call_foreach_with_index(RegisterParent(this), parent0, parents ...);
    }

    //! per-item PreOp of parent Index into its File (api/merge.hpp:115-139)
    class RegisterParent
    {
    public:
        explicit RegisterParent(GpuMergeNode* node) : node_(node) { }
        template <typename Index, typename Parent>
        void operator () (const Index&, Parent& parent) {
            thrill::data::File::Writer* writer = &node_->writers_[Index::index];
            auto pre_op_fn = [writer](const ValueType& input) -> void { writer->Put(input); };
            auto lop_chain = parent.stack().push(pre_op_fn).fold();
            parent.node()->AddChild(node_, lop_chain, Index::index);
        }

    private:
        GpuMergeNode* node_;
    };

    bool OnPreOpFile(const thrill::data::File& file, size_t parent_index) final {
        if (!parent_stack_empty_[parent_index]) return false;
        *files_[parent_index] = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t parent_index) final {
        if (!parent_stack_empty_[parent_index] || item_bytes != sizeof(ValueType)) return false;
        device_inputs_[parent_index] = file;
        return true;
    }

    void StopPreOp(size_t parent_index) final { writers_[parent_index].Close(); }

    DIAMemUse ExecuteMemUse() final { return DIAMemUse::Max(); }

    //! MainOp (:465-700) and the merge of PushData (:160-190) behind tg_merge_file.  Collective.  The result stays in HBM.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        std::vector<std::unique_ptr<PinnedFileView> > views;
        std::array<tg_merge_input, kNumInputs> in;
        for (size_t i = 0; i < kNumInputs; ++i) {
            if (device_inputs_[i]) {
                in[i] = tg_merge_input { device_inputs_[i]->get(), nullptr, 0 };
                continue;
            }
            views.emplace_back(new PinnedFileView(*files_[i], context_.local_worker_id()));
            in[i] = tg_merge_input { nullptr, views.back()->data(), views.back()->size() };
        }
        size_t out_items = 0;
        Check(c, tg_merge_file(c, &desc_, in.data(), static_cast<uint32_t>(kNumInputs), &out_items), "tg_merge_file");
        views.clear();
        for (size_t i = 0; i < kNumInputs; ++i) {
            files_[i]->Clear();
            device_inputs_[i].reset();
        }
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    DIAMemUse PushDataMemUse() final { return 0; }

    void PushData(bool consume) final {
        if (device_result_ && AllChildrenAreGpuNodes(*this)) {
            bool all = true;
            for (const auto& ch : this->children_)
                all = dynamic_cast<GpuNodeBase*>(ch.node)->OnPreOpDeviceFile(device_result_, sizeof(ValueType), ch.parent_index) && all;
            if (all) return;
        }
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, sizeof(ValueType), merged_file_);
            have_host_file_ = true;
        }
        this->PushFile(merged_file_, consume);
    }

    void Dispose() final { merged_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    tg_key_desc desc_;
    const std::array<bool, kNumInputs> parent_stack_empty_;
    thrill::data::FilePtr files_[kNumInputs];
    thrill::data::File::Writer writers_[kNumInputs];
    std::array<DeviceFilePtr, kNumInputs> device_inputs_;
    thrill::data::File merged_file_ { context_.GetFile(this) };
    DeviceFilePtr device_result_;
    bool have_host_file_ = false;
};

//! api::InnerJoin (api/inner_join.hpp:700-827): the JoinNode protocol (one File per parent, registered with
//! AddChild(this, chain, index), :133-157; StopPreOp per parent) with the hash exchange, the local sorts and the join of
//! Execute / PushData (:159-312) behind tg_inner_join_file.  Either side may arrive as a device File from a parent GPU node.
//! kOutBytes: the serialized size of ValueType (24 for the (key, v1, v2) tuple, 16 for the (v1, v2) pair).
template <typename ValueType, typename LeftType, typename RightType, uint32_t kOutBytes>
class GpuJoinNode final : public thrill::api::DOpNode<ValueType>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueType>;
    using Super::context_;

public:
    template <typename LeftDIA, typename RightDIA>
    GpuJoinNode(const LeftDIA& left, const RightDIA& right, const tg_join_desc& desc)
        : Super(left.ctx(), "GpuInnerJoin", { left.id(), right.id() }, { left.node(), right.node() }),
          desc_(desc), parent_stack_empty_({ { LeftDIA::stack_empty, RightDIA::stack_empty } }) {
        for (size_t i = 0; i < 2; ++i) {
            files_[i] = context_.GetFilePtr(this);
            writers_[i] = files_[i]->GetWriter();
        }
        thrill::data::File::Writer* w0 = &writers_[0];
        thrill::data::File::Writer* w1 = &writers_[1];
        auto pre_op_fn0 = [w0](const LeftType& input) { w0->Put(input); };
        auto pre_op_fn1 = [w1](const RightType& input) { w1->Put(input); };
        left.node()->AddChild(this, left.stack().push(pre_op_fn0).fold(), 0);
        right.node()->AddChild(this, right.stack().push(pre_op_fn1).fold(), 1);
    }

    bool OnPreOpFile(const thrill::data::File& file, size_t parent_index) final {
        if (!parent_stack_empty_[parent_index]) return false;
        *files_[parent_index] = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t parent_index) final {
        if (!parent_stack_empty_[parent_index] || item_bytes != 16) return false;
        device_inputs_[parent_index] = file;
        return true;
    }

    void StopPreOp(size_t parent_index) final { writers_[parent_index].Close(); }

    DIAMemUse ExecuteMemUse() final { return DIAMemUse::Max(); }

    //! both exchanges, the local sorts and the join behind tg_inner_join_file.  Collective.  The result stays in HBM.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        std::vector<std::unique_ptr<PinnedFileView> > views;
        std::array<tg_merge_input, 2> in;
        for (size_t i = 0; i < 2; ++i) {
            if (device_inputs_[i]) {
                in[i] = tg_merge_input { device_inputs_[i]->get(), nullptr, 0 };
                continue;
            }
            views.emplace_back(new PinnedFileView(*files_[i], context_.local_worker_id()));
            in[i] = tg_merge_input { nullptr, views.back()->data(), views.back()->size() };
        }
        size_t out_items = 0;
        Check(c, tg_inner_join_file(c, &desc_, &in[0], &in[1], &out_items), "tg_inner_join_file");
        views.clear();
        for (size_t i = 0; i < 2; ++i) {
            files_[i]->Clear();
            device_inputs_[i].reset();
        }
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    DIAMemUse PushDataMemUse() final { return 0; }

    //! GPU children take the result in HBM (a 16-byte JoinValues result can feed thrill_gpu::ReducePair); a host File is
    //! written only if another kind of child needs one
    void PushData(bool consume) final {
        if (device_result_ && AllChildrenAreGpuNodes(*this)) {
            bool all = true;
            for (const auto& ch : this->children_)
                all = dynamic_cast<GpuNodeBase*>(ch.node)->OnPreOpDeviceFile(device_result_, kOutBytes, ch.parent_index) && all;
            if (all) return;
        }
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, kOutBytes, joined_file_);
            have_host_file_ = true;
        }
        this->PushFile(joined_file_, consume);
    }

    void Dispose() final { joined_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    tg_join_desc desc_;
    const std::array<bool, 2> parent_stack_empty_;
    thrill::data::FilePtr files_[2];
    thrill::data::File::Writer writers_[2];
    std::array<DeviceFilePtr, 2> device_inputs_;
    thrill::data::File joined_file_ { context_.GetFile(this) };
    DeviceFilePtr device_result_;
    bool have_host_file_ = false;
};

//! The iterator a GpuGroupNode hands to the group function: the public members of api::GroupByIterator
//! (api/group_by_iterator.hpp:47-127), HasNext() and Next(), over the items of one group of the sorted host File.  The node
//! drives it with the same two calls the stock nodes use (HasNextForReal, GetNextKey), so a function that stops before the end
//! of its group is called again with the rest of it, as in the reference.
template <typename ValueIn>
class GroupIterator
{
public:
    using Key = typename ValueIn::first_type;

    explicit GroupIterator(thrill::data::File::Reader& reader)
        : reader_(reader), elem_(reader_.template Next<ValueIn>()), key_(elem_.first) { }

    GroupIterator(const GroupIterator&) = delete;
    GroupIterator& operator = (const GroupIterator&) = delete;

    bool HasNext() { return !is_reader_empty_ && equal_key_; }

    ValueIn Next() {
        assert(!is_reader_empty_);
        ValueIn elem = elem_;
        if (reader_.HasNext()) {
            elem_ = reader_.template Next<ValueIn>();
            if (elem_.first != key_) {
                key_ = elem_.first;
                equal_key_ = false;
            }
        }
        else {
            is_reader_empty_ = true;
        }
        return elem;
    }

    //! (the node's loop) items are left
    bool HasNextForReal() const { return !is_reader_empty_; }
    //! (the node's loop) the key of the next group; opens it for HasNext()
    const Key& GetNextKey() {
        equal_key_ = true;
        return key_;
    }

private:
    thrill::data::File::Reader& reader_;
    bool is_reader_empty_ = false;
    bool equal_key_ = true;
    ValueIn elem_;
    Key key_;
};

//! DIA::GroupByKey (api/group_by_key.hpp:46-428) and DIA::GroupToIndex (api/group_to_index.hpp:36-290) of a DIA of
//! pair<uint64_t, 8-byte value> grouped by .first.  The exchange to the key's owner and the sort by the key run behind
//! tg_group_by_key_file / tg_group_to_index_file (Execute, collective); PushData fetches the grouped items into a host File once
//! and runs the stock nodes' RunUserFunc loop (group_by_key.hpp:314-331, group_to_index.hpp:186-215) over a GroupIterator.
//! The group function and ValueOut are arbitrary, so the children get host items of ValueOut, never a device File.
template <typename ValueOut, typename ValueIn, typename GroupFunction>
class GpuGroupNode final : public thrill::api::DOpNode<ValueOut>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueOut>;
    using Super::context_;

public:
    //! to_index: GroupToIndex with result_size and neutral_element; otherwise GroupByKey
    template <typename ParentDIA>
    GpuGroupNode(const ParentDIA& parent, const GroupFunction& group_function, bool to_index, size_t result_size,
                 const ValueOut& neutral_element)
        : Super(parent.ctx(), to_index ? "GpuGroupToIndex" : "GpuGroupByKey", { parent.id() }, { parent.node() }),
          group_function_(group_function), parent_stack_empty_(ParentDIA::stack_empty),
          to_index_(to_index), result_size_(result_size), neutral_(neutral_element) {
        auto pre_op_fn = [this](const ValueIn& input) { input_writer_.Put(input); };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    DIAMemUse PreOpMemUse() final { return DIAMemUse::Max(); }

    void StartPreOp(size_t /* parent_index */) final { input_writer_ = input_file_.GetWriter(); }

    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        input_file_ = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueIn)) return false;
        device_input_ = file;
        return true;
    }

    void StopPreOp(size_t /* parent_index */) final { input_writer_.Close(); }

    DIAMemUse ExecuteMemUse() final { return DIAMemUse::Max(); }

    //! MainOp (group_by_key.hpp:348-376, group_to_index.hpp:234-254) behind tg_group_*_file.  Collective.  The grouped items
    //! stay in HBM until PushData.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        std::unique_ptr<PinnedFileView> view;
        tg_merge_input in;
        if (device_input_) {
            in = tg_merge_input { device_input_->get(), nullptr, 0 };
        }
        else {
            view.reset(new PinnedFileView(input_file_, context_.local_worker_id()));
            in = tg_merge_input { nullptr, view->data(), view->size() };
        }
        size_t out_items = 0;
        if (to_index_)
            Check(c, tg_group_to_index_file(c, &in, result_size_, &out_items, &range_begin_, &range_end_), "tg_group_to_index_file");
        else
            Check(c, tg_group_by_key_file(c, &in, &out_items), "tg_group_by_key_file");
        view.reset();
        input_file_.Clear();
        device_input_.reset();
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    DIAMemUse PushDataMemUse() final { return 0; }

    //! RunUserFunc of the stock nodes over the grouped items.  They are fetched once and read without consuming them, so the
    //! result can be pushed again until Dispose.  The key argument is the iterator's key, as in the stock nodes.
    void PushData(bool /* consume */) final {
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, sizeof(ValueIn), grouped_file_);
            have_host_file_ = true;
        }
        auto r = grouped_file_.GetReader(/* consume */ false);
        if (!to_index_) {
            if (!r.HasNext()) return;
            GroupIterator<ValueIn> it(r);
            while (it.HasNextForReal())
                this->PushItem(group_function_(it, it.GetNextKey()));
            return;
        }
        size_t curr_index = range_begin_;
        if (r.HasNext()) {
            GroupIterator<ValueIn> it(r);
            while (it.HasNextForReal()) {
                if (it.GetNextKey() != curr_index) this->PushItem(neutral_);
                else this->PushItem(group_function_(it, it.GetNextKey()));
                ++curr_index;
            }
        }
        while (curr_index < range_end_) {
            this->PushItem(neutral_);
            ++curr_index;
        }
    }

    void Dispose() final { grouped_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    GroupFunction group_function_;
    const bool parent_stack_empty_;
    const bool to_index_;
    const size_t result_size_;
    const ValueOut neutral_;
    uint64_t range_begin_ = 0, range_end_ = 0;
    thrill::data::File input_file_ { context_.GetFile(this) };
    thrill::data::File::Writer input_writer_;
    thrill::data::File grouped_file_ { context_.GetFile(this) };
    DeviceFilePtr device_input_, device_result_;
    bool have_host_file_ = false;
};

//! DIA::PrefixSum / DIA::ExPrefixSum (PrefixSumNode, api/prefix_sum.hpp:28-128) and DIA::ZipWithIndex (ZipWithIndexNode,
//! api/zip_with_index.hpp:40-128): the stock node protocol (a File of the parent's items, or the parent's File whole through
//! OnPreOpFile) with the collective call in Execute: tg_prefix_sum_file (the all-gather of the local totals, the carry and the
//! scan) or tg_zip_with_index_file.  The input may arrive as a device File from a parent GPU node, and the result, one item per
//! input item on the same worker, is handed to GPU children in HBM.  zip: ZipWithIndex with index_first; otherwise PrefixSum
//! with desc, initial and inclusive.
template <typename ValueOut, typename ValueIn>
class GpuScanNode final : public thrill::api::DOpNode<ValueOut>, public GpuNodeBase
{
    using Super = thrill::api::DOpNode<ValueOut>;
    using Super::context_;

public:
    template <typename ParentDIA>
    GpuScanNode(const ParentDIA& parent, const char* label, bool zip, const tg_scan_desc& desc, const ValueIn& initial,
                bool inclusive, bool index_first)
        : Super(parent.ctx(), label, { parent.id() }, { parent.node() }),
          zip_(zip), desc_(desc), initial_(initial), inclusive_(inclusive), index_first_(index_first),
          parent_stack_empty_(ParentDIA::stack_empty) {
        auto pre_op_fn = [this](const ValueIn& input) { input_writer_.Put(input); };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    void StartPreOp(size_t /* parent_index */) final { input_writer_ = input_file_.GetWriter(); }

    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        input_file_ = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueIn)) return false;
        device_input_ = file;
        return true;
    }

    void StopPreOp(size_t /* parent_index */) final { input_writer_.Close(); }

    DIAMemUse ExecuteMemUse() final { return DIAMemUse::Max(); }

    //! Execute (prefix_sum.hpp:84-90, zip_with_index.hpp:86-94) and the outputs of PushData behind one call.  Collective.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        std::unique_ptr<PinnedFileView> view;
        tg_merge_input in;
        if (device_input_) {
            in = tg_merge_input { device_input_->get(), nullptr, 0 };
        }
        else {
            view.reset(new PinnedFileView(input_file_, context_.local_worker_id()));
            in = tg_merge_input { nullptr, view->data(), view->size() };
        }
        size_t out_items = 0;
        if (zip_)
            Check(c, tg_zip_with_index_file(c, &in, index_first_ ? 1 : 0, &out_items), "tg_zip_with_index_file");
        else
            Check(c, tg_prefix_sum_file(c, &desc_, &in, &initial_, inclusive_ ? 1 : 0, &out_items), "tg_prefix_sum_file");
        view.reset();
        input_file_.Clear();
        device_input_.reset();
        tg_dev_file f;
        Check(c, tg_output_detach(c, &f), "tg_output_detach");
        device_result_ = std::make_shared<DeviceFile>(c, f);
        have_host_file_ = false;
    }

    DIAMemUse PushDataMemUse() final { return 0; }

    void PushData(bool consume) final {
        if (device_result_ && AllChildrenAreGpuNodes(*this)) {
            bool all = true;
            for (const auto& ch : this->children_)
                all = dynamic_cast<GpuNodeBase*>(ch.node)->OnPreOpDeviceFile(device_result_, sizeof(ValueOut), ch.parent_index) && all;
            if (all) return;
        }
        if (!have_host_file_) {
            FetchDeviceFileIntoFile(WorkerCtx(context_), context_, *device_result_, sizeof(ValueOut), result_file_);
            have_host_file_ = true;
        }
        this->PushFile(result_file_, consume);
    }

    void Dispose() final { result_file_.Clear(); device_result_.reset(); have_host_file_ = false; }

private:
    const bool zip_;
    const tg_scan_desc desc_;
    const ValueIn initial_;
    const bool inclusive_, index_first_;
    const bool parent_stack_empty_;
    thrill::data::File input_file_ { context_.GetFile(this) };
    thrill::data::File::Writer input_writer_;
    thrill::data::File result_file_ { context_.GetFile(this) };
    DeviceFilePtr device_input_, device_result_;
    bool have_host_file_ = false;
};
template <typename ValueType>
using GpuPrefixSumNode = GpuScanNode<ValueType, ValueType>;
template <typename ValueOut, typename ValueIn>
using GpuZipWithIndexNode = GpuScanNode<ValueOut, ValueIn>;

//! DIA::Sum / Min / Max / AllReduce (AllReduceNode, api/all_reduce.hpp:27-85): the stock node protocol (a File of the parent's
//! items, or the parent's File whole through OnPreOpFile) with the collective call in Execute: tg_all_reduce_file (the tile
//! reduce, one all-gather of the workers' records, the fold on the device).  A parent GPU node hands its result over in HBM, so
//! a GPU chain that ends in an action fetches nothing but the value.  The result is the stock node's bit for bit, except for the
//! bracketing of double sums (include/thrill_gpu.h states the bound).
template <typename ValueType>
class GpuAllReduceNode final : public thrill::api::ActionResultNode<ValueType>, public GpuNodeBase
{
    using Super = thrill::api::ActionResultNode<ValueType>;
    using Super::context_;

public:
    template <typename ParentDIA>
    GpuAllReduceNode(const ParentDIA& parent, const char* label, const tg_scan_desc& desc, const ValueType& initial,
                     bool with_initial)
        : Super(parent.ctx(), label, { parent.id() }, { parent.node() }),
          desc_(desc), initial_(initial), with_initial_(with_initial), parent_stack_empty_(ParentDIA::stack_empty) {
        auto pre_op_fn = [this](const ValueType& input) { input_writer_.Put(input); };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    void StartPreOp(size_t /* parent_index */) final { input_writer_ = input_file_.GetWriter(); }

    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        input_file_ = file.Copy();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueType)) return false;
        device_input_ = file;
        return true;
    }

    void StopPreOp(size_t /* parent_index */) final { input_writer_.Close(); }

    //! Execute (all_reduce.hpp:67-70) behind one call.  Collective.
    void Execute() final {
        tg_ctx* c = WorkerCtx(context_);
        std::unique_ptr<PinnedFileView> view;
        tg_merge_input in;
        if (device_input_) {
            in = tg_merge_input { device_input_->get(), nullptr, 0 };
        }
        else {
            view.reset(new PinnedFileView(input_file_, context_.local_worker_id()));
            in = tg_merge_input { nullptr, view->data(), view->size() };
        }
        Check(c, tg_all_reduce_file(c, &desc_, &in, with_initial_ ? &initial_ : nullptr, &result_), "tg_all_reduce_file");
        view.reset();
        input_file_.Clear();
        device_input_.reset();
    }

    const ValueType& result() const final { return result_; }

private:
    const tg_scan_desc desc_;
    const ValueType initial_;
    const bool with_initial_;
    const bool parent_stack_empty_;
    thrill::data::File input_file_ { context_.GetFile(this) };
    thrill::data::File::Writer input_writer_;
    DeviceFilePtr device_input_;
    ValueType result_ = ValueType();
};

//! DIA::Size / SizeFuture (SizeNode, api/size.hpp): the local count from a device File's items(), a host File's num_items() or
//! the per-item PreOp, then the stock all-reduce of the counts.  No kernel, and no item crosses PCIe.
template <typename ValueType>
class GpuSizeNode final : public thrill::api::ActionResultNode<size_t>, public GpuNodeBase
{
    using Super = thrill::api::ActionResultNode<size_t>;
    using Super::context_;

public:
    template <typename ParentDIA>
    explicit GpuSizeNode(const ParentDIA& parent)
        : Super(parent.ctx(), "GpuSize", { parent.id() }, { parent.node() }),
          parent_stack_empty_(ParentDIA::stack_empty) {
        auto pre_op_fn = [this](const ValueType&) { ++local_size_; };
        auto lop_chain = parent.stack().push(pre_op_fn).fold();
        parent.node()->AddChild(this, lop_chain);
    }

    bool OnPreOpFile(const thrill::data::File& file, size_t /* parent_index */) final {
        if (!parent_stack_empty_) return false;
        local_size_ = file.num_items();
        return true;
    }

    bool OnPreOpDeviceFile(const DeviceFilePtr& file, size_t item_bytes, size_t /* parent_index */) final {
        if (!parent_stack_empty_ || item_bytes != sizeof(ValueType)) return false;
        local_size_ = file->items();
        return true;
    }

    void Execute() final { global_size_ = context_.net.AllReduce(local_size_); }

    const size_t& result() const final { return global_size_; }

private:
    const bool parent_stack_empty_;
    size_t local_size_ = 0;
    size_t global_size_ = 0;
};

/******************************************************************************/
// front doors (same argument meaning as DIA<T>::Sort / DIA<T>::ReducePair)

template <typename ValueType, typename Stack, typename CompareFunction = std::less<ValueType> >
auto Sort(const DIA<ValueType, Stack>& dia, const CompareFunction& /* compare_function */ = CompareFunction()) {
    static_assert(SortDesc<ValueType, CompareFunction>::supported,
                  "thrill_gpu::Sort: this (ValueType, CompareFunction) pair has no GPU descriptor; "
                  "use the stock dia.Sort(cmp)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuSortNode<ValueType> >(
        dia, SortDesc<ValueType, CompareFunction>::make());
    return DIA<ValueType>(node);
}

//! DIA<T>::SortStable(cmp) (api/sort.hpp:873-937): equal keys keep their global input order.  The GPU sort is stable by
//! construction (stable partition passes, exchange in worker order), so this is the same node with the flag set.
template <typename ValueType, typename Stack, typename CompareFunction = std::less<ValueType> >
auto SortStable(const DIA<ValueType, Stack>& dia, const CompareFunction& /* compare_function */ = CompareFunction()) {
    static_assert(SortDesc<ValueType, CompareFunction>::supported,
                  "thrill_gpu::SortStable: this (ValueType, CompareFunction) pair has no GPU descriptor; "
                  "use the stock dia.SortStable(cmp)");
    assert(dia.IsValid());
    tg_key_desc d = SortDesc<ValueType, CompareFunction>::make();
    d.stable = 1;
    auto node = tlx::make_counting<GpuSortNode<ValueType> >(dia, d);
    return DIA<ValueType>(node);
}

template <typename Key, typename Value, typename Stack, typename ReduceFunction>
auto ReducePair(const DIA<std::pair<Key, Value>, Stack>& dia, const ReduceFunction& /* reduce_function */) {
    static_assert(std::is_same<Key, uint64_t>::value && sizeof(Value) == 8 &&
                  ReduceDesc<Value, ReduceFunction>::supported,
                  "thrill_gpu::ReducePair: this (Key, Value, ReduceFunction) has no GPU descriptor; "
                  "use the stock dia.ReducePair(fn)");
    assert(dia.IsValid());
    using ValueType = std::pair<Key, Value>;
    auto node = tlx::make_counting<GpuReduceNode<ValueType> >(
        dia, tg_kv_desc { 16, ReduceDesc<Value, ReduceFunction>::op });
    return DIA<ValueType>(node);
}

//! DIA<T>::ReduceByKey(key_extractor, reduce_function) (api/reduce_by_key.hpp:312-363) for the recognised functor pair:
//! key_extractor = thrill_gpu::KeyFirst, reduce_function = thrill_gpu::OnSecond<F> with F one of the ReducePair functions
//! (std::plus<double>, std::plus<uint64_t>, thrill_gpu::MinU64, thrill_gpu::MaxU64).  ReducePair is exactly this pair of
//! functors in the reference too (:444-449).
template <typename Key, typename Value, typename Stack, typename ValueFunction>
auto ReduceByKey(const DIA<std::pair<Key, Value>, Stack>& dia, const KeyFirst& /* key_extractor */,
                 const OnSecond<ValueFunction>& reduce_function) {
    return ReducePair(dia, reduce_function.fn);
}

//! DIA<pair<uint64_t index, V>>::ReduceToIndex(key = .first, reduce function on .second, size, neutral_element)
//! (api/reduce_to_index.hpp:239-393 front doors; examples/page_rank/page_rank.hpp:125-135)
template <typename Key, typename Value, typename Stack, typename ReduceFunction>
auto ReduceToIndex(const DIA<std::pair<Key, Value>, Stack>& dia, const ReduceFunction& /* reduce_function */,
                   size_t size, const std::pair<Key, Value>& neutral_element = std::pair<Key, Value>()) {
    static_assert(std::is_same<Key, uint64_t>::value && sizeof(Value) == 8 &&
                  ReduceDesc<Value, ReduceFunction>::supported,
                  "thrill_gpu::ReduceToIndex: this (Key, Value, ReduceFunction) has no GPU descriptor; "
                  "use the stock dia.ReduceToIndex(key_extractor, fn, size)");
    assert(dia.IsValid());
    using ValueType = std::pair<Key, Value>;
    auto node = tlx::make_counting<GpuReduceNode<ValueType> >(
        dia, tg_kv_desc { 16, ReduceDesc<Value, ReduceFunction>::op }, true, size, neutral_element);
    return DIA<ValueType>(node);
}

template <bool...> struct BoolPack { };
template <bool... B> using AllOf = std::is_same<BoolPack<true, B...>, BoolPack<B..., true> >;

//! api::Merge(comparator, dia0, dia1, ...) (api/merge.hpp:673-713) of 2..16 DIAs for the (type, comparator) pairs thrill_gpu::Sort
//! recognises with 8- or 16-byte items.  Equal items come out in (input, position) order, one of the orders the stock
//! operator allows.  DIA::Merge(second, cmp) (:715-721) is Merge(cmp, dia, second).
template <typename Comparator, typename FirstDIA, typename... DIAs>
auto Merge(const Comparator& /* comparator */, const FirstDIA& first_dia, const DIAs& ... dias) {
    using ValueType = typename FirstDIA::ValueType;
    static_assert(SortDesc<ValueType, Comparator>::supported && (sizeof(ValueType) == 8 || sizeof(ValueType) == 16),
                  "thrill_gpu::Merge: this (ValueType, Comparator) pair has no GPU descriptor for Merge (8- or 16-byte items); "
                  "use the stock api::Merge(cmp, dias...)");
    static_assert(sizeof ... (DIAs) >= 1 && sizeof ... (DIAs) <= 15, "thrill_gpu::Merge: 2..16 DIAs");
    static_assert(AllOf<std::is_same<typename DIAs::ValueType, ValueType>::value ...>::value,
                  "thrill_gpu::Merge: every DIA must have the same item type");
    first_dia.AssertValid();
    tlx::vexpand((dias.AssertValid(), 0) ...);
    auto node = tlx::make_counting<GpuMergeNode<ValueType, 1 + sizeof ... (DIAs)> >(
        SortDesc<ValueType, Comparator>::make(), first_dia, dias ...);
    return DIA<ValueType>(node);
}

//! api::InnerJoin(left, right, key_extractor1, key_extractor2, join_function) (api/inner_join.hpp:700-827) for pair DIAs joined on
//! .first: left = DIA<pair<uint64_t, V1>>, right = DIA<pair<uint64_t, V2>> with 8-byte V1 and V2, key extractors KeyFirst,
//! join_function JoinKeyValues (-> tuple<uint64_t, V1, V2>) or JoinValues (-> pair<V1, V2>).  Worker Hash128to64(0, key) % p
//! holds a key's results, ordered by (key, left global position, right global position), one of the orders the stock operator
//! allows.  InnerJoin(a, a, ...) is a self-join with one parent on both edges.
template <typename LeftDIA, typename RightDIA, typename JoinFunction>
auto InnerJoin(const LeftDIA& left, const RightDIA& right, const KeyFirst& /* key_extractor1 */,
               const KeyFirst& /* key_extractor2 */, const JoinFunction& join_function) {
    using LeftType = typename LeftDIA::ValueType;
    using RightType = typename RightDIA::ValueType;
    static_assert(JoinDesc<JoinFunction>::supported,
                  "thrill_gpu::InnerJoin: the join function has no GPU descriptor (JoinKeyValues or JoinValues); "
                  "use the stock api::InnerJoin(left, right, key1, key2, join_fn)");
    static_assert(std::is_same<typename LeftType::first_type, uint64_t>::value &&
                  std::is_same<typename RightType::first_type, uint64_t>::value &&
                  sizeof(typename LeftType::second_type) == 8 && sizeof(typename RightType::second_type) == 8 &&
                  std::is_trivially_copyable<typename LeftType::second_type>::value &&
                  std::is_trivially_copyable<typename RightType::second_type>::value,
                  "thrill_gpu::InnerJoin: both DIAs must hold pair<uint64_t, 8-byte value>; "
                  "use the stock api::InnerJoin(left, right, key1, key2, join_fn)");
    using ValueType = decltype(join_function(std::declval<LeftType>(), std::declval<RightType>()));
    left.AssertValid();
    right.AssertValid();
    auto node = tlx::make_counting<GpuJoinNode<ValueType, LeftType, RightType, JoinDesc<JoinFunction>::out_bytes> >(
        left, right, tg_join_desc { 16, JoinDesc<JoinFunction>::fn });
    return DIA<ValueType>(node);
}

//! the item types thrill_gpu::GroupByKey / GroupToIndex take: pair<uint64_t, 8-byte trivially copyable value>
template <typename ValueIn>
struct IsGroupPair : std::false_type { };
template <typename V>
struct IsGroupPair<std::pair<uint64_t, V> >
    : std::integral_constant<bool, sizeof(V) == 8 && std::is_trivially_copyable<V>::value> { };

//! DIA<T>::GroupByKey<ValueOut>(key_extractor, groupby_function) (api/group_by_key.hpp:419-428) for a DIA of pair<uint64_t,
//! 8-byte value> grouped by .first (key_extractor KeyFirst).  group_function(iterator, key) is any function: it is called on the
//! host once per group, with an iterator that has HasNext() and Next(), and returns a ValueOut.  Worker key % p holds a key's
//! group (the stock placement with the default std::hash); groups come in ascending key order, the items of a group in global
//! input order (one of the orders the stock operator allows).  Location detection and other hash functions are not offered.
template <typename ValueOut, typename ValueIn, typename Stack, typename GroupFunction>
auto GroupByKey(const DIA<ValueIn, Stack>& dia, const KeyFirst& /* key_extractor */, const GroupFunction& group_function) {
    static_assert(IsGroupPair<ValueIn>::value,
                  "thrill_gpu::GroupByKey: the DIA must hold pair<uint64_t, 8-byte value> grouped by KeyFirst; "
                  "use the stock dia.GroupByKey<ValueOut>(key_extractor, group_function)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuGroupNode<ValueOut, ValueIn, GroupFunction> >(
        dia, group_function, false, 0, ValueOut());
    return DIA<ValueOut>(node);
}

//! DIA<T>::GroupToIndex<ValueOut>(key_extractor, groupby_function, size, neutral_element) (api/group_to_index.hpp:257-290) for a
//! DIA of pair<uint64_t index, 8-byte value> grouped by .first: worker r pushes one ValueOut per index of
//! Range(0, size).Partition(r, p), group_function(iterator, index) where the index has items and neutral_element where it has
//! none.  An index >= size is an error (die) on every worker.
template <typename ValueOut, typename ValueIn, typename Stack, typename GroupFunction>
auto GroupToIndex(const DIA<ValueIn, Stack>& dia, const KeyFirst& /* key_extractor */, const GroupFunction& group_function,
                  size_t size, const ValueOut& neutral_element = ValueOut()) {
    static_assert(IsGroupPair<ValueIn>::value,
                  "thrill_gpu::GroupToIndex: the DIA must hold pair<uint64_t, 8-byte value> grouped by KeyFirst; "
                  "use the stock dia.GroupToIndex<ValueOut>(key_extractor, group_function, size)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuGroupNode<ValueOut, ValueIn, GroupFunction> >(
        dia, group_function, true, size, neutral_element);
    return DIA<ValueOut>(node);
}

//! DIA<T>::PrefixSum(sum_function, initial_element) (api/dia.hpp:1850, api/prefix_sum.hpp:132-160) for the recognised pairs:
//! uint64_t with std::plus<uint64_t>, MinU64 or MaxU64; double with std::plus<double>; pair<uint64_t, V> with ScanSecond<F>.
//! out_i = carry + x_0 + ... + x_i, carry = initial_element + the local totals of the workers below (each folded from T()),
//! as in the stock node.  Items stay on their worker.  Double sums are bracketed by tiles: bitwise reproducible, and within
//! the rounding bound of tg_prefix_sum (include/thrill_gpu.h) of the exact sums while no partial sum can overflow.
template <typename ValueType, typename Stack, typename SumFunction>
auto PrefixSum(const DIA<ValueType, Stack>& dia, const SumFunction& /* sum_function */,
               const typename DIA<ValueType, Stack>::ValueType& initial_element = ValueType()) {
    static_assert(ScanDesc<ValueType, SumFunction>::supported,
                  "thrill_gpu::PrefixSum: this (ValueType, SumFunction) pair has no GPU descriptor; "
                  "use the stock dia.PrefixSum(sum_function, initial_element)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuPrefixSumNode<ValueType> >(
        dia, "GpuPrefixSum", false,
        tg_scan_desc { ScanDesc<ValueType, SumFunction>::item_bytes, ScanDesc<ValueType, SumFunction>::op },
        initial_element, true, false);
    return DIA<ValueType>(node);
}

//! DIA<T>::ExPrefixSum(sum_function, initial_element) (api/dia.hpp:1867, api/ex_prefix_sum.hpp): out_0 = carry,
//! out_i = carry + x_0 + ... + x_{i-1}; otherwise as PrefixSum
template <typename ValueType, typename Stack, typename SumFunction>
auto ExPrefixSum(const DIA<ValueType, Stack>& dia, const SumFunction& /* sum_function */,
                 const typename DIA<ValueType, Stack>::ValueType& initial_element = ValueType()) {
    static_assert(ScanDesc<ValueType, SumFunction>::supported,
                  "thrill_gpu::ExPrefixSum: this (ValueType, SumFunction) pair has no GPU descriptor; "
                  "use the stock dia.ExPrefixSum(sum_function, initial_element)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuPrefixSumNode<ValueType> >(
        dia, "GpuExPrefixSum", false,
        tg_scan_desc { ScanDesc<ValueType, SumFunction>::item_bytes, ScanDesc<ValueType, SumFunction>::op },
        initial_element, false, false);
    return DIA<ValueType>(node);
}

//! DIA<T>::ZipWithIndex(zip_function) (api/zip_with_index.hpp:140-152) of 8-byte trivially copyable items with
//! zip_function IndexFirst (-> pair<uint64_t, T>(index, item), the input of ReduceToIndex / GroupToIndex) or IndexSecond
//! (-> pair<T, uint64_t>(item, index), the (char, index) tuples of the suffix sorters).  Items stay on their worker.
template <typename ValueType, typename Stack, typename ZipFunction>
auto ZipWithIndex(const DIA<ValueType, Stack>& dia, const ZipFunction& zip_function) {
    static_assert((std::is_same<ZipFunction, IndexFirst>::value || std::is_same<ZipFunction, IndexSecond>::value) &&
                  sizeof(ValueType) == 8 && std::is_trivially_copyable<ValueType>::value,
                  "thrill_gpu::ZipWithIndex: 8-byte items with IndexFirst or IndexSecond only; "
                  "use the stock dia.ZipWithIndex(zip_function)");
    assert(dia.IsValid());
    using ValueOut = decltype(zip_function(std::declval<ValueType>(), size_t(0)));
    auto node = tlx::make_counting<GpuZipWithIndexNode<ValueOut, ValueType> >(
        dia, "GpuZipWithIndex", true, tg_scan_desc { 8, 0 }, ValueType(), true,
        std::is_same<ZipFunction, IndexFirst>::value);
    return DIA<ValueOut>(node);
}

//! DIA<T>::AllReduceFuture(fn[, initial]) (api/all_reduce.hpp:157-221) for the recognised pairs: uint64_t with std::plus<uint64_t>,
//! MinU64 / common::minimum<uint64_t> or MaxU64 / common::maximum<uint64_t>; double with std::plus<double>,
//! common::minimum<double> or common::maximum<double>; pair<uint64_t, V> with ScanSecond<F>, F any of these.  Each worker folds
//! its items from its first one (worker 0 from initial), an empty worker contributes T() (the initial value if there is one),
//! and the workers' values are folded in rank order: the stock result, bit for bit, but for the bracketing of double sums
//! (bitwise reproducible, within the bound of tg_all_reduce in include/thrill_gpu.h).
template <typename ValueType, typename Stack, typename Function>
thrill::api::Future<ValueType> AllReduceFuture(const DIA<ValueType, Stack>& dia, const Function& /* function */) {
    static_assert(ActionDesc<ValueType, Function>::supported,
                  "thrill_gpu::AllReduce: this (ValueType, Function) pair has no GPU descriptor; use the stock dia.AllReduce(fn)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuAllReduceNode<ValueType> >(
        dia, "GpuAllReduce", tg_scan_desc { ActionDesc<ValueType, Function>::item_bytes, ActionDesc<ValueType, Function>::op },
        ValueType(), false);
    return thrill::api::Future<ValueType>(node);
}
template <typename ValueType, typename Stack, typename Function>
thrill::api::Future<ValueType> AllReduceFuture(const DIA<ValueType, Stack>& dia, const Function& /* function */,
                                               const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    static_assert(ActionDesc<ValueType, Function>::supported,
                  "thrill_gpu::AllReduce: this (ValueType, Function) pair has no GPU descriptor; use the stock dia.AllReduce(fn)");
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuAllReduceNode<ValueType> >(
        dia, "GpuAllReduce", tg_scan_desc { ActionDesc<ValueType, Function>::item_bytes, ActionDesc<ValueType, Function>::op },
        initial_value, true);
    return thrill::api::Future<ValueType>(node);
}
//! DIA<T>::AllReduce(fn[, initial]) (api/all_reduce.hpp:87-155)
template <typename ValueType, typename Stack, typename Function>
ValueType AllReduce(const DIA<ValueType, Stack>& dia, const Function& function) {
    return AllReduceFuture(dia, function).get();
}
template <typename ValueType, typename Stack, typename Function>
ValueType AllReduce(const DIA<ValueType, Stack>& dia, const Function& function,
                    const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return AllReduceFuture(dia, function, initial_value).get();
}
//! DIA<T>::Sum / SumFuture([fn[, initial]]) (api/sum.hpp): AllReduce with std::plus<T> by default
template <typename ValueType, typename Stack, typename SumFunction = std::plus<ValueType> >
thrill::api::Future<ValueType> SumFuture(const DIA<ValueType, Stack>& dia, const SumFunction& sum_function = SumFunction()) {
    return AllReduceFuture(dia, sum_function);
}
template <typename ValueType, typename Stack, typename SumFunction>
thrill::api::Future<ValueType> SumFuture(const DIA<ValueType, Stack>& dia, const SumFunction& sum_function,
                                         const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return AllReduceFuture(dia, sum_function, initial_value);
}
template <typename ValueType, typename Stack, typename SumFunction = std::plus<ValueType> >
ValueType Sum(const DIA<ValueType, Stack>& dia, const SumFunction& sum_function = SumFunction()) {
    return SumFuture(dia, sum_function).get();
}
template <typename ValueType, typename Stack, typename SumFunction>
ValueType Sum(const DIA<ValueType, Stack>& dia, const SumFunction& sum_function,
              const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return SumFuture(dia, sum_function, initial_value).get();
}
//! DIA<T>::Min / MinFuture([initial]) (api/min.hpp): AllReduce with common::minimum<T> (std::min: b < a ? b : a)
template <typename ValueType, typename Stack>
thrill::api::Future<ValueType> MinFuture(const DIA<ValueType, Stack>& dia) {
    return AllReduceFuture(dia, thrill::common::minimum<ValueType>());
}
template <typename ValueType, typename Stack>
thrill::api::Future<ValueType> MinFuture(const DIA<ValueType, Stack>& dia,
                                         const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return AllReduceFuture(dia, thrill::common::minimum<ValueType>(), initial_value);
}
template <typename ValueType, typename Stack>
ValueType Min(const DIA<ValueType, Stack>& dia) { return MinFuture(dia).get(); }
template <typename ValueType, typename Stack>
ValueType Min(const DIA<ValueType, Stack>& dia, const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return MinFuture(dia, initial_value).get();
}
//! DIA<T>::Max / MaxFuture([initial]) (api/max.hpp): AllReduce with common::maximum<T> (std::max: a < b ? b : a)
template <typename ValueType, typename Stack>
thrill::api::Future<ValueType> MaxFuture(const DIA<ValueType, Stack>& dia) {
    return AllReduceFuture(dia, thrill::common::maximum<ValueType>());
}
template <typename ValueType, typename Stack>
thrill::api::Future<ValueType> MaxFuture(const DIA<ValueType, Stack>& dia,
                                         const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return AllReduceFuture(dia, thrill::common::maximum<ValueType>(), initial_value);
}
template <typename ValueType, typename Stack>
ValueType Max(const DIA<ValueType, Stack>& dia) { return MaxFuture(dia).get(); }
template <typename ValueType, typename Stack>
ValueType Max(const DIA<ValueType, Stack>& dia, const typename DIA<ValueType, Stack>::ValueType& initial_value) {
    return MaxFuture(dia, initial_value).get();
}

//! DIA<T>::SizeFuture / Size (api/size.hpp:86-103): the number of items of the DIA, on every worker.  Any item type.
template <typename ValueType, typename Stack>
thrill::api::Future<size_t> SizeFuture(const DIA<ValueType, Stack>& dia) {
    assert(dia.IsValid());
    auto node = tlx::make_counting<GpuSizeNode<ValueType> >(dia);
    return thrill::api::Future<size_t>(node);
}
template <typename ValueType, typename Stack>
size_t Size(const DIA<ValueType, Stack>& dia) { return SizeFuture(dia).get(); }

} // namespace thrill_gpu

#endif // !THRILL_GPU_NODES_HEADER
