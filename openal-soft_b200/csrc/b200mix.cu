// b200mix.cu — host side of the C ABI in include/b200mix.h.
//
// Owns the device-resident mirrors of the reference's mixer state (voices, buffers,
// mix buffers, HRTF accumulator carry) and issues the per-update launch sequence:
//   [k_apply_updates]  k_mix_voices  [k_hrtf_fir]  k_reduce_rows / post-process  (D2H)
// on one CUDA stream.  No CPU mixing path exists: every entry point fails with
// B200MIX_ERR_CUDA when the CUDA runtime/device is unusable.
#include "../../include/b200mix.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include <dlfcn.h>

#include "mixer_kernels.cuh"
#include "effect_kernels.cuh"
#include "shard_kernels.cuh"
#include "panmix_tc.cuh"
#include "param_kernels.hpp"
#include "efx_kernels.hpp"
#include "resampler_tables.hpp"
#include "hrtf_store.hpp"
#include "adpcm.hpp"
#include "callback_plan.hpp"
#include "device_memory.hpp"
#include "voice_book.hpp"
#include "slot_table.hpp"
#include "output_stage.hpp"

using namespace b200mix;

namespace {

thread_local std::string g_create_error;

} // namespace

struct b200mix_device {
    b200mix_device_desc desc{};
    int cuda_dev{0};
    int num_sms{0};
    cudaStream_t stream{nullptr};
    std::string error;
    uint64_t launches{0};

    // tables
    BsincTable bsinc[3];
    DevArray<float> d_bsinc[3], d_cubic[2];

    // state
    DevArray<VoiceRec> d_voices; DevArray<BufferRec> d_buffers;
    std::vector<BufferRec> h_buffers;
    std::vector<DevArray<char>> buf_store;       // per buffer: the samples its h_buffers record views
    VoiceBook book;                               // host mirror of the voices, source of d_order & co.
    DevArray<uint32_t> d_order;                   // book.order
    DevArray<float2> d_hrtf_tgt, d_hrtf_old;
    DevArray<float> d_dry_cur, d_dry_tgt, d_send_cur, d_send_tgt;
    VoiceResult *d_results{nullptr};              // inside d_outblock
    b200mix_voice_result *h_results{nullptr};     // inside h_outblock (pinned)
    DevArray<char> d_outblock; PinnedArray<char> h_outblock; size_t out_real_bytes{0};

    // mix buffers
    uint32_t dry_alloc_ch{0};
    DevArray<float> d_dry, d_wet;
    float *d_real{nullptr};                       // d_dry, or inside d_outblock
    DevArray<float> d_partial; size_t partial_floats{0};
    uint32_t fir_rows{0};                         // partial rows the last update's HRIR FIR stored
    float *h_real{nullptr};                       // pinned [real][1024]
    OutputStage out;                              // post-process, limiter, distance comp, interleaved output

    UploadArena stage;                            // b200mix_voices_update's inputs (see ensure_stage)

    // aux sends and effect slots
    SlotTable slots;                         // host side of the slots, source of d_slots
    DevArray<SlotRec> d_slots;
    std::vector<std::vector<DevArray<char>>> slot_allocs;   // per slot: what its record points into
    DevArray<float> d_xscratch; DevArray<uint32_t> d_sendinfo;   // parked lines and state bits
    // direct/send filters (allocated by the first b200mix_voices_filters)
    DevArray<FilterRec> d_filt;
    UploadArena fstage;                      // b200mix_voices_filters' inputs
    DevArray<float> d_fscratch, d_dline;     // [rows][1024]; [max_voices][1024] filtered direct-path lines
    DevArray<uint32_t> d_order2;             // book.order2
    DevArray<uint32_t> d_slot_start; DevArray<SendEntry> d_entries;   // book.slot_start / book.entries
    bool efx_ready{false};                   // efx_kernels_init has run (first b200mix_slot_efx)
    DevArray<float2> d_twiddle; DevArray<float> d_cubic_filter;   // gCubicTable (reverb modulation taps)

    // attached HRTF data set (device-side HrtfStore::getCoeffs)
    DevArray<float2> d_st_fields; DevArray<uint2> d_st_elevs; DevArray<float2> d_st_coeffs;
    DevArray<uint8_t> d_st_delays; uint32_t st_num_fields{0}, st_ir{0};
    DevArray<uint4> d_qhdr; DevArray<uint32_t> d_queue;   // streaming queues (ensure_queues)
    bool mid_render{false}; uint32_t mid_frames{0};   // between render_begin and render_end
    // parked dry bus (kernel variants without register dry accumulators)
    DevArray<SendEntry> d_dry_entries; DevArray<uint32_t> d_dry_slot_start;   // book.dry_entries
    DevArray<float> d_dry_partial;           // [kDryChunksMax][cd][1024]
    DevArray<float> d_dry_geff;              // [max_voices][cd]
    DevArray<float> d_send_geff;             // [max_voices*num_sends][cw]
    DevArray<float4> d_dry_gramp, d_send_gramp;
    DevArray<float> d_send_partial;          // [send_chunks][max_slots][cw][1024]
    // RealOut bus of the direct-channel voices (allocated by the first b200mix_voices_update_direct)
    DevArray<SendEntry> d_real_entries; DevArray<uint32_t> d_real_slot_start;   // book.real_entries
    DevArray<float> d_real_cur, d_real_tgt, d_real_geff;   // [max_voices][real_channels]
    DevArray<float4> d_real_gramp;
    bool real_mixed{false};                  // the last update mixed the RealOut bus
    bool profile{false};
    Event ev_mix0, ev_mix1;
    bool ev_valid{false};
    // stage marks of the last update (profile >= 2): see b200mix_last_stage_ms
    static constexpr int kStages = 8;
    Event ev_stage[kStages + 1];
    bool stage_valid{false}; int profile_level{0};

    // GPU parameter stage (b200mix_sources_update): pinned input staging + device scratch
    UploadArena src;
    bool panmix_tc{false};                   // wide dry buses: pan-mix past the fades on the tensor cores

    // voice-sharded device set (b200mix_shard_*): transport 0 none, 1 peer stores, 2 NCCL
    struct Shard {
        uint32_t rank{0}, world{1}; int transport{0};
        DevArray<char> own;
        char *peer[kShardMaxWorld]{};
        size_t off_real{0}, off_wet{0}, real_floats{0}, wet_src_floats{0};
        uint32_t owned_max{0};
        uint32_t epoch{0};
        DevArray<uint32_t> d_counters;         // [0] real push, [1] real sum, [2] wet sum, [4..] wet push per owner
        PinnedArray<uint32_t> h_status;        // pinned copy of ShardCtl::status
        Event ev[4];                           // wet exchange begin/end, RealOut reduce begin/end
        bool ev_wet{false}, ev_real{false};
        // NCCL transport (dlopen'ed: the library carries no link-time NCCL dependency)
        void *nccl_lib{nullptr}; void *comm{nullptr};
        int (*reduce)(const void*, void*, size_t, int, int, int, void*, cudaStream_t){nullptr};
        int (*allreduce)(const void*, void*, size_t, int, int, void*, cudaStream_t){nullptr};
        int (*comm_destroy)(void*){nullptr};
    } shard;

    uint32_t ir_pad{0};
    // resample kernel (resolved at create): k_mix_voices<kMixGS, kMixGroups, mix_cdr>
    void (*mix_fn)(const MixParams){nullptr};
    size_t mix_smem{0}; int mix_cdr{0}; int mix_blocks_per_sm{1};
    uint32_t reverb_seq{0};          // update counter of k_reverb_process' early/late hand-off (24 bits used)
    DevArray<uint32_t> d_claim;      // voice claim counters of the parking k_mix_voices
    int fir_blocks_per_sm{0};        // k_hrtf_fir CTAs per SM (HRTF devices)
    uint64_t fir_done{0};            // `launches` once the last update's k_hrtf_fir was launched

    // callback buffers (b200mix_buffer_callback): the registrations (plan slots), the host's
    // mirror of the voices that play them (positions advance by the same arithmetic as on the
    // device, so planning needs no read-back), and the pinned arenas their samples travel in,
    // alternating so that one can be filled while the other's copy is in flight
    struct CbBuf {
        bool used{false};
        uint32_t buffer{0};
        b200mix_callback_buffer cb{};
        cbplan::State st{};
        uint32_t frame_bytes{0};             // bytes per sample frame in the arena (int16 for ADPCM)
    };
    std::vector<CbBuf> cbs;
    std::vector<int32_t> cb_of_buffer;       // buffer id -> plan slot or -1
    struct CbVoice { int32_t slot{-1}; cbplan::Voice v{}; };
    std::vector<CbVoice> cbv;                // per voice
    uint32_t cb_bound{0};                    // voices bound to a callback buffer
    UploadArena cb_arena[2]; int cb_idx{0};
    DevArray<char> d_cb_zero;                // zeros behind every callback buffer's own record
    std::vector<int32_t> cb_reps;            // per slot: the voice the update is planned from (-1: none)
    std::vector<std::vector<uint32_t>> cb_members;   // per slot: its other mixing voices
    struct CbWork { cbplan::State start; cbplan::Loads loads; size_t region{0}, bytes{0}; };
    std::vector<CbWork> cb_work;             // per slot, for the update being planned
    ~b200mix_device() { if(stream) cudaStreamDestroy(stream); }
};

namespace {
constexpr uint32_t kCbMaxChannels = 16;      // a callback buffer's frame is at most 16*8 bytes
constexpr size_t kCbPad = 256;               // zero bytes that cover one such frame
}

namespace {

#define CUDA_TRY(dev, expr) do { cudaError_t e_ = (expr); if(e_ != cudaSuccess) {            \
    (dev)->error = std::string(#expr) + ": " + cudaGetErrorString(e_); return B200MIX_ERR_CUDA; } } while(0)

// Copies a host vector to the front of a device array, then synchronises the stream: the vector
// may be rebuilt (or go away) before an asynchronous copy would have read it.
template<typename T>
int upload(b200mix_device *d, DevArray<T> &dst, const std::vector<T> &src)
{
    if(!src.empty())
        CUDA_TRY(d, cudaMemcpyAsync(dst.get(), src.data(), src.size()*sizeof(T), cudaMemcpyHostToDevice, d->stream));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    return B200MIX_OK;
}

using MixKernel = void(*)(const MixParams);

// HRIR FIR kernel of an HRTF device: 17 outputs per thread / 64 front pad for ir <= 64,
// 19 / 128 for ir <= 128
struct FirVariant { MixKernel fn; size_t smem; };
FirVariant get_fir(uint32_t ir_size)
{
    if(ir_size <= 64u)
        return FirVariant{k_hrtf_fir<17, 64>, sizeof(FirSmem<kFirGS, 17, 64>)*kFirGroups};
    return FirVariant{k_hrtf_fir<19, 128>, sizeof(FirSmem<kFirGS, 19, 128>)*kFirGroups};
}

constexpr uint32_t kDryChunksMax = 128;

// The parts allocated on first use below go into locals and move into the device only once all
// succeeded: a failure leaves the device as it was, and the call can be retried.
// Parked lines and state bits of every voice: the parking k_mix_voices writes them, the sends,
// the direct filters and the parked dry bus read them.
int ensure_park_lines(b200mix_device *d)
{
    if(d->d_xscratch) return B200MIX_OK;
    const uint32_t nv = d->desc.max_voices;
    DevArray<float> xscratch; DevArray<uint32_t> sendinfo;
    CUDA_TRY(d, xscratch.alloc(size_t(nv)*kLine, d->stream));
    CUDA_TRY(d, sendinfo.alloc(nv, d->stream));
    d->d_xscratch = std::move(xscratch); d->d_sendinfo = std::move(sendinfo);
    return B200MIX_OK;
}

// Storage of the parked dry bus (variants with CDR == 0 that meet a non-HRTF voice).
int ensure_dry_park(b200mix_device *d)
{
    const b200mix_device_desc &dd = d->desc;
    if(d->d_dry_entries) return B200MIX_OK;
    if(int rc = ensure_park_lines(d)) return rc;
    if(dd.dry_channels > 4u && dd.dry_channels <= uint32_t(kPmN))
    {
        CUDA_TRY(d, cudaFuncSetAttribute(k_panmix_tc, cudaFuncAttributeMaxDynamicSharedMemorySize,
            kPmStages*kPmStageBytes + 1024));
        // B200MIX_PANMIX_SIMT=1 keeps the whole pan-mix on k_send_mix (A/B measurements only)
        const char *simt = std::getenv("B200MIX_PANMIX_SIMT");
        d->panmix_tc = !(simt && simt[0] == '1');
    }
    DevArray<SendEntry> entries; DevArray<uint32_t> slotStart;
    DevArray<float> partial, geff; DevArray<float4> gramp;
    CUDA_TRY(d, entries.alloc(dd.max_voices, d->stream));
    CUDA_TRY(d, slotStart.alloc(2, d->stream));
    CUDA_TRY(d, partial.alloc(size_t(kDryChunksMax)*dd.dry_channels*kLine, d->stream));
    CUDA_TRY(d, geff.alloc(size_t(dd.max_voices)*dd.dry_channels, d->stream));
    CUDA_TRY(d, gramp.alloc(size_t(dd.max_voices)*dd.dry_channels, d->stream));
    d->d_dry_entries = std::move(entries); d->d_dry_slot_start = std::move(slotStart);
    d->d_dry_partial = std::move(partial); d->d_dry_geff = std::move(geff); d->d_dry_gramp = std::move(gramp);
    return B200MIX_OK;
}

// Storage of the RealOut bus (the first direct-channel voice): the parked lines, the voices'
// RealOut gains and the bus' entries.
int ensure_real_bus(b200mix_device *d)
{
    const b200mix_device_desc &dd = d->desc;
    if(d->d_real_entries) return B200MIX_OK;
    if(int rc = ensure_park_lines(d)) return rc;
    const size_t gains = size_t(dd.max_voices)*dd.real_channels;
    DevArray<SendEntry> entries; DevArray<uint32_t> slotStart;
    DevArray<float> cur, tgt, geff; DevArray<float4> gramp;
    CUDA_TRY(d, entries.alloc(dd.max_voices, d->stream));
    CUDA_TRY(d, slotStart.alloc(2, d->stream));
    CUDA_TRY(d, cur.alloc(gains, d->stream));
    CUDA_TRY(d, tgt.alloc(gains, d->stream));
    CUDA_TRY(d, geff.alloc(gains, d->stream));
    CUDA_TRY(d, gramp.alloc(gains, d->stream));
    d->d_real_entries = std::move(entries); d->d_real_slot_start = std::move(slotStart);
    d->d_real_cur = std::move(cur); d->d_real_tgt = std::move(tgt);
    d->d_real_geff = std::move(geff); d->d_real_gramp = std::move(gramp);
    return B200MIX_OK;
}

// Queue tables of the streaming voices (the first voice that reads a queue).
int ensure_queues(b200mix_device *d)
{
    if(d->d_qhdr) return B200MIX_OK;
    const uint32_t nv = d->desc.max_voices;
    DevArray<uint4> qhdr; DevArray<uint32_t> queue;
    CUDA_TRY(d, qhdr.alloc(nv, d->stream));
    CUDA_TRY(d, queue.alloc(size_t(nv)*kMaxQueue, d->stream));
    d->d_qhdr = std::move(qhdr); d->d_queue = std::move(queue);
    return B200MIX_OK;
}

// Refreshes the slot table and uploads every record.
int refresh_slots(b200mix_device *d)
{
    d->slots.refresh();
    std::vector<SlotRec> recs(d->slots.size());
    for(uint32_t sl = 0;sl < recs.size();++sl) recs[sl] = d->slots[sl].rec;
    return upload(d, d->d_slots, recs);
}

// Disables the slot.  The device's record is zeroed before the memory it points into is freed.
int free_slot(b200mix_device *d, uint32_t slot)
{
    d->slots.release(slot);
    if(int rc = refresh_slots(d)) return rc;
    d->slot_allocs[slot].clear();
    return B200MIX_OK;
}

// Installs an effect on `slot`: releases what the slot held; `fill` allocates (`alloc`: `count` zeroed
// T, owned by the slot until free_slot) and fills the record and the table's host state; the table is
// refreshed and uploaded.  An install that fails leaves the slot disabled, holding no memory.
template<typename Fill>
int install_slot(b200mix_device *d, uint32_t slot, Fill &&fill)
{
    if(int rc = free_slot(d, slot)) return rc;
    auto alloc = [&]<typename T>(T *&p, size_t count) -> int {
        DevArray<char> a;
        CUDA_TRY(d, a.alloc(count*sizeof(T), d->stream));
        p = reinterpret_cast<T*>(a.get());
        d->slot_allocs[slot].push_back(std::move(a));
        return B200MIX_OK;
    };
    if(int rc = fill(d->slots[slot].rec, alloc)) { free_slot(d, slot); return rc; }
    d->book.dry_active = true;
    return refresh_slots(d);
}

static size_t align16(size_t v) { return UploadArena::align(v); }

// b200mix_voices_update's arena: a call packs [VoiceUpdate n][coefficients or directions]
// [dry or RealOut gains][send gains] and ships them with one copy.  It holds at least 256 voices,
// each with room for the wider of the Dry mix's gains and RealOut's (direct-channel voices).
int ensure_stage(b200mix_device *d, uint32_t n)
{
    const b200mix_device_desc &dd = d->desc;
    const uint32_t cap = std::max<uint32_t>(n, 256u);
    const size_t bytes = align16(size_t(cap)*sizeof(VoiceUpdate))
        + align16(size_t(cap)*std::max<size_t>(size_t(dd.ir_size)*2, 4)*sizeof(float))
        + align16(size_t(cap)*std::max(dd.dry_channels, dd.real_channels)*sizeof(float))
        + align16(size_t(cap)*dd.num_sends*dd.wet_channels*sizeof(float)) + 64;
    CUDA_TRY(d, d->stage.reserve(n, cap, bytes, bytes, d->stream));
    return B200MIX_OK;
}

const BsincTable *bsinc_for(const b200mix_device *d, uint32_t resampler)
{
    if(resampler < B200MIX_RESAMPLER_FAST_BSINC12 || resampler > B200MIX_RESAMPLER_BSINC48)
        return nullptr;
    return &d->bsinc[(resampler - B200MIX_RESAMPLER_FAST_BSINC12) >> 1];
}

// Plan slot of the callback buffer an entry plays (-1: none).
int32_t cb_slot_of(const b200mix_device *d, uint32_t flags, uint32_t buffer)
{
    return (!(flags & B200MIX_VF_STOPPED) && buffer != B200MIX_NO_BUFFER && !d->cb_of_buffer.empty())
        ? d->cb_of_buffer[buffer] : -1;
}

// The checks b200mix_voices_update and b200mix_sources_update make of every entry before the call
// changes anything; `what` prefixes the error.  They may allocate the queue tables and the parked
// dry bus, which leave the device as it was if they fail.  `nobuf_ok`: the entry may name
// B200MIX_NO_BUFFER; `hrtf`: the voice does not mix into Dry (it has its own HRIR, or is a
// direct-channel voice).
template<typename Entry>
int check_entry(b200mix_device *d, const char *what, const Entry &p, bool nobuf_ok, bool hrtf)
{
    const b200mix_device_desc &dd = d->desc;
    const bool stopped = (p.flags & B200MIX_VF_STOPPED) != 0;
    const bool nobuf = nobuf_ok && p.buffer == B200MIX_NO_BUFFER;
    auto bad = [&](const char *why) { d->error = std::string(what) + ": " + why; return B200MIX_ERR_INVALID; };
    if(p.voice >= dd.max_voices || p.resampler > B200MIX_RESAMPLER_BSINC48
        || (!stopped && !nobuf && p.buffer >= dd.max_buffers))
        return bad("voice/buffer/resampler out of range");
    if((p.flags & B200MIX_VF_LOOPING) && p.loop_end <= p.loop_start)
        return bad("empty loop");
    // nothing to read without a buffer; a callback voice reads from the update's arena
    if(!stopped && !nobuf && cb_slot_of(d, p.flags, p.buffer) < 0)
    {
        if(p.flags & B200MIX_VF_STATIC)
        {
            const BufferRec &hb = d->h_buffers[p.buffer];
            if(!hb.data || !hb.frames) return bad("static voice on a buffer without data");
            if((p.flags & B200MIX_VF_LOOPING) && p.loop_end > hb.frames) return bad("loop end beyond the buffer");
        }
        // a streaming voice reads its queue: make sure the (empty) queue table exists
        else if(int rc = ensure_queues(d)) return rc;
    }
    for(uint32_t s = 0;s < dd.num_sends;++s)
        if(p.send_slot[s] != B200MIX_NO_SLOT && p.send_slot[s] >= dd.max_slots)
            return bad("send slot out of range");
    if(!stopped && !hrtf && d->mix_cdr == 0)
        if(int rc = ensure_dry_park(d)) return rc;
    return B200MIX_OK;
}

// k_apply_updates' parameters that do not depend on the entry point.
ApplyParams apply_params(const b200mix_device *d, const VoiceUpdate *updates)
{
    const b200mix_device_desc &dd = d->desc;
    ApplyParams A{};
    A.voices = d->d_voices; A.updates = updates;
    A.hrtf_tgt = d->d_hrtf_tgt; A.hrtf_old = d->d_hrtf_old;
    A.dry_cur = d->d_dry_cur; A.dry_tgt = d->d_dry_tgt;
    A.send_cur = d->d_send_cur; A.send_tgt = d->d_send_tgt;
    A.ir = dd.ir_size; A.ir_pad = d->ir_pad; A.cd = dd.dry_channels; A.cw = dd.wet_channels;
    A.num_sends = dd.num_sends;
    A.filt = d->d_filt; A.filt_paths = 1u + dd.num_sends;
    A.qhdr = d->d_qhdr;
    A.real_cur = d->d_real_cur; A.real_tgt = d->d_real_tgt; A.creal = dd.real_channels;
    return A;
}

// Entries given as directions: the HRIRs are blended on the device from the attached data set.
void apply_dirs(const b200mix_device *d, ApplyParams &A, const float4 *dirs)
{
    A.dirs = dirs;
    A.st_fields = d->d_st_fields; A.st_elevs = d->d_st_elevs; A.st_coeffs = d->d_st_coeffs;
    A.st_delays = d->d_st_delays; A.st_num_fields = d->st_num_fields; A.st_ir = d->st_ir;
}

// Every output-stage setter: refused while a render_begin is pending; then, on the mixer's GPU, the
// stage checks the arguments and builds and commits the new state (OutputStage).
template<typename... Params, typename... Args>
int set_output(b200mix_device *d, const char *what, int (OutputStage::*set)(Params...), Args... args)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(d->mid_render) { d->error = std::string(what) + ": a render_begin is pending"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    return (d->out.*set)(args...);
}

} // namespace

extern "C" {

static void shard_release(b200mix_device *d);
static int ensure_filters(b200mix_device *d);

uint32_t b200mix_version(void) { return (1u<<16) | 3u; }

const char *b200mix_last_error(const b200mix_device *dev)
{ return dev ? dev->error.c_str() : g_create_error.c_str(); }

int b200mix_create(const b200mix_device_desc *desc, b200mix_device **out)
{
    if(!desc || !out || desc->struct_size != sizeof(b200mix_device_desc))
    { g_create_error = "bad descriptor"; return B200MIX_ERR_INVALID; }
    if(desc->dry_channels > B200MIX_MAX_DRY_CHANNELS || desc->wet_channels > B200MIX_MAX_WET_CHANNELS
        || desc->num_sends > B200MIX_MAX_SENDS || desc->ir_size > B200MIX_HRIR_LENGTH
        || desc->real_channels > B200MIX_MAX_DRY_CHANNELS || desc->max_voices == 0)
    { g_create_error = "descriptor out of range"; return B200MIX_ERR_INVALID; }
    if((desc->post_process == B200MIX_POST_UHJ && desc->dry_channels < 3)
        || (desc->post_process == B200MIX_POST_TSME && desc->dry_channels < 4))
    { g_create_error = "UHJ post-process needs W,X,Y dry channels"; return B200MIX_ERR_INVALID; }
    if((desc->post_process == B200MIX_POST_HRTF || desc->post_process == B200MIX_POST_UHJ
        || desc->post_process == B200MIX_POST_TSME)
        && (desc->real_left >= desc->real_channels || desc->real_right >= desc->real_channels))
    { g_create_error = "real_left/real_right outside RealOut"; return B200MIX_ERR_INVALID; }

    auto *d = new(std::nothrow) b200mix_device{};
    if(!d) { g_create_error = "out of host memory"; return B200MIX_ERR_NOMEM; }
    d->desc = *desc;
    auto fail = [&](int code) { g_create_error = d->error; b200mix_destroy(d); return code; };

    int count = 0;
    if(cudaGetDeviceCount(&count) != cudaSuccess || count < 1)
    { d->error = "no CUDA device: the b200mix mixer has no CPU path"; return fail(B200MIX_ERR_CUDA); }
    if(desc->cuda_device >= 0) d->cuda_dev = desc->cuda_device;
    else if(cudaGetDevice(&d->cuda_dev) != cudaSuccess) d->cuda_dev = 0;
    if(cudaSetDevice(d->cuda_dev) != cudaSuccess)
    { d->error = "cudaSetDevice failed"; return fail(B200MIX_ERR_CUDA); }
    cudaDeviceProp prop{};
    if(cudaGetDeviceProperties(&prop, d->cuda_dev) != cudaSuccess)
    { d->error = "cudaGetDeviceProperties failed"; return fail(B200MIX_ERR_CUDA); }
    d->num_sms = prop.multiProcessorCount;
    if(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess)
    { d->error = "cudaStreamCreate failed"; return fail(B200MIX_ERR_CUDA); }

    auto run = [&]() -> int {
        // resampler tables (core/bsinc_tables.cpp:150-155)
        d->bsinc[0] = BuildBsincTable(60, 11, 2);
        d->bsinc[1] = BuildBsincTable(60, 23, 2);
        d->bsinc[2] = BuildBsincTable(80, 47, 1);
        for(int i = 0;i < 3;++i)
        {
            CUDA_TRY(d, d->d_bsinc[i].alloc(d->bsinc[i].tab.size()));
            if(int rc = upload(d, d->d_bsinc[i], d->bsinc[i].tab)) return rc;
        }
        const std::vector<float> cubic[2] = {BuildSplineTable(), BuildGaussianTable()};
        for(int i = 0;i < 2;++i)
        {
            CUDA_TRY(d, d->d_cubic[i].alloc(cubic[i].size()));
            if(int rc = upload(d, d->d_cubic[i], cubic[i])) return rc;
        }

        const b200mix_device_desc &dd = d->desc;
        d->ir_pad = (dd.ir_size + 7u) & ~7u;
        CUDA_TRY(d, d->d_voices.alloc(dd.max_voices, d->stream));
        CUDA_TRY(d, d->d_buffers.alloc(std::max(dd.max_buffers, 1u), d->stream));
        d->h_buffers.assign(std::max(dd.max_buffers, 1u), BufferRec{});
        d->buf_store.resize(d->h_buffers.size());
        d->book.init(dd.max_voices, dd.max_buffers, dd.num_sends, dd.max_slots);
        if(dd.ir_size)
        {
            CUDA_TRY(d, d->d_hrtf_tgt.alloc(size_t(dd.max_voices)*d->ir_pad, d->stream));
            CUDA_TRY(d, d->d_hrtf_old.alloc(size_t(dd.max_voices)*d->ir_pad, d->stream));
        }
        CUDA_TRY(d, d->d_dry_cur.alloc(size_t(dd.max_voices)*std::max(dd.dry_channels, 1u), d->stream));
        CUDA_TRY(d, d->d_dry_tgt.alloc(size_t(dd.max_voices)*std::max(dd.dry_channels, 1u), d->stream));
        if(dd.num_sends && dd.wet_channels)
        {
            const size_t per = size_t(dd.num_sends)*dd.wet_channels;
            CUDA_TRY(d, d->d_send_cur.alloc(dd.max_voices*per, d->stream));
            CUDA_TRY(d, d->d_send_tgt.alloc(dd.max_voices*per, d->stream));
        }
        CUDA_TRY(d, d->d_order.alloc(dd.max_voices, d->stream));

        // resample kernel: non-HRTF devices with <= 4 dry channels mix the dry bus in registers;
        // HRTF devices and wider dry mixes resample + park (k_hrtf_fir mixes the HRTF voices,
        // k_send_mix sums the dry bus)
        const bool hrtfDev = dd.ir_size > 0;
        if(!hrtfDev && dd.dry_channels <= 4)
        {
            d->mix_cdr = 4;
            d->mix_fn = k_mix_voices<kMixGS, kMixGroups, 4>;
            d->mix_smem = sizeof(GroupSmem<4>)*kMixGroups;
        }
        else
        {
            d->mix_cdr = 0;
            d->mix_fn = k_mix_voices<kMixGS, kMixGroups, 0>;
            d->mix_smem = sizeof(GroupSmem<0>)*kMixGroups;
        }
        CUDA_TRY(d, cudaFuncSetAttribute(d->mix_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(d->mix_smem)));
        int perSm = 0;
        CUDA_TRY(d, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, d->mix_fn, kMixGS*kMixGroups,
            d->mix_smem));
        d->mix_blocks_per_sm = std::max(perSm, 1);
        if(d->mix_cdr == 0)
        {
            // the parking variant writes every mixed voice's line and state bits
            if(int rc = ensure_park_lines(d)) return rc;
            CUDA_TRY(d, d->d_claim.alloc(2, d->stream));
        }
        if(hrtfDev)
        {
            const FirVariant fir = get_fir(dd.ir_size);
            CUDA_TRY(d, cudaFuncSetAttribute(fir.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(fir.smem)));
            CUDA_TRY(d, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, fir.fn, kFirGS*kFirGroups, fir.smem));
            // the FIR grid sets the partial rows, hence the summation order: it is fixed at
            // kFirCtasPerSm per SM (the launch bounds), not at whatever more might fit
            d->fir_blocks_per_sm = std::max(std::min(perSm, kFirCtasPerSm), 1);
        }

        d->dry_alloc_ch = std::max<uint32_t>(std::max(dd.dry_channels, 1u), uint32_t(d->mix_cdr));
        CUDA_TRY(d, d->d_dry.alloc(size_t(d->dry_alloc_ch)*kLine, d->stream));
        // RealOut and the voice results share one block (and one pinned mirror): a render that
        // returns both needs ONE device-to-host copy
        {
            const size_t realFloats = size_t(std::max(dd.real_channels, 1u))*kLine;
            static_assert(sizeof(VoiceResult) == 16 && sizeof(b200mix_voice_result) == 16, "result layout");
            const size_t blockBytes = realFloats*sizeof(float) + size_t(dd.max_voices)*sizeof(VoiceResult);
            CUDA_TRY(d, d->d_outblock.alloc(blockBytes, d->stream));
            char *blk = d->d_outblock;
            d->d_results = reinterpret_cast<VoiceResult*>(blk + realFloats*sizeof(float));
            CUDA_TRY(d, d->h_outblock.alloc(blockBytes));
            d->h_real = reinterpret_cast<float*>(d->h_outblock.get());
            d->h_results = reinterpret_cast<b200mix_voice_result*>(d->h_outblock + realFloats*sizeof(float));
            d->out_real_bytes = realFloats*sizeof(float);
            if(dd.post_process == B200MIX_POST_NONE) d->d_real = d->d_dry;
            else d->d_real = reinterpret_cast<float*>(blk);
        }
        if(dd.max_slots && dd.wet_channels)
            CUDA_TRY(d, d->d_wet.alloc(size_t(dd.max_slots)*dd.wet_channels*kLine, d->stream));
        // partial rows: the FIR's HrtfAccumData rows (HRTF devices), or the register dry bus'
        // rows in two regions, k_mix_voices' and k_mix_deferred's (voices with direct filters)
        d->partial_floats = hrtfDev ? size_t(d->num_sms)*d->fir_blocks_per_sm*(2*kAccumLen)
            : size_t(d->num_sms)*d->mix_blocks_per_sm*size_t(d->mix_cdr)*kLine;
        CUDA_TRY(d, d->d_partial.alloc(std::max<size_t>((hrtfDev ? 1 : 2)*d->partial_floats, 4), d->stream));
        if(int rc = d->out.init(dd, d->stream, d->error)) return rc;
        if(dd.max_slots && dd.wet_channels && dd.num_sends)
        {
            d->slots.init(dd.max_slots, uint32_t(d->num_sms));
            d->slot_allocs.resize(dd.max_slots);
            CUDA_TRY(d, d->d_slots.alloc(dd.max_slots, d->stream));
            CUDA_TRY(d, cudaFuncSetAttribute(k_conv_mac, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(ConvMacSmem))));
            CUDA_TRY(d, cudaFuncSetAttribute(k_reverb_upmix, cudaFuncAttributeMaxDynamicSharedMemorySize, int(8*kLine*sizeof(float))));
            if(int rc = ensure_park_lines(d)) return rc;
            CUDA_TRY(d, d->d_send_geff.alloc(size_t(dd.max_voices)*dd.num_sends*dd.wet_channels, d->stream));
            CUDA_TRY(d, d->d_send_gramp.alloc(size_t(dd.max_voices)*dd.num_sends*dd.wet_channels, d->stream));
            CUDA_TRY(d, d->d_slot_start.alloc(dd.max_slots + 1, d->stream));
            CUDA_TRY(d, d->d_entries.alloc(size_t(dd.max_voices)*dd.num_sends, d->stream));
            std::vector<float2> tw(128);
            for(int k = 0;k < 128;++k)
            {
                const double a = -2.0*3.14159265358979323846*double(k)/256.0;
                tw[k] = make_float2(float(std::cos(a)), float(std::sin(a)));
            }
            const std::vector<float> cf = BuildCubicFilter();
            CUDA_TRY(d, d->d_cubic_filter.alloc(cf.size()));
            if(int rc = upload(d, d->d_cubic_filter, cf)) return rc;
            CUDA_TRY(d, d->d_twiddle.alloc(tw.size()));
            if(int rc = upload(d, d->d_twiddle, tw)) return rc;
        }
        if(int rc = ensure_stage(d, std::min(dd.max_voices, 4096u))) return rc;
        CUDA_TRY(d, cudaStreamSynchronize(d->stream));
        return B200MIX_OK;
    };
    int rc;
    try { rc = run(); }
    catch(const std::exception &e) { d->error = e.what(); rc = B200MIX_ERR_NOMEM; }
    if(rc != B200MIX_OK) return fail(rc);
    *out = d;
    return B200MIX_OK;
}

void b200mix_destroy(b200mix_device *d)
{
    if(!d) return;
    if(d->stream)
    {
        cudaSetDevice(d->cuda_dev);
        cudaStreamSynchronize(d->stream);
    }
    shard_release(d);
    delete d;
}

int b200mix_set_hrtf_decoder(b200mix_device *d, uint32_t channels, uint32_t ir_size,
    const float *coeffs, const float *hf_scale, const float *splitter_coeff)
{
    return set_output(d, "set_hrtf_decoder", &OutputStage::set_hrtf_decoder, channels, ir_size, coeffs, hf_scale,
        splitter_coeff);
}

int b200mix_set_ambi_decoder(b200mix_device *d, uint32_t in_channels, const float *gains_hf,
    const float *gains_lf, float xover_coeff)
{
    return set_output(d, "set_ambi_decoder", &OutputStage::set_ambi_decoder, in_channels, gains_hf, gains_lf,
        xover_coeff);
}

// Voices that play callback plan slot s (playing or stopping).
static uint32_t cb_slot_voices(const b200mix_device *d, int32_t s)
{
    uint32_t n = 0;
    for(uint32_t v = 0;v < d->cbv.size() && v < d->book.voice_hi;++v)
        n += d->cbv[v].slot == s && (d->cbv[v].v.state == 1u || d->cbv[v].v.state == 2u);
    return n;
}

// Ends the callback registration of `buffer` (if any); refused while a voice plays it.
static int cb_unregister(b200mix_device *d, uint32_t buffer, const char *what)
{
    if(d->cb_of_buffer.empty() || d->cb_of_buffer[buffer] < 0) return B200MIX_OK;
    const int32_t s = d->cb_of_buffer[buffer];
    if(cb_slot_voices(d, s))
    { d->error = std::string(what) + ": the callback buffer is played by a voice; stop it first"; return B200MIX_ERR_INVALID; }
    for(auto &cv : d->cbv)
        if(cv.slot == s) { cv.slot = -1; --d->cb_bound; }
    d->cbs[size_t(s)] = b200mix_device::CbBuf{};
    d->cb_of_buffer[buffer] = -1;
    d->h_buffers[buffer] = BufferRec{};
    CUDA_TRY(d, cudaMemcpyAsync(d->d_buffers + buffer, &d->h_buffers[buffer], sizeof(BufferRec),
        cudaMemcpyHostToDevice, d->stream));
    return B200MIX_OK;
}

int b200mix_buffer_callback(b200mix_device *d, uint32_t buffer, const b200mix_callback_buffer *cb)
{
    if(!d) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    if(buffer >= dd.max_buffers || !cb || cb->struct_size != sizeof(b200mix_callback_buffer) || !cb->callback
        || cb->sample_type > B200MIX_FMT_MSADPCM || cb->channels < 1 || !cb->storage
        || cb->samples_per_block < 1 || cb->bytes_per_block < 1)
    { d->error = "buffer_callback: bad arguments"; return B200MIX_ERR_INVALID; }
    static const uint32_t sz[] = {1, 2, 4, 4, 8, 1, 1};
    const bool adpcm = cb->sample_type >= B200MIX_FMT_IMA4;
    const bool ms = cb->sample_type == B200MIX_FMT_MSADPCM;
    if(adpcm ? (cb->channels > 2 || !AdpcmBlockValid(ms, cb->samples_per_block)
                || cb->bytes_per_block != AdpcmBlockBytes(ms, cb->channels, cb->samples_per_block))
             : (cb->samples_per_block != 1u || cb->bytes_per_block != cb->channels*sz[cb->sample_type]))
    { d->error = "buffer_callback: block size does not match the format"; return B200MIX_ERR_INVALID; }
    if(cb->channels > kCbMaxChannels)
    { d->error = "buffer_callback: more than 16 channels"; return B200MIX_ERR_UNSUPPORTED; }
    // PrepareCallback's size (al/buffer.cpp:468-473): MixerLineSize*MaxPitch + MaxResamplerEdge
    // samples in whole blocks.  No request of the reference's chunk loop passes it, so the
    // callbacks of an update never stop half way.
    const uint64_t lineBlocks = ((1024u + 256u)*10u + 24u + cb->samples_per_block - 1u) / cb->samples_per_block;
    if(cb->storage_bytes < lineBlocks*cb->bytes_per_block)
    { d->error = "buffer_callback: storage smaller than the reference's callback storage"; return B200MIX_ERR_INVALID; }
    if(uint64_t(cb->num_blocks)*cb->bytes_per_block > cb->storage_bytes || cb->stopped > 1u)
    { d->error = "buffer_callback: state outside the storage"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(!d->d_cb_zero)
        CUDA_TRY(d, d->d_cb_zero.alloc(kCbPad, d->stream));
    if(d->cb_of_buffer.empty())
    {
        d->cb_of_buffer.assign(dd.max_buffers, -1);
        d->cbv.assign(dd.max_voices, b200mix_device::CbVoice{});
    }
    BufferRec &h = d->h_buffers[buffer];
    int32_t s = d->cb_of_buffer[buffer];
    if(s < 0)
    {
        if(h.data && d->book.bufrefs[buffer])
        { d->error = "buffer_callback: the buffer is attached to an active voice (AL_INVALID_OPERATION)"; return B200MIX_ERR_INVALID; }
        if(h.data)
        {
            CUDA_TRY(d, cudaStreamSynchronize(d->stream));
            d->buf_store[buffer].reset();
        }
        for(s = 0;size_t(s) < d->cbs.size() && d->cbs[size_t(s)].used;++s) {}
        if(size_t(s) == d->cbs.size()) d->cbs.emplace_back();
        d->cb_of_buffer[buffer] = s;
    }
    b200mix_device::CbBuf &c = d->cbs[size_t(s)];
    c.used = true; c.buffer = buffer; c.cb = *cb;
    c.st = cbplan::State{cb->num_blocks, cb->block_offset, cb->stopped};
    c.frame_bytes = cb->channels*(adpcm ? 2u : sz[cb->sample_type]);
    // the kernel reads the samples from the update's arena: the record carries the format, and
    // zeros to read should a voice ever meet it without a plan
    h = BufferRec{};
    h.data = d->d_cb_zero.get();
    h.type = adpcm ? uint32_t(B200MIX_FMT_I16) : cb->sample_type;
    h.channels = cb->channels;
    h.pad = uint32_t(s) + 1u;
    CUDA_TRY(d, cudaMemcpyAsync(d->d_buffers + buffer, &h, sizeof(BufferRec), cudaMemcpyHostToDevice, d->stream));
    return B200MIX_OK;
}

int b200mix_buffer_callback_state(b200mix_device *d, uint32_t buffer, uint32_t *num_blocks,
    uint32_t *block_offset, uint32_t *stopped)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(buffer >= d->desc.max_buffers || d->cb_of_buffer.empty() || d->cb_of_buffer[buffer] < 0)
    { d->error = "buffer_callback_state: not a callback buffer"; return B200MIX_ERR_INVALID; }
    const cbplan::State &st = d->cbs[size_t(d->cb_of_buffer[buffer])].st;
    if(num_blocks) *num_blocks = st.num_blocks;
    if(block_offset) *block_offset = st.block_offset;
    if(stopped) *stopped = st.stopped;
    return B200MIX_OK;
}

int b200mix_buffer_data(b200mix_device *d, uint32_t buffer, uint32_t sample_type, uint32_t channels,
    uint32_t frames, const void *data, size_t bytes)
{
    if(!d) return B200MIX_ERR_INVALID;
    static const size_t sz[] = {1, 2, 4, 4, 8, 1, 1};
    if(buffer >= d->desc.max_buffers || sample_type > B200MIX_FMT_ALAW || channels < 1 || !data)
    { d->error = "buffer_data: bad arguments"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(int rc = cb_unregister(d, buffer, "buffer_data")) return rc;
    const size_t need = size_t(frames)*channels*sz[sample_type];
    if(bytes < need) { d->error = "buffer_data: short data"; return B200MIX_ERR_INVALID; }
    BufferRec &h = d->h_buffers[buffer];
    if(h.data && d->book.bufrefs[buffer])
    { d->error = "buffer_data: the buffer is attached to an active voice (AL_INVALID_OPERATION)"; return B200MIX_ERR_INVALID; }
    DevArray<char> &store = d->buf_store[buffer];
    if(h.data)
    {
        CUDA_TRY(d, cudaStreamSynchronize(d->stream));
        store.reset();
        h = BufferRec{};
    }
    // +16 bytes so vector/tail reads past the last frame stay inside the allocation
    CUDA_TRY(d, store.alloc(need + 16));
    CUDA_TRY(d, cudaMemcpyAsync(store.get(), data, need, cudaMemcpyHostToDevice, d->stream));
    h.data = store.get(); h.frames = frames; h.type = sample_type; h.channels = channels;
    CUDA_TRY(d, cudaMemcpyAsync(d->d_buffers + buffer, &h, sizeof(BufferRec), cudaMemcpyHostToDevice,
        d->stream));
    return B200MIX_OK;
}

int b200mix_buffer_data_adpcm(b200mix_device *d, uint32_t buffer, uint32_t sample_type,
    uint32_t channels, uint32_t samples_per_block, uint32_t blocks, const void *data, size_t bytes)
{
    if(!d) return B200MIX_ERR_INVALID;
    const bool ms = sample_type == B200MIX_FMT_MSADPCM;
    if((sample_type != B200MIX_FMT_IMA4 && !ms) || channels < 1 || channels > 2 || !data
        || !AdpcmBlockValid(ms, samples_per_block))
    { d->error = "buffer_data_adpcm: bad arguments"; return B200MIX_ERR_INVALID; }
    if(bytes < AdpcmBlockBytes(ms, channels, samples_per_block)*blocks
        || uint64_t(blocks)*samples_per_block > 0x7fffffffull)
    { d->error = "buffer_data_adpcm: short data"; return B200MIX_ERR_INVALID; }
    std::vector<int16_t> pcm(size_t(blocks)*samples_per_block*channels);
    if(ms) DecodeMSADPCM(static_cast<const uint8_t*>(data), channels, samples_per_block, blocks, pcm.data());
    else DecodeIMA4(static_cast<const uint8_t*>(data), channels, samples_per_block, blocks, pcm.data());
    const int rc = b200mix_buffer_data(d, buffer, B200MIX_FMT_I16, channels, blocks*samples_per_block,
        pcm.data(), pcm.size()*sizeof(int16_t));
    // the upload above reads pageable memory: make sure it is consumed before pcm goes away
    if(rc == B200MIX_OK) CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    return rc;
}

int b200mix_buffer_free(b200mix_device *d, uint32_t buffer)
{
    if(!d || buffer >= d->desc.max_buffers) return B200MIX_ERR_INVALID;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(int rc = cb_unregister(d, buffer, "buffer_free")) return rc;
    BufferRec &h = d->h_buffers[buffer];
    if(h.data && d->book.bufrefs[buffer])
    { d->error = "buffer_free: the buffer is attached to an active voice; stop the voice first"; return B200MIX_ERR_INVALID; }
    if(h.data)
    {
        CUDA_TRY(d, cudaStreamSynchronize(d->stream));
        d->buf_store[buffer].reset();
        h = BufferRec{};
        CUDA_TRY(d, cudaMemcpyAsync(d->d_buffers + buffer, &h, sizeof(BufferRec),
            cudaMemcpyHostToDevice, d->stream));
    }
    return B200MIX_OK;
}

int b200mix_slot_disable(b200mix_device *d, uint32_t slot)
{
    if(!d || slot >= d->slots.size()) { if(d) d->error = "slot_disable: bad slot"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    return free_slot(d, slot);
}

int b200mix_slot_convolution(b200mix_device *d, uint32_t slot, uint32_t ir_channels,
    uint32_t ir_frames, const float *ir)
{
    if(!d || slot >= d->slots.size() || !ir_channels || ir_channels > 16 || !ir_frames || !ir)
    { if(d) d->error = "slot_convolution: bad arguments (or the device has no sends/slots)"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    // mNumConvolveSegs (alc/effects/convolution.cpp:375-376)
    const uint32_t nseg = std::max<uint32_t>((ir_frames + kConvBlock - 1)/kConvBlock, 2u) - 1u;

    // Filter spectra: segment s holds taps [128(s+1), 128(s+2)), zero padded to 256,
    // transformed in f64 and scaled by 1/256 (convolution.cpp:425-468); layout is ours.
    std::vector<float> H(size_t(ir_channels)*nseg*kConvFft, 0.0f), head(size_t(ir_channels)*kConvBlock, 0.0f);
    std::vector<double> cs(kConvFft), sn(kConvFft);
    for(int k = 0;k < kConvFft;++k)
    {
        cs[k] = std::cos(2.0*3.14159265358979323846*k/kConvFft);
        sn[k] = std::sin(2.0*3.14159265358979323846*k/kConvFft);
    }
    for(uint32_t c = 0;c < ir_channels;++c)
    {
        const float *h = ir + size_t(c)*ir_frames;
        for(uint32_t k = 0;k < uint32_t(kConvBlock) && k < ir_frames;++k) head[c*kConvBlock + k] = h[k];
        for(uint32_t sg = 0;sg < nseg;++sg)
        {
            const size_t base = size_t(kConvBlock)*(sg + 1);
            float *dst = H.data() + (size_t(c)*nseg + sg)*kConvFft;
            const uint32_t cnt = base < ir_frames ? std::min<uint32_t>(kConvBlock, uint32_t(ir_frames - base)) : 0u;
            for(int bin = 0;bin <= kConvBlock;++bin)
            {
                double re = 0.0, im = 0.0;
                for(uint32_t j = 0;j < cnt;++j)
                {
                    const int ph = int((uint64_t(bin)*j) % kConvFft);
                    re += double(h[base + j])*cs[ph];
                    im -= double(h[base + j])*sn[ph];
                }
                const double sc = 1.0/double(kConvFft);
                if(bin == 0) dst[0] = float(re*sc);
                else if(bin == kConvBlock) dst[1] = float(re*sc);
                else { dst[bin*2] = float(re*sc); dst[bin*2+1] = float(im*sc); }
            }
        }
    }
    return install_slot(d, slot, [&](SlotRec &r, auto &alloc) -> int {
        r.type = B200MIX_EFFECT_CONVOLUTION; r.channels = ir_channels; r.frames = ir_frames; r.segs = nseg;
        if(int rc = alloc(r.ring, 1)) return rc;
        if(int rc = alloc(r.H, size_t(ir_channels)*nseg*kConvFft)) return rc;
        if(int rc = alloc(r.X, size_t(nseg + kConvMaxBlocks)*kConvFft)) return rc;
        if(int rc = alloc(r.head, size_t(ir_channels)*kConvBlock)) return rc;
        if(int rc = alloc(r.inbuf, kConvFft)) return rc;
        if(int rc = alloc(r.ov, size_t(ir_channels)*kConvFft)) return rc;
        if(int rc = alloc(r.yspec, size_t(ir_channels)*kConvMaxChunks*kConvMaxBlocks*kConvFft)) return rc;
        if(int rc = alloc(r.lines, size_t(ir_channels)*kLine)) return rc;
        if(int rc = alloc(r.gains, size_t(ir_channels)*32)) return rc;
        if(int rc = alloc(r.gtgt, size_t(ir_channels)*32)) return rc;
        CUDA_TRY(d, cudaMemcpyAsync(r.H, H.data(), H.size()*sizeof(float), cudaMemcpyHostToDevice, d->stream));
        CUDA_TRY(d, cudaMemcpyAsync(r.head, head.data(), head.size()*sizeof(float), cudaMemcpyHostToDevice, d->stream));
        return B200MIX_OK;
    });
}

// b200mix_reverb_params -> the parameter part of a ReverbDev (state and pointers untouched)
static void reverb_fill_params(ReverbDev &h, const b200mix_reverb_params *p)
{
    std::memcpy(h.early_tap, p->early_tap, sizeof(h.early_tap)); h.early_tap_coeff = p->early_tap_coeff;
    std::memcpy(h.late_tap, p->late_tap, sizeof(h.late_tap));
    h.mix_x = p->mix_x; h.mix_y = p->mix_y;
    std::memcpy(h.filter_lp, p->filter_lp, sizeof(h.filter_lp));
    std::memcpy(h.filter_hp, p->filter_hp, sizeof(h.filter_hp));
    h.early_ap_coeff = p->early_ap_coeff;
    std::memcpy(h.early_ap_offset, p->early_ap_offset, sizeof(h.early_ap_offset));
    std::memcpy(h.early_offset, p->early_offset, sizeof(h.early_offset));
    h.early_coeff = p->early_coeff;
    std::memcpy(h.late_offset, p->late_offset, sizeof(h.late_offset));
    h.density_gain = p->density_gain;
    std::memcpy(h.t60_mid_gain, p->t60_mid_gain, sizeof(h.t60_mid_gain));
    std::memcpy(h.t60_hf, p->t60_hf, sizeof(h.t60_hf)); std::memcpy(h.t60_lf, p->t60_lf, sizeof(h.t60_lf));
    h.mod_step = p->mod_step; h.mod_depth = p->mod_depth; h.late_ap_coeff = p->late_ap_coeff;
    std::memcpy(h.late_ap_offset, p->late_ap_offset, sizeof(h.late_ap_offset));
    h.upmix = p->upmix ? 1u : 0u; h.order_scale[0] = p->order_scale[0]; h.order_scale[1] = p->order_scale[1];
    h.split_coeff = p->splitter_coeff;
}

static int reverb_check_params(b200mix_device *d, const b200mix_reverb_params *p)
{
    auto pow2 = [](uint32_t v) { return v >= 4u && !(v & (v-1u)); };
    if(!pow2(p->main_len) || !pow2(p->late_in_len) || !pow2(p->early_ap_len) || !pow2(p->early_len)
        || !pow2(p->late_ap_len) || !pow2(p->late_len) || !p->late_offset[0] || !p->late_ap_offset[0])
    { d->error = "slot_reverb: line lengths must be powers of two, feedback delays non-zero"; return B200MIX_ERR_INVALID; }
    for(int j = 0;j < 4;++j)
        if(!p->early_ap_offset[j] || p->late_ap_offset[j] < p->late_ap_offset[0])
        { d->error = "slot_reverb: all-pass delays must be non-zero, late all-pass sorted"; return B200MIX_ERR_INVALID; }
    return B200MIX_OK;
}

// the parameter prefix of ReverbDev (everything before the filter states)
static constexpr size_t kReverbParamBytes = offsetof(ReverbDev, z_lp);

// ReverbPipeline::clear (reverb.cpp:550-566) for one pipeline object on the device: delay lines,
// the object's ReverbDev from the mirror SlotTable::Reverb::clear left, and its output gains.
static int reverb_clear_pipeline(b200mix_device *d, uint32_t slot, int obj)
{
    const SlotRec &S = d->slots[slot].rec;
    const ReverbDev &h = d->slots[slot].rv.h[obj];
    CUDA_TRY(d, cudaMemsetAsync(h.late_in, 0, size_t(4)*h.late_in_len*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemsetAsync(h.early_ap, 0, size_t(4)*h.early_ap_len*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemsetAsync(h.early_d, 0, size_t(4)*h.early_len*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemsetAsync(h.late_ap, 0, size_t(4)*h.late_ap_len*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemsetAsync(h.late_d, 0, size_t(4)*h.late_len*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemcpyAsync(reinterpret_cast<ReverbDev*>(S.H) + obj, &h, sizeof(ReverbDev), cudaMemcpyHostToDevice,
        d->stream));
    CUDA_TRY(d, cudaMemsetAsync(S.gtgt + size_t(obj)*8*32, 0, size_t(8)*32*sizeof(float), d->stream));
    CUDA_TRY(d, cudaMemsetAsync(S.gains + size_t(obj)*8*32, 0, size_t(8)*32*sizeof(float), d->stream));
    // the host mirror was read by a pageable-memory copy above: wait before it changes again
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    return B200MIX_OK;
}

int b200mix_slot_reverb(b200mix_device *d, uint32_t slot, const b200mix_reverb_params *p)
{
    if(!d || slot >= d->slots.size() || !p || p->struct_size != sizeof(*p))
    { if(d) d->error = "slot_reverb: bad arguments (or the device has no sends/slots)"; return B200MIX_ERR_INVALID; }
    if(int rc = reverb_check_params(d, p)) return rc;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    return install_slot(d, slot, [&](SlotRec &r, auto &alloc) -> int {
        SlotTable::Reverb &R = d->slots[slot].rv;
        r.type = B200MIX_EFFECT_REVERB; r.channels = 16;       // 2 pipeline objects x (4 early + 4 late) lines
        float *main_d = nullptr;
        if(int rc = alloc(main_d, size_t(4)*p->main_len)) return rc;
        for(int obj = 0;obj < 2;++obj)
        {
            ReverbDev &h = R.h[obj];
            h.main_len = p->main_len; h.late_in_len = p->late_in_len; h.early_ap_len = p->early_ap_len;
            h.early_len = p->early_len; h.late_ap_len = p->late_ap_len; h.late_len = p->late_len;
            // a pipeline that has not been updated yet is in ReverbPipeline::clear()'s state
            reverb_fill_params(h, p);
            R.clear(obj);
            h.main_d = main_d;
            if(int rc = alloc(h.late_in, size_t(4)*p->late_in_len)) return rc;
            if(int rc = alloc(h.early_ap, size_t(4)*p->early_ap_len)) return rc;
            if(int rc = alloc(h.early_d, size_t(4)*p->early_len)) return rc;
            if(int rc = alloc(h.late_ap, size_t(4)*p->late_ap_len)) return rc;
            if(int rc = alloc(h.late_d, size_t(4)*p->late_len)) return rc;
        }
        // deviceUpdate leaves DeviceClear; the first update is a full one: it switches to pipeline
        // object 1 and goes straight to Normal (reverb.cpp:1243-1280)
        R.cur = 1;
        reverb_fill_params(R.h[1], p);
        R.fade[1] = p->fade_samples; R.fade[0] = 1u;
        ReverbDev *dev = nullptr;
        if(int rc = alloc(dev, 2)) return rc;
        r.H = reinterpret_cast<float*>(dev);
        if(int rc = alloc(r.lines, size_t(16)*kLine)) return rc;
        if(int rc = alloc(r.gains, size_t(16)*32)) return rc;
        if(int rc = alloc(r.gtgt, size_t(16)*32)) return rc;
        CUDA_TRY(d, cudaMemcpyAsync(dev, R.h, 2*sizeof(ReverbDev), cudaMemcpyHostToDevice, d->stream));
        return B200MIX_OK;
    });
}

int b200mix_slot_efx(b200mix_device *d, uint32_t slot, const b200mix_efx_props *props,
    const b200mix_efx_target *target)
{
    if(!d || slot >= d->slots.size() || !props || !target || props->struct_size != sizeof(*props)
        || target->struct_size != sizeof(*target) || props->type < B200MIX_EFFECT_ECHO
        || props->type > B200MIX_EFFECT_PSHIFTER)
    { if(d) d->error = "slot_efx: bad arguments (or the device has no sends/slots)"; return B200MIX_ERR_INVALID; }
    const b200mix_device_desc &dd = d->desc;
    if(target->wet_channels != dd.wet_channels
        || target->out_channels != (d->slots[slot].rec.target != B200MIX_NO_SLOT ? dd.wet_channels : dd.dry_channels))
    { d->error = "slot_efx: the target maps do not match the device's wet / output mix"; return B200MIX_ERR_INVALID; }
    EfxParams P;
    if(int rc = efx_update(*props, *target, P))
    { d->error = rc == B200MIX_ERR_UNSUPPORTED ? "slot_efx: not supported in this configuration (see b200mix.h)"
        : "slot_efx: bad properties / maps"; return rc; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(!d->efx_ready) { CUDA_TRY(d, efx_kernels_init()); d->efx_ready = true; }
    SlotTable::Slot &S = d->slots[slot];
    SlotTable::Efx &H = S.efx;
    const bool fresh = S.rec.type != props->type || H.p.lines != P.lines
        || H.p.echo_len != P.echo_len || H.p.cho_len != P.cho_len;
    if(P.type == B200MIX_EFFECT_AUTOWAH && P.lines > kEfxMaxLines - 2u)
    { d->error = "slot_efx: autowah handles up to 14 wet channels"; return B200MIX_ERR_UNSUPPORTED; }
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    if(fresh)
    {
        // EffectState::deviceUpdate: new state, cleared
        EfxDev h{};
        h.p = P; h.comp_env = 1.0f;
        if(int rc = install_slot(d, slot, [&](SlotRec &r, auto &alloc) -> int {
            r.type = props->type; r.channels = P.lines; r.fade_len = P.fade_len;
            EfxDev *dev = nullptr;
            if(int rc = alloc(dev, 1)) return rc;
            if(int rc = alloc(r.lines, size_t(P.lines)*kLine)) return rc;
            if(int rc = alloc(r.gains, size_t(P.lines)*32)) return rc;
            if(int rc = alloc(r.gtgt, size_t(P.lines)*32)) return rc;
            if(P.echo_len) { if(int rc = alloc(h.echo_buf, P.echo_len)) return rc; }
            if(P.cho_len) { if(int rc = alloc(h.cho_buf, size_t(4)*P.cho_len)) return rc; }
            if(P.type == B200MIX_EFFECT_FSHIFTER)
            {   // FshifterState::deviceUpdate (fshifter.cpp:140-148): cleared FIFOs, mPos = HilSize - HilStep
                if(int rc = alloc(h.fs_in, size_t(4)*1024)) return rc;
                if(int rc = alloc(h.fs_outfifo, size_t(4)*256)) return rc;
                if(int rc = alloc(h.fs_accum, size_t(4)*1024)) return rc;
                h.fs_count = 0u; h.fs_pos = 1024u - 256u;
            }
            if(P.type == B200MIX_EFFECT_PSHIFTER)
            {   // PshifterState::deviceUpdate (pshifter.cpp:131-145): cleared FIFOs and phases, mPos = StftSize - StftStep
                if(int rc = alloc(h.ps_fifo, size_t(9)*1024)) return rc;
                if(int rc = alloc(h.ps_accum, size_t(9)*1024)) return rc;
                if(int rc = alloc(h.ps_last, size_t(513))) return rc;
                if(int rc = alloc(h.ps_sum, size_t(513))) return rc;
                h.ps_count = 0u; h.ps_pos = 1024u - 128u;
            }
            r.H = reinterpret_cast<float*>(dev);
            CUDA_TRY(d, cudaMemcpyAsync(dev, &h, sizeof(h), cudaMemcpyHostToDevice, d->stream));
            H.mod_range = P.mod_range ? P.mod_range : 1u;
            H.lfo_range = P.cho_lfo_range ? P.cho_lfo_range : 1u;
            return B200MIX_OK;
        })) return rc;
    }
    else
    {
        EfxDev *dev = reinterpret_cast<EfxDev*>(S.rec.H);
        // EffectState::update: new parameters, state kept.  The ring modulator rescales its
        // phase index to the new range (modulator.cpp:117-118); the host mirrors the index
        CUDA_TRY(d, cudaMemcpyAsync(&dev->p, &P, sizeof(EfxParams), cudaMemcpyHostToDevice, d->stream));
        if(props->type == B200MIX_EFFECT_MODULATOR)
        {
            H.mod_index = uint32_t(uint64_t(H.mod_index) * P.mod_range_new / H.mod_range);
            H.mod_range = P.mod_range;
            CUDA_TRY(d, cudaMemcpyAsync(&dev->mod_index, &H.mod_index, sizeof(uint32_t), cudaMemcpyHostToDevice, d->stream));
        }
        if(props->type == B200MIX_EFFECT_CHORUS)
        {
            // mLfoOffset follows the LFO range (chorus.cpp:185-211)
            H.lfo_offset = P.cho_rate_on ? H.lfo_offset * P.cho_lfo_range_new / H.lfo_range : 0u;
            H.lfo_range = P.cho_lfo_range;
            CUDA_TRY(d, cudaMemcpyAsync(&dev->cho_lfo_offset, &H.lfo_offset, sizeof(uint32_t), cudaMemcpyHostToDevice,
                d->stream));
        }
        if(props->type == B200MIX_EFFECT_FSHIFTER)
        {   // a direction switched off zeroes that side's phase accumulators (fshifter.cpp:189-192,205-208)
            static const uint32_t zero = 0u;
            for(int c = 0;c < 4;++c)
                if(P.fs_reset_phase[c])
                    CUDA_TRY(d, cudaMemcpyAsync(&dev->fs_phase[c], &zero, sizeof(uint32_t), cudaMemcpyHostToDevice, d->stream));
        }
        if(props->type == B200MIX_EFFECT_VMORPHER)
            // update() installs newly constructed formant filters: their histories restart at 0
            // (vmorpher.cpp:252-260)
            CUDA_TRY(d, cudaMemsetAsync(dev->vm_s, 0, sizeof(EfxDev::vm_s), d->stream));
        S.rec.fade_len = P.fade_len;
        if(int rc = refresh_slots(d)) return rc;
    }
    H.p = P;
    CUDA_TRY(d, cudaMemcpyAsync(S.rec.gtgt, P.gains, size_t(P.lines)*32*sizeof(float), cudaMemcpyHostToDevice, d->stream));
    if(P.snap_gains)
        CUDA_TRY(d, cudaMemcpyAsync(S.rec.gains, P.gains, size_t(P.lines)*32*sizeof(float), cudaMemcpyHostToDevice,
            d->stream));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    return B200MIX_OK;
}

int b200mix_slot_target(b200mix_device *d, uint32_t slot, uint32_t target)
{
    if(!d || slot >= d->slots.size() || (target != B200MIX_NO_SLOT && target >= d->slots.size()))
    { if(d) d->error = "slot_target: slot out of range"; return B200MIX_ERR_INVALID; }
    uint32_t hops = 0;
    for(uint32_t t = target;t != B200MIX_NO_SLOT;t = d->slots[t].rec.target)
        if(t == slot || ++hops > d->slots.size())
        { d->error = "slot_target: the chain would loop"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    d->slots[slot].rec.target = target;
    return refresh_slots(d);
}

int b200mix_slot_reverb_update(b200mix_device *d, uint32_t slot, const b200mix_reverb_params *p,
    uint32_t full_update)
{
    if(!d || slot >= d->slots.size() || !p || p->struct_size != sizeof(*p)
        || d->slots[slot].rec.type != B200MIX_EFFECT_REVERB)
    { if(d) d->error = "slot_reverb_update: no reverb installed on this slot / bad arguments"; return B200MIX_ERR_INVALID; }
    if(int rc = reverb_check_params(d, p)) return rc;
    SlotTable::Reverb &R = d->slots[slot].rv;
    ReverbDev *dev = reinterpret_cast<ReverbDev*>(d->slots[slot].rec.H);
    const ReverbDev &h0 = R.h[0];
    if(p->main_len != h0.main_len || p->late_in_len != h0.late_in_len || p->early_ap_len != h0.early_ap_len
        || p->early_len != h0.early_len || p->late_ap_len != h0.late_ap_len || p->late_len != h0.late_len)
    { d->error = "slot_reverb_update: line lengths differ from the installed ones"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));      // host mirrors are about to change
    if(full_update)
    {
        // reverb.cpp:1275-1279
        R.state = SlotTable::Pipeline::Fading;
        R.cur ^= 1;
        const int old = R.cur ^ 1;
        R.h[old].early_tap_coeff = 0.0f;
        CUDA_TRY(d, cudaMemcpyAsync(&dev[old].early_tap_coeff, &R.h[old].early_tap_coeff, sizeof(float),
            cudaMemcpyHostToDevice, d->stream));
        // the object coming back into use has not advanced mOffset while it was idle
        R.h[R.cur].offset = R.offset;
        CUDA_TRY(d, cudaMemcpyAsync(&dev[R.cur].offset, &R.h[R.cur].offset, sizeof(uint32_t), cudaMemcpyHostToDevice,
            d->stream));
    }
    reverb_fill_params(R.h[R.cur], p);
    R.fade[R.cur] = p->fade_samples;
    CUDA_TRY(d, cudaMemcpyAsync(dev + R.cur, &R.h[R.cur], kReverbParamBytes, cudaMemcpyHostToDevice, d->stream));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    d->slots.refresh();                                 // the up-mix flag follows the parameters
    return B200MIX_OK;
}

int b200mix_slot_output_gains(b200mix_device *d, uint32_t slot, uint32_t lines, const float *gains)
{
    if(!d || slot >= d->slots.size() || !d->slots[slot].rec.type || !gains)
    { if(d) d->error = "slot_output_gains: bad arguments"; return B200MIX_ERR_INVALID; }
    const SlotTable::Slot &S = d->slots[slot];
    const bool reverb = S.rec.type == B200MIX_EFFECT_REVERB;
    if(lines != (reverb ? 8u : S.rec.channels))
    { d->error = "slot_output_gains: wrong line count"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    // gains address the slot's output target: the Dry mix or the target slot's Wet mix
    const uint32_t width = d->slots[slot].rec.target != B200MIX_NO_SLOT ? d->desc.wet_channels : d->desc.dry_channels;
    std::vector<float> g(size_t(lines)*32, 0.0f);
    for(uint32_t c = 0;c < lines;++c)
        for(uint32_t o = 0;o < width;++o)
            g[c*32 + o] = gains[c*width + o];
    // a reverb's gains are those of its CURRENT pipeline object (update3DPanning, reverb.cpp:1293-1296)
    float *dst = S.rec.gtgt + (reverb ? size_t(S.rv.cur)*8*32 : 0);
    CUDA_TRY(d, cudaMemcpyAsync(dst, g.data(), g.size()*sizeof(float), cudaMemcpyHostToDevice, d->stream));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    return B200MIX_OK;
}

int b200mix_hrtf_attach(b200mix_device *d, const b200mix_hrtf *h)
{
    if(!d || !h) return B200MIX_ERR_INVALID;
    if(h->ir_size > d->desc.ir_size)
    { d->error = "hrtf_attach: data set HRIRs are longer than the device's ir_size"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    d->d_st_fields.reset(); d->d_st_elevs.reset(); d->d_st_coeffs.reset(); d->d_st_delays.reset();
    std::vector<float2> fields(h->fields.size());
    for(size_t i = 0;i < fields.size();++i)
    {
        uint32_t ev = h->fields[i].ev_count; float evf;
        std::memcpy(&evf, &ev, sizeof(evf));
        fields[i] = make_float2(h->fields[i].distance, evf);
    }
    std::vector<uint2> elevs(h->elevs.size());
    for(size_t i = 0;i < elevs.size();++i) elevs[i] = make_uint2(h->elevs[i].az_count, h->elevs[i].ir_offset);
    CUDA_TRY(d, d->d_st_fields.alloc(fields.size()));
    CUDA_TRY(d, d->d_st_elevs.alloc(elevs.size()));
    CUDA_TRY(d, d->d_st_coeffs.alloc(h->coeffs.size()/2));
    CUDA_TRY(d, d->d_st_delays.alloc(h->delays.size()));
    CUDA_TRY(d, cudaMemcpy(d->d_st_fields, fields.data(), fields.size()*sizeof(float2), cudaMemcpyHostToDevice));
    CUDA_TRY(d, cudaMemcpy(d->d_st_elevs, elevs.data(), elevs.size()*sizeof(uint2), cudaMemcpyHostToDevice));
    CUDA_TRY(d, cudaMemcpy(d->d_st_coeffs, h->coeffs.data(), h->coeffs.size()*sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(d, cudaMemcpy(d->d_st_delays, h->delays.data(), h->delays.size(), cudaMemcpyHostToDevice));
    d->st_num_fields = uint32_t(fields.size()); d->st_ir = h->ir_size;
    return B200MIX_OK;
}

static int voices_update_impl(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *hrtf_coeffs, const float *dirs, const float *dry_gains, const float *send_gains,
    bool direct);

// The voices of each callback buffer are the channels of one source: cb_reps[slot] = the first one
// that mixes this update (-1: none), cb_members[slot] the others, which must agree with it on what
// the planner reads.  One pass over the voices.
static int cb_group(b200mix_device *d)
{
    std::vector<int32_t> &reps = d->cb_reps;
    reps.assign(d->cbs.size(), -1);
    d->cb_members.resize(d->cbs.size());
    for(auto &m : d->cb_members) m.clear();
    for(uint32_t v = 0;v < d->book.voice_hi;++v)
    {
        const b200mix_device::CbVoice &cv = d->cbv[v];
        if(cv.slot < 0 || (cv.v.state != 1u && cv.v.state != 2u)) continue;
        int32_t &r = reps[size_t(cv.slot)];
        if(r < 0) { r = int32_t(v); continue; }
        const cbplan::Voice &a = d->cbv[size_t(r)].v, &b = cv.v;
        if(a.pos != b.pos || a.frac != b.frac || a.step != b.step || a.state != b.state
            || a.have_buffer != b.have_buffer)
        {
            d->error = "voices_update: voices sharing a callback buffer disagree on step, position or state";
            return B200MIX_ERR_INVALID;
        }
        d->cb_members[size_t(cv.slot)].push_back(v);
    }
    return B200MIX_OK;
}

int b200mix_voices_update(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *hrtf_coeffs, const float *dry_gains, const float *send_gains)
{
    return voices_update_impl(d, n, params, hrtf_coeffs, nullptr, dry_gains, send_gains, false);
}

int b200mix_voices_update_dirs(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *dirs, const float *dry_gains, const float *send_gains)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(!dirs) { d->error = "voices_update_dirs: null directions"; return B200MIX_ERR_INVALID; }
    if(!d->d_st_coeffs) { d->error = "voices_update_dirs: no HRTF data set attached"; return B200MIX_ERR_INVALID; }
    return voices_update_impl(d, n, params, nullptr, dirs, dry_gains, send_gains, false);
}

int b200mix_voices_update_direct(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *real_gains, const float *send_gains)
{
    if(!d) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    // where the reference's RealOut.RemixMap is empty (UHJ / TSME) or RealOut is Dry, it never
    // mixes direct channels (CalcPanningAndFilters, alc/alu.cpp:1535-1599)
    if(dd.post_process != B200MIX_POST_HRTF && dd.post_process != B200MIX_POST_AMBIDEC)
    { d->error = "voices_update_direct: the device's output takes no direct channels"; return B200MIX_ERR_UNSUPPORTED; }
    if(d->shard.world > 1u)
    { d->error = "voices_update_direct: not on a sharded device set"; return B200MIX_ERR_UNSUPPORTED; }
    if(d->out.has_stabilizer())
    { d->error = "voices_update_direct: not with a front stabilizer"; return B200MIX_ERR_UNSUPPORTED; }
    return voices_update_impl(d, n, params, nullptr, nullptr, real_gains, send_gains, true);
}

// `direct`: b200mix_voices_update_direct, whose `dry_gains` are RealOut gains.
static int voices_update_impl(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *hrtf_coeffs, const float *dirs, const float *dry_gains, const float *send_gains,
    bool direct)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(n == 0) return B200MIX_OK;
    if(!params) { d->error = "voices_update: null params"; return B200MIX_ERR_INVALID; }
    const b200mix_device_desc &dd = d->desc;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    for(uint32_t i = 0;i < n;++i)
    {
        const b200mix_voice_params &p = params[i];
        if(direct && (p.flags & (B200MIX_VF_DIRECT | B200MIX_VF_HRTF)) != B200MIX_VF_DIRECT)
        { d->error = "voices_update_direct: every entry has B200MIX_VF_DIRECT and not B200MIX_VF_HRTF"; return B200MIX_ERR_INVALID; }
        if(int rc = check_entry(d, "voices_update", p, true, direct || (p.flags & B200MIX_VF_HRTF) != 0)) return rc;
        // MaxPitch clamp of the parameter stage (alc/alu.cpp:1682-1685,1996-1999): CalculateBufferSize
        // relies on it
        if(p.step > (10u << 16))
        { d->error = "voices_update: step above MaxPitch<<16"; return B200MIX_ERR_INVALID; }
        // with directions the delays are computed on the device
        if(!dirs && (p.hrtf_delay[0] >= B200MIX_HRTF_HISTORY || p.hrtf_delay[1] >= B200MIX_HRTF_HISTORY))
        { d->error = "voices_update: HRTF delay out of range"; return B200MIX_ERR_INVALID; }
        // callback voice: plays a buffer made by b200mix_buffer_callback
        const int32_t cbSlot = cb_slot_of(d, p.flags, p.buffer);
        if(cbSlot >= 0 && (p.flags & B200MIX_VF_STATIC))
        { d->error = "voices_update: a callback buffer is not static (IsCallback)"; return B200MIX_ERR_INVALID; }
        if(cbSlot >= 0 && d->cbv[p.voice].slot != cbSlot && !(p.flags & B200MIX_VF_RESET))
        { d->error = "voices_update: a voice starts a callback buffer with B200MIX_VF_RESET"; return B200MIX_ERR_INVALID; }
    }

    if(direct)
        if(int rc = ensure_real_bus(d)) return rc;
    CUDA_TRY(d, d->stage.wait());
    if(int rc = ensure_stage(d, n)) return rc;
    d->stage.begin();
    VoiceUpdate *const upd = d->stage.host_part<VoiceUpdate>(n);
    for(uint32_t i = 0;i < n;++i)
    {
        const b200mix_voice_params &p = params[i];
        const bool nobuf = p.buffer == B200MIX_NO_BUFFER;
        const bool stopped = (p.flags & B200MIX_VF_STOPPED) != 0;
        VoiceUpdate &u = upd[i];
        u.voice = p.voice; u.flags = (p.flags & ~kVfDirect) | (direct ? kVfDirect : 0u);
        u.buffer = p.buffer; u.resampler = p.resampler;
        if(nobuf) { u.flags |= kUpNoBuffer; u.buffer = 0u; }
        u.position = p.position; u.position_frac = p.position_frac;
        u.loop_start = p.loop_start; u.loop_end = p.loop_end; u.step = p.step;
        u.bsinc_sf = 0.0f; u.bsinc_m = 0; u.bsinc_l = 0; u.bsinc_off = 0;
        if(const BsincTable *t = bsinc_for(d, p.resampler))
        {
            const BsincState st = PrepareBsinc(*t, p.step);
            u.bsinc_sf = st.sf; u.bsinc_m = st.m; u.bsinc_l = st.l; u.bsinc_off = st.offset;
        }
        u.delay0 = dirs ? 0 : p.hrtf_delay[0]; u.delay1 = dirs ? 0 : p.hrtf_delay[1]; u.gain = p.hrtf_gain;
        for(uint32_t s = 0;s < B200MIX_MAX_SENDS;++s)
            u.send_slot[s] = (s < dd.num_sends) ? p.send_slot[s] : B200MIX_NO_SLOT;
        u.has_coeffs = (hrtf_coeffs != nullptr || (dirs != nullptr && (p.flags & B200MIX_VF_HRTF))) && dd.ir_size > 0;
        u.has_dry = dry_gains != nullptr && !direct;
        // mixing-order cost key: resampler taps per output
        const uint32_t cost = (p.step == 65536u) ? 1u : (u.bsinc_m ? u.bsinc_m : (p.resampler >= 2u ? 4u : 2u));
        d->book.set(p.voice, {!stopped, cost, (p.flags & B200MIX_VF_HRTF) != 0, p.send_slot,
            (p.flags & B200MIX_VF_STATIC) && !nobuf ? p.buffer : B200MIX_NO_SLOT, (p.flags & B200MIX_VF_RESET) != 0,
            direct});
        if(!d->cbv.empty())
        {
            // the planner's mirror of the voice: what k_apply_updates does to its record
            b200mix_device::CbVoice &cv = d->cbv[p.voice];
            const int32_t slot = nobuf && !stopped ? cv.slot : cb_slot_of(d, p.flags, p.buffer);
            if(slot != cv.slot)
            {
                d->cb_bound = d->cb_bound + (slot >= 0) - (cv.slot >= 0);
                cv.slot = slot;
            }
            if(slot >= 0)
            {
                cbplan::Voice &m = cv.v;
                if(p.flags & B200MIX_VF_RESET)
                {
                    m.pos = p.position; m.frac = p.position_frac; m.have_buffer = true;
                    d->cbs[size_t(slot)].st = cbplan::State{};
                }
                if(p.flags & B200MIX_VF_STOPPING) m.state = 2u;
                else if(p.flags & B200MIX_VF_PLAYING) m.state = 1u;
                m.step = p.step;
                if(nobuf) m.have_buffer = false;
            }
        }
    }
    if(d->cb_bound)
        if(int rc = cb_group(d)) return rc;
    ApplyParams A = apply_params(d, d->stage.dev_of(upd));
    auto pack = [d](const float *src, size_t count) { return d->stage.pack(src, count); };
    if(dirs && dd.ir_size)
        apply_dirs(d, A, reinterpret_cast<const float4*>(pack(dirs, size_t(n)*4)));
    else if(hrtf_coeffs && dd.ir_size)
        A.coeffs = pack(hrtf_coeffs, size_t(n)*dd.ir_size*2);
    if(direct && dry_gains && dd.real_channels)
        A.real = pack(dry_gains, size_t(n)*dd.real_channels);
    else if(!direct && dry_gains && dd.dry_channels)
        A.dry = pack(dry_gains, size_t(n)*dd.dry_channels);
    if(send_gains && dd.num_sends && dd.wet_channels)
        A.send = pack(send_gains, size_t(n)*dd.num_sends*dd.wet_channels);
    CUDA_TRY(d, d->stage.ship(d->stream));
    k_apply_updates<<<n, 64, 0, d->stream>>>(A);
    ++d->launches;
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

// Could any path of this source need a filter?  (All of these leave GainHF == GainLF == 1 exactly
// when false, alc/alu.cpp:1854-1961 — a cheap scan so that scenes without filters never allocate
// or run the filter stage.)
static bool source_may_filter(const b200mix_source_props &P, uint32_t num_sends)
{
    if(P.direct.gain_hf != 1.0f || P.direct.gain_lf != 1.0f || P.air_absorption_factor != 0.0f) return true;
    if(P.inner_angle < 360.0f && (P.outer_gain_hf != 1.0f)) return true;
    for(uint32_t s = 0;s < num_sends;++s)
        if(P.sends[s].gain_hf != 1.0f || P.sends[s].gain_lf != 1.0f
            || (P.sends[s].active && P.sends[s].slot_air_absorption_gain_hf < 1.0f)) return true;
    return false;
}

int b200mix_sources_update(b200mix_device *d, uint32_t n, const b200mix_source_voice *voices,
    const b200mix_source_props *props, const b200mix_listener_params *listener, const b200mix_voice_env *env)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(n == 0) return B200MIX_OK;
    const b200mix_device_desc &dd = d->desc;
    if(!voices || !props || !listener || !env || env->struct_size != sizeof(*env)
        || listener->struct_size != sizeof(*listener) || env->render_mode > 2u
        || env->num_sends != dd.num_sends || !env->device_rate || listener->distance_model > 6u)
    { d->error = "sources_update: bad arguments (env->num_sends must equal the device's)"; return B200MIX_ERR_INVALID; }
    if(env->render_mode == 2u && (!dd.ir_size || !d->d_st_coeffs))
    { d->error = "sources_update: HRTF rendering needs an HRTF device and b200mix_hrtf_attach"; return B200MIX_ERR_INVALID; }
    if(env->render_mode != 2u && (env->dry.channels != dd.dry_channels || !env->dry.scale || !env->dry.index))
    { d->error = "sources_update: env->dry must describe the device's Dry mix"; return B200MIX_ERR_INVALID; }
    if(dd.num_sends && (env->wet_stride != dd.wet_channels))
    { d->error = "sources_update: env->wet_stride must equal the device's wet_channels"; return B200MIX_ERR_INVALID; }
    for(uint32_t s = 0;s < dd.num_sends;++s)
        if(env->wet[s].channels > dd.wet_channels || (env->wet[s].channels && (!env->wet[s].scale || !env->wet[s].index)))
        { d->error = "sources_update: bad wet map"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));

    bool mayFilter = d->d_filt != nullptr;
    const bool hrtfMode = env->render_mode == 2u;
    for(uint32_t i = 0;i < n;++i)
    {
        const b200mix_source_voice &p = voices[i];
        const b200mix_source_props &P = props[i];
        if(P.struct_size != sizeof(P) || P.distance_model > 6u)
        { d->error = "sources_update: bad source props"; return B200MIX_ERR_INVALID; }
        if(int rc = check_entry(d, "sources_update", p, false, hrtfMode)) return rc;
        // callback voices are planned from the steps b200mix_voices_update gives; this stage
        // computes them on the device, where the planner cannot see them
        if(cb_slot_of(d, p.flags, p.buffer) >= 0)
        { d->error = "sources_update: callback buffers play through b200mix_voices_update"; return B200MIX_ERR_UNSUPPORTED; }
        if(!mayFilter && source_may_filter(P, dd.num_sends)) mayFilter = true;
    }
    if(mayFilter)
        if(int rc = ensure_filters(d)) return rc;
    // staging: [voices n][props n] in, [VoiceUpdate n][dirs n][dry][send][hf/lf][FilterUpdate] scratch
    const uint32_t paths = 1u + dd.num_sends;
    CUDA_TRY(d, d->src.wait());
    {
        const uint32_t cap = std::max<uint32_t>(n, 2u*uint32_t(d->src.capacity()));
        const size_t in = align16(size_t(cap)*sizeof(b200mix_source_voice)) + align16(size_t(cap)*sizeof(b200mix_source_props));
        const size_t out = align16(size_t(cap)*sizeof(VoiceUpdate)) + align16(size_t(cap)*16)
            + align16(size_t(cap)*std::max(dd.dry_channels, 1u)*4) + align16(size_t(cap)*std::max(dd.num_sends*dd.wet_channels, 1u)*4)
            + align16(size_t(cap)*(1u + B200MIX_MAX_SENDS)*8) + align16(size_t(cap)*paths*sizeof(FilterUpdate));
        CUDA_TRY(d, d->src.reserve(n, cap, in, in + out + 64, d->stream));
    }

    if(mayFilter) d->book.set_device_filters();
    for(uint32_t i = 0;i < n;++i)
    {
        const b200mix_source_voice &p = voices[i];
        const bool act = !(p.flags & B200MIX_VF_STOPPED);
        // the voice no longer plays a callback buffer
        if(!d->cbv.empty() && d->cbv[p.voice].slot >= 0)
        {
            d->cbv[p.voice].slot = -1;
            --d->cb_bound;
        }
        // the step is not known here: the cost key takes the resampler's widest filter, and is
        // kept while the voice stays active
        const BsincTable *t = bsinc_for(d, p.resampler);
        uint32_t cost = d->book.cost[p.voice];
        if(bool(d->book.active[p.voice]) != act || (!cost && act)) cost = t ? t->m[0] : (p.resampler >= 2u ? 4u : 2u);
        d->book.set(p.voice, {act, cost, hrtfMode, p.send_slot,
            (p.flags & B200MIX_VF_STATIC) ? p.buffer : B200MIX_NO_SLOT, (p.flags & B200MIX_VF_RESET) != 0, false});
    }
    UploadArena &U = d->src;
    U.begin();
    CalcVoicesParams Q{};
    Q.voices = U.pack(voices, n);
    Q.props = U.pack(props, n);
    CUDA_TRY(d, U.ship(d->stream));
    Q.n = n; Q.listener = *listener;
    Q.device_rate = env->device_rate; Q.num_sends = dd.num_sends; Q.render_mode = env->render_mode;
    Q.cd = dd.dry_channels; Q.cw = dd.wet_channels; Q.ir = dd.ir_size;
    if(!hrtfMode)
    {
        Q.dry_channels = env->dry.channels;
        for(uint32_t c = 0;c < env->dry.channels;++c) { Q.dry_scale[c] = env->dry.scale[c]; Q.dry_index[c] = env->dry.index[c]; }
    }
    for(uint32_t s = 0;s < dd.num_sends;++s)
    {
        Q.wet_channels[s] = env->wet[s].channels;
        for(uint32_t c = 0;c < env->wet[s].channels;++c) { Q.wet_scale[s][c] = env->wet[s].scale[c]; Q.wet_index[s][c] = env->wet[s].index[c]; }
    }
    for(int t = 0;t < 3;++t)
    {
        Q.bsinc[t].scaleBase = d->bsinc[t].scaleBase; Q.bsinc[t].scaleRange = d->bsinc[t].scaleRange;
        for(unsigned k = 0;k < kBsincScales;++k) { Q.bsinc[t].m[k] = d->bsinc[t].m[k]; Q.bsinc[t].filterOffset[k] = d->bsinc[t].filterOffset[k]; }
    }
    Q.updates = U.carve<VoiceUpdate>(n);
    Q.dirs = U.carve<float4>(n);
    Q.dry = U.carve<float>(size_t(n)*std::max(dd.dry_channels, 1u));
    Q.send = (dd.num_sends && dd.wet_channels) ? U.carve<float>(size_t(n)*dd.num_sends*dd.wet_channels) : nullptr;
    Q.gains_hflf = U.carve<float>(size_t(n)*(1u + B200MIX_MAX_SENDS)*2);
    Q.fupd = U.carve<FilterUpdate>(size_t(n)*paths);
    const bool filters = d->d_filt != nullptr;
    CUDA_TRY(d, launch_calc_voices(Q, filters, d->stream));
    d->launches += filters ? 2 : 1;

    ApplyParams A = apply_params(d, Q.updates);
    if(hrtfMode) apply_dirs(d, A, Q.dirs);
    else A.dry = Q.dry;
    A.send = Q.send;
    k_apply_updates<<<n, 64, 0, d->stream>>>(A);
    ++d->launches;
    if(filters)
    {
        k_apply_filter_updates<<<(2u*n*paths + 127u)/128u, 128, 0, d->stream>>>(d->d_filt, paths, Q.fupd, n*paths);
        ++d->launches;
    }
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

int b200mix_get_voice_targets(b200mix_device *d, uint32_t voice, uint32_t *step, float bsinc[4],
    float *hrtf_gain, uint32_t hrtf_delay[2], float *hrtf_coeffs, float *dry_gains, float *send_gains,
    float *filters)
{
    if(!d || voice >= d->desc.max_voices) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    VoiceRec rec;
    CUDA_TRY(d, cudaMemcpy(&rec, d->d_voices + voice, offsetof(VoiceRec, prev), cudaMemcpyDeviceToHost));
    if(step) *step = rec.step;
    if(bsinc)
    {
        bsinc[0] = rec.bsinc_sf;
        std::memcpy(&bsinc[1], &rec.bsinc_m, 4); std::memcpy(&bsinc[2], &rec.bsinc_l, 4);
        std::memcpy(&bsinc[3], &rec.bsinc_off, 4);
    }
    if(hrtf_gain) *hrtf_gain = rec.tgt_gain;
    if(hrtf_delay) { hrtf_delay[0] = rec.tgt_delay0; hrtf_delay[1] = rec.tgt_delay1; }
    if(hrtf_coeffs && d->d_hrtf_tgt)
        CUDA_TRY(d, cudaMemcpy(hrtf_coeffs, d->d_hrtf_tgt + size_t(voice)*d->ir_pad, size_t(dd.ir_size)*8, cudaMemcpyDeviceToHost));
    if(dry_gains && dd.dry_channels)
        CUDA_TRY(d, cudaMemcpy(dry_gains, d->d_dry_tgt + size_t(voice)*dd.dry_channels, size_t(dd.dry_channels)*4, cudaMemcpyDeviceToHost));
    if(send_gains && d->d_send_tgt)
        CUDA_TRY(d, cudaMemcpy(send_gains, d->d_send_tgt + size_t(voice)*dd.num_sends*dd.wet_channels,
            size_t(dd.num_sends)*dd.wet_channels*4, cudaMemcpyDeviceToHost));
    if(filters)
    {
        const uint32_t paths = 1u + dd.num_sends;
        for(uint32_t pth = 0;pth < paths;++pth)
        {
            float *o = filters + size_t(pth)*11;
            for(int k = 0;k < 11;++k) o[k] = k == 1 ? 1.0f : (k == 6 ? 1.0f : 0.0f);
            if(!d->d_filt) continue;
            FilterRec fr;
            CUDA_TRY(d, cudaMemcpy(&fr, d->d_filt + size_t(voice)*paths + pth, sizeof(fr), cudaMemcpyDeviceToHost));
            o[0] = fr.active ? 1.0f : 0.0f;
            for(int k = 0;k < 5;++k) { o[1+k] = fr.tgt[0][k]; o[6+k] = fr.tgt[1][k]; }
        }
    }
    return B200MIX_OK;
}

int b200mix_voice_queue(b200mix_device *d, uint32_t voice, uint32_t count, const uint32_t *buffers,
    uint32_t loop_index)
{
    if(!d) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    if(voice >= dd.max_voices || (count && !buffers))
    { d->error = "voice_queue: bad arguments"; return B200MIX_ERR_INVALID; }
    if(count > B200MIX_MAX_QUEUE)
    { d->error = "voice_queue: more than B200MIX_MAX_QUEUE items"; return B200MIX_ERR_UNSUPPORTED; }
    if(loop_index != B200MIX_NO_LOOP && loop_index >= count)
    { d->error = "voice_queue: loop index outside the list"; return B200MIX_ERR_INVALID; }
    QueueSet Q{};
    Q.voice = voice; Q.count = count; Q.loop = loop_index;
    for(uint32_t i = 0;i < count;++i)
    {
        if(buffers[i] >= dd.max_buffers || !d->h_buffers[buffers[i]].data || d->h_buffers[buffers[i]].pad)
        { d->error = "voice_queue: buffer id without data"; return B200MIX_ERR_INVALID; }
        Q.items[i] = buffers[i];
    }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(int rc = ensure_queues(d)) return rc;
    k_set_queue<<<1, 32, 0, d->stream>>>(d->d_voices, d->d_qhdr, d->d_queue, Q);
    ++d->launches;
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

// Filter state of every voice path (allocated by the first filter a host or the GPU parameter
// stage sets; a device that never sees one pays nothing).
static int ensure_filters(b200mix_device *d)
{
    if(d->d_filt) return B200MIX_OK;
    const b200mix_device_desc &dd = d->desc;
    const uint32_t paths = 1u + dd.num_sends;
    const size_t count = size_t(dd.max_voices)*paths;
    if(int rc = ensure_park_lines(d)) return rc;
    DevArray<FilterRec> filt; DevArray<float> dline; DevArray<uint32_t> order2;
    CUDA_TRY(d, filt.alloc(count));
    CUDA_TRY(d, dline.alloc(size_t(dd.max_voices)*kLine, d->stream));
    CUDA_TRY(d, order2.alloc(dd.max_voices, d->stream));
    k_filter_init<<<unsigned((count*32u + 255u)/256u), 256, 0, d->stream>>>(filt, count);
    CUDA_TRY(d, cudaGetLastError());
    ++d->launches;
    d->d_filt = std::move(filt); d->d_dline = std::move(dline); d->d_order2 = std::move(order2);
    return B200MIX_OK;
}

int b200mix_voices_filters(b200mix_device *d, uint32_t n, const b200mix_voice_filter *filters)
{
    static_assert(sizeof(FilterUpdate) == sizeof(b200mix_voice_filter), "FilterUpdate mirrors the ABI struct");
    if(!d) return B200MIX_ERR_INVALID;
    if(n == 0) return B200MIX_OK;
    if(!filters) { d->error = "voices_filters: null filters"; return B200MIX_ERR_INVALID; }
    const b200mix_device_desc &dd = d->desc;
    const uint32_t paths = 1u + dd.num_sends;
    for(uint32_t i = 0;i < n;++i)
        if(filters[i].voice >= dd.max_voices || filters[i].path >= paths)
        { d->error = "voices_filters: voice/path out of range"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(int rc = ensure_filters(d)) return rc;
    for(uint32_t i = 0;i < n;++i)
        if(filters[i].path == 0) d->book.set_direct_filter(filters[i].voice, filters[i].active != 0);
    UploadArena &U = d->fstage;
    CUDA_TRY(d, U.wait());
    const size_t cap = std::max<size_t>(n, 2u*U.capacity());
    CUDA_TRY(d, U.reserve(n, cap, cap*sizeof(FilterUpdate), cap*sizeof(FilterUpdate), d->stream));
    U.begin();
    const FilterUpdate *fupd = U.pack(reinterpret_cast<const FilterUpdate*>(filters), n);
    CUDA_TRY(d, U.ship(d->stream));
    k_apply_filter_updates<<<(2u*n + 127u)/128u, 128, 0, d->stream>>>(d->d_filt, paths, fupd, n);
    ++d->launches;
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

// One bus mix of parked lines, the parked dry bus (one pseudo slot) or the aux sends (`slots`
// slots): the entries' gain ramps -> k_send_mix in M.chunks entry chunks, with samples
// 128..1023 on the tensor cores when `tc` -> the chunks' partial rows summed into M.wet ->
// the Current gains advanced.
static int run_bus_mix(b200mix_device *d, const SendMixParams &M, uint32_t num_entries, uint32_t slots,
    bool tc)
{
    const uint32_t chunks = M.chunks;
    if(num_entries)
    {
        const uint32_t tot = num_entries*M.cw;
        k_send_gains_prepare<<<(tot + 127)/128, 128, 0, d->stream>>>(M, num_entries);
        ++d->launches;
    }
    const uint32_t tiles = tc ? 1u : (chunks > 1u ? uint32_t(kLine/128) : (M.frames + 127u)/128u);
    if(M.cw > 4u) k_send_mix<16><<<dim3(slots, tiles, chunks), 256, 0, d->stream>>>(M);
    else k_send_mix<4><<<dim3(slots, tiles, chunks), 256, 0, d->stream>>>(M);
    ++d->launches;
    if(tc)
    {
        // dline stays null until a direct filter is set: no sendinfo lookups per entry before then
        PanMixTcParams TQ{M.slot_start, M.entries, M.sendinfo, M.xscratch, d->d_dline, M.geff, M.cw, chunks,
            M.partial};
        k_panmix_tc<<<chunks, 128, kPmStages*kPmStageBytes + 1024, d->stream>>>(TQ);
        ++d->launches;
    }
    if(chunks > 1u)
    {
        const uint32_t len = slots*M.cw*kLine;
        if(chunks <= 16u)
            k_reduce_few<<<(len/4 + 255)/256, 256, 0, d->stream>>>(M.partial, chunks, len, M.wet, 1);
        else
            k_reduce_rows<<<(len/4 + kReduceCols - 1)/kReduceCols, 1024, 0, d->stream>>>(
                M.partial, chunks, len, M.wet, 1);
        ++d->launches;
    }
    if(num_entries)
    {
        const uint32_t tot = num_entries*M.cw;
        k_send_gains_update<<<(tot + 127)/128, 128, 0, d->stream>>>(M, num_entries);
        ++d->launches;
    }
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

static inline void stage_mark(b200mix_device *d, int i)
{ if(d->profile_level >= 2) cudaEventRecord(d->ev_stage[i], d->stream); }

// The callback buffers' part of an update (callback_plan.hpp).  First every callback buffer's
// callbacks run on this thread; then, straight into the pinned arena, each buffer's plan record and
// the blocks it has stored (ADPCM decoded to int16) are packed, its storage is compacted as the
// reference does after the mix, and its voices' mirror advances; table and samples go to the GPU
// with one copy on the mixer stream.  *plan stays null when no callback voice mixes this update.
static int cb_plan_update(b200mix_device *d, uint32_t frames, const BufferRec *&plan)
{
    plan = nullptr;
    if(int rc = cb_group(d)) { d->error = "render: " + d->error; return rc; }
    const std::vector<int32_t> &reps = d->cb_reps;
    bool any = false;
    for(int32_t r : reps) any = any || r >= 0;
    if(!any) return B200MIX_OK;
    d->cb_work.resize(d->cbs.size());
    // 1. the callbacks.  Registration guarantees the reference's storage size, which no request of
    //    its chunk loop passes: plan_loads cannot stop half way through the buffers.
    size_t size = align16(d->cbs.size()*sizeof(BufferRec));
    for(size_t s = 0;s < d->cbs.size();++s)
    {
        if(reps[s] < 0) continue;
        b200mix_device::CbBuf &c = d->cbs[s];
        b200mix_device::CbWork &w = d->cb_work[s];
        const b200mix_callback_buffer &cb = c.cb;
        auto request = [&cb](uint64_t offset, uint32_t bytes) -> int64_t {
            return cb.callback(cb.userptr, static_cast<char*>(cb.storage) + offset, int(bytes));
        };
        w.start = c.st;
        if(!cbplan::plan_loads(c.st, cb.samples_per_block, cb.bytes_per_block, d->cbv[size_t(reps[s])].v,
            frames, cb.storage_bytes, request, w.loads))
        { d->error = "render: a callback request passes the callback buffer's storage"; return B200MIX_ERR_INVALID; }
        // [pad | the stored blocks as the kernel reads them | pad], a pad holding one frame and
        // 16 bytes: a load held at the last stored sample may address the frame before the first
        // (none stored) or the first (empty span); the bulk copies round their runs up to 16 bytes
        const size_t pad = align16(c.frame_bytes) + 16u;
        w.bytes = w.loads.chunks ? size_t(c.st.num_blocks)*cb.samples_per_block*c.frame_bytes : 0u;
        w.region = size + pad;
        size = w.region + align16(w.bytes) + pad;
    }
    // 2. the arena (two alternate: the other one's copy may still be in flight)
    UploadArena &U = d->cb_arena[d->cb_idx];
    CUDA_TRY(d, U.wait());
    CUDA_TRY(d, U.reserve(size, size*2, size*2, size*2, d->stream));
    U.begin();
    uint8_t *arena = U.host_part<uint8_t>(size);
    const uintptr_t devArena = reinterpret_cast<uintptr_t>(U.dev_of(arena));
    // 3. pack, then what the reference does after the mix
    std::memset(arena, 0, size);
    for(size_t s = 0;s < d->cbs.size();++s)
    {
        if(reps[s] < 0) continue;
        b200mix_device::CbBuf &c = d->cbs[s];
        const b200mix_device::CbWork &w = d->cb_work[s];
        const b200mix_callback_buffer &cb = c.cb;
        cbplan::Voice &vm = d->cbv[size_t(reps[s])].v;
        const cbplan::Span span = cbplan::span_of(w.start, vm, cb.samples_per_block, c.st);
        BufferRec rec = d->h_buffers[c.buffer];
        rec.data = reinterpret_cast<const void*>(devArena
            + uintptr_t(int64_t(w.region) + span.base*int64_t(c.frame_bytes)));
        rec.frames = w.loads.chunks ? span.frames : 0u;
        std::memcpy(arena + s*sizeof(BufferRec), &rec, sizeof(rec));
        uint8_t *dst = arena + w.region;
        const uint8_t *src = static_cast<const uint8_t*>(cb.storage);
        if(!w.bytes) {}
        else if(cb.sample_type == B200MIX_FMT_IMA4)
            DecodeIMA4(src, cb.channels, cb.samples_per_block, c.st.num_blocks, reinterpret_cast<int16_t*>(dst));
        else if(cb.sample_type == B200MIX_FMT_MSADPCM)
            DecodeMSADPCM(src, cb.channels, cb.samples_per_block, c.st.num_blocks, reinterpret_cast<int16_t*>(dst));
        else
            std::memcpy(dst, src, w.bytes);
        const cbplan::After after = cbplan::finish_update(c.st, cb.samples_per_block, cb.bytes_per_block,
            vm, frames);
        if(after.consumed_bytes)
            std::memmove(cb.storage, static_cast<char*>(cb.storage) + after.consumed_bytes, after.kept_bytes);
        // the source's other channel voices move with it
        for(uint32_t v : d->cb_members[s]) d->cbv[v].v = vm;
    }
    CUDA_TRY(d, U.ship(d->stream));
    d->cb_idx ^= 1;
    plan = reinterpret_cast<const BufferRec*>(devArena);
    return B200MIX_OK;
}

// Phase A of an update: clear the mix buffers, mix every voice, reduce the partial rows and
// finish the aux sends -> the slots' Wet buffers are complete (alc/alu.cpp:2196-2206).
static int render_phase_a(b200mix_device *d, uint32_t frames, bool want_results, bool force_sends)
{
    const b200mix_device_desc &dd = d->desc;
    if(frames < 1 || frames > B200MIX_LINE_SIZE)
    { d->error = "render: frames out of range"; return B200MIX_ERR_INVALID; }
    if(const char *why = d->out.missing()) { d->error = std::string("render: ") + why; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    // callback buffers: their callbacks run here, before anything of the update is launched
    const BufferRec *cbplan = nullptr;
    if(d->cb_bound)
        if(int rc = cb_plan_update(d, frames, cbplan)) return rc;

    VoiceBook &B = d->book;
    const VoiceBook::Rebuilt re = B.refresh(d->d_filt != nullptr, d->mix_cdr == 0 && d->d_dry_entries,
        (d->slots.active || force_sends) && d->d_wet && d->d_slot_start);
    d->real_mixed = !B.real_entries.empty();

    stage_mark(d, 0);
    // clear MixBuffer (alc/alu.cpp:2417) and the wet buffers (alc/alu.cpp:2196-2198)
    // (the dry mix is left alone while nothing can write or read it: HRTF-only scenes; an
    // HRTF post-process whose RealOut is just L/R overwrites it instead of accumulating, unless
    // the RealOut bus has mixed direct-channel voices into it)
    if(d->book.dry_active || dd.post_process != B200MIX_POST_HRTF)
        CUDA_TRY(d, cudaMemsetAsync(d->d_dry, 0, size_t(d->dry_alloc_ch)*kLine*sizeof(float), d->stream));
    if(d->d_real != d->d_dry && (!d->out.overwrites_real() || d->real_mixed))
        CUDA_TRY(d, cudaMemsetAsync(d->d_real, 0, size_t(dd.real_channels)*kLine*sizeof(float), d->stream));
    if(d->d_wet)
        CUDA_TRY(d, cudaMemsetAsync(d->d_wet, 0, size_t(dd.max_slots)*dd.wet_channels*kLine*sizeof(float), d->stream));

    if(re.order)
        if(int rc = upload(d, d->d_order, B.order)) return rc;
    if(re.order2)
        if(int rc = upload(d, d->d_order2, B.order2)) return rc;
    if(re.dry)
    {
        const uint32_t ss[2] = {0u, uint32_t(B.dry_entries.size())};
        CUDA_TRY(d, cudaMemcpyAsync(d->d_dry_slot_start, ss, sizeof(ss), cudaMemcpyHostToDevice, d->stream));
        if(int rc = upload(d, d->d_dry_entries, B.dry_entries)) return rc;
    }
    if(re.sends)
    {
        if(int rc = upload(d, d->d_slot_start, B.slot_start)) return rc;
        if(int rc = upload(d, d->d_entries, B.entries)) return rc;
    }
    if(re.real && d->d_real_entries)
    {
        const uint32_t ss[2] = {0u, uint32_t(B.real_entries.size())};
        CUDA_TRY(d, cudaMemcpyAsync(d->d_real_slot_start, ss, sizeof(ss), cudaMemcpyHostToDevice, d->stream));
        if(int rc = upload(d, d->d_real_entries, B.real_entries)) return rc;
    }
    const uint32_t numOrder = uint32_t(B.order.size()), numOrder2 = uint32_t(B.order2.size());
    const uint32_t numDry = uint32_t(B.dry_entries.size()), numEntries = uint32_t(B.entries.size());
    const bool hrtfDev = dd.ir_size > 0;
    const uint32_t nv = std::max(B.voice_hi, 1u);
    const uint32_t maxBlocks = uint32_t(d->num_sms*d->mix_blocks_per_sm);
    const uint32_t blocks = std::max(1u, std::min(maxBlocks, (numOrder + kMixGroups - 1)/kMixGroups));

    MixParams P{};
    P.voices = d->d_voices; P.buffers = d->d_buffers;
    P.hrtf_tgt = d->d_hrtf_tgt; P.hrtf_old = d->d_hrtf_old;
    P.dry_cur = d->d_dry_cur; P.dry_tgt = d->d_dry_tgt;
    P.partial = d->d_partial;
    P.results = want_results ? d->d_results : nullptr;
    for(int i = 0;i < 3;++i) P.bsinc_tab[i] = d->d_bsinc[i];
    for(int i = 0;i < 2;++i) P.cubic_tab[i] = d->d_cubic[i];
    P.max_voices = nv; P.frames = frames; P.ir_pad = d->ir_pad;
    P.cd = dd.dry_channels; P.num_sends = dd.num_sends;
    P.order = d->d_order; P.num_order = numOrder;
    P.xscratch = d->d_xscratch; P.sendinfo = d->d_sendinfo;
    P.filt = d->d_filt; P.filt_paths = 1u + dd.num_sends;
    P.qhdr = d->d_qhdr; P.queue = d->d_queue;
    P.claim = d->d_claim;
    P.dline = d->d_dline;
    P.cbplan = cbplan;
    // the voice loop: resample (and park) -> direct filters -> deferred dry pass or HRIR FIR
    stage_mark(d, 1);
    if(d->profile) cudaEventRecord(d->ev_mix0, d->stream);
    d->mix_fn<<<blocks, kMixGS*kMixGroups, d->mix_smem, d->stream>>>(P);
    ++d->launches;
    CUDA_TRY(d, cudaGetLastError());
    const uint64_t mixDone = d->launches;

    stage_mark(d, 2);
    // ---- voices with an active direct filter: filter the parked lines, then mix them ----
    size_t rows2 = 0;
    if(d->d_filt && numOrder2)
    {
        FilterRunParams FP{};
        FP.filt = d->d_filt; FP.filt_paths = 1u + dd.num_sends; FP.sendinfo = d->d_sendinfo;
        FP.direct_order = d->d_order2; FP.num_direct = numOrder2;
        FP.xscratch = d->d_xscratch; FP.dline = d->d_dline; FP.frames = frames;
        k_filters<<<(numOrder2 + 31u)/32u, 32, 0, d->stream>>>(FP);
        ++d->launches;
        if(d->mix_cdr > 0)
        {
            // The grid is the number of partial rows, so it fixes the order in which the
            // deferred voices' sums are added: it follows the resample kernel's occupancy, as
            // the main pass's does, not this kernel's own.
            const uint32_t blocks2 = std::max(1u, std::min(maxBlocks, (numOrder2 + kMixGroups - 1)/kMixGroups));
            rows2 = blocks2;
            MixParams P2 = P;
            P2.order = d->d_order2; P2.num_order = numOrder2;
            P2.partial = d->d_partial + d->partial_floats;
            P2.results = nullptr;
            k_mix_deferred<kMixGS, kMixGroups, 4><<<blocks2, kMixGS*kMixGroups,
                sizeof(DeferredSmem<kMixGroups, 4>), d->stream>>>(P2);
            ++d->launches;
        }
        CUDA_TRY(d, cudaGetLastError());
    }
    // the HRIR FIR's partial rows are summed by the HRTF post-process (OutputStage::post)
    d->fir_rows = 0;
    if(hrtfDev)
    {
        const FirVariant fir = get_fir(dd.ir_size);
        d->fir_rows = std::max(1u, std::min(uint32_t(d->num_sms*d->fir_blocks_per_sm),
            (numOrder + kFirGroups - 1)/kFirGroups));
        // straight behind the resample kernel (no direct filters in between), its set-up runs
        // under the resample kernel's last CTAs
        CUDA_TRY(d, launch_ex(d->stream, d->launches, d->launches == mixDone, fir.fn, dim3(d->fir_rows),
            dim3(kFirGS*kFirGroups), fir.smem, P));
        d->fir_done = d->launches;
    }
    if(d->profile) { cudaEventRecord(d->ev_mix1, d->stream); d->ev_valid = true; }

    stage_mark(d, 3);
    if(d->mix_cdr > 0)
    {
        const uint32_t len = uint32_t(d->mix_cdr)*kLine;
        k_reduce_rows<<<(len/4 + kReduceCols - 1)/kReduceCols, 1024, 0, d->stream>>>(d->d_partial, blocks, len, d->d_dry, 1);
        ++d->launches;
        if(rows2)
        {
            k_reduce_rows<<<(len/4 + kReduceCols - 1)/kReduceCols, 1024, 0, d->stream>>>(d->d_partial + d->partial_floats,
                uint32_t(rows2), len, d->d_dry, 1);
            ++d->launches;
        }
    }
    CUDA_TRY(d, cudaGetLastError());

    stage_mark(d, 4);
    // ---- parked dry bus: non-HRTF voices of a variant without register accumulators ----
    if(d->mix_cdr == 0 && d->d_dry_entries)
    {
        if(numDry)
        {
            SendMixParams DM{};
            DM.slot_start = d->d_dry_slot_start; DM.entries = d->d_dry_entries; DM.sendinfo = d->d_sendinfo;
            DM.xscratch = d->d_xscratch; DM.send_cur = d->d_dry_cur; DM.send_tgt = d->d_dry_tgt;
            DM.wet = d->d_dry; DM.frames = frames; DM.cw = dd.dry_channels; DM.num_sends = 1;
            DM.valid_bit = kSiDry; DM.dline = d->d_dline ? d->d_dline : d->d_xscratch;
            // a CTA's 8 warps share its entries evenly: chunks of 64 entries keep the first
            // (fading) tile's serial work per warp short
            const uint32_t chunks = std::max(1u, std::min(kDryChunksMax, (numDry + 63u)/64u));
            DM.chunks = chunks; DM.partial = d->d_dry_partial; DM.geff = d->d_dry_geff; DM.gramp = d->d_dry_gramp;
            // Above 4 dry channels (third-order output) a full update's pan-mix past the gain fades
            // is a dense GEMM over the voices: samples 128..1023 go to the tensor cores
            // (k_panmix_tc), k_send_mix keeps the first tile with the fades
            const bool tc = d->panmix_tc && dd.dry_channels > 4u && dd.dry_channels <= uint32_t(kPmN)
                && frames == uint32_t(kLine) && chunks > 1u;
            if(int rc = run_bus_mix(d, DM, numDry, 1u, tc)) return rc;
        }
    }

    // ---- RealOut bus: direct-channel voices (core/voice.cpp:947-963 with mDirect.Buffer = RealOut)
    // in index order, one pseudo slot of real_channels; RealOut is then (direct sum) + the
    // post-process' output, the reference's association ----
    if(d->real_mixed)
    {
        SendMixParams RM{};
        RM.slot_start = d->d_real_slot_start; RM.entries = d->d_real_entries; RM.sendinfo = d->d_sendinfo;
        RM.xscratch = d->d_xscratch; RM.send_cur = d->d_real_cur; RM.send_tgt = d->d_real_tgt;
        RM.wet = d->d_real; RM.frames = frames; RM.cw = dd.real_channels; RM.num_sends = 1;
        RM.valid_bit = kSiReal; RM.dline = d->d_dline ? d->d_dline : d->d_xscratch;
        RM.chunks = 1; RM.geff = d->d_real_geff; RM.gramp = d->d_real_gramp;
        if(int rc = run_bus_mix(d, RM, uint32_t(B.real_entries.size()), 1u, false)) return rc;
    }

    stage_mark(d, 5);
    // ---- aux sends (core/voice.cpp:967-980) ----
    if((d->slots.active || force_sends) && d->d_wet && d->d_slot_start)
    {
        SendMixParams SM{};
        SM.slot_start = d->d_slot_start; SM.entries = d->d_entries; SM.sendinfo = d->d_sendinfo;
        SM.xscratch = d->d_xscratch; SM.send_cur = d->d_send_cur; SM.send_tgt = d->d_send_tgt;
        SM.wet = d->d_wet; SM.frames = frames; SM.cw = dd.wet_channels; SM.num_sends = dd.num_sends;
        SM.valid_bit = kSiSend;
        if(d->d_filt && numEntries)
        {
            if(d->d_fscratch.size() < size_t(numEntries)*kLine)
            {
                CUDA_TRY(d, regrow(d->d_fscratch, size_t(std::max(numEntries, 64u))*kLine, d->stream));
                CUDA_TRY(d, cudaMemsetAsync(d->d_fscratch, 0, d->d_fscratch.bytes(), d->stream));
            }
            SM.filt = d->d_filt; SM.filt_paths = 1u + dd.num_sends; SM.fscratch = d->d_fscratch;
            FilterRunParams FP{};
            FP.filt = d->d_filt; FP.filt_paths = 1u + dd.num_sends; FP.sendinfo = d->d_sendinfo;
            FP.entries = d->d_entries; FP.num_entries = numEntries;
            FP.xscratch = d->d_xscratch; FP.fscratch = d->d_fscratch; FP.frames = frames;
            k_filters<<<(numEntries + 31u)/32u, 32, 0, d->stream>>>(FP);
            ++d->launches;
        }
        SM.geff = d->d_send_geff; SM.gramp = d->d_send_gramp;
        // a CTA's 8 warps share its entries evenly: chunks of 128 entries per slot
        const uint32_t chunks = std::max(1u, std::min(16u, (B.max_slot_entries + 127u)/128u));
        const size_t partialFloats = size_t(chunks)*dd.max_slots*dd.wet_channels*kLine;
        if(chunks > 1u && d->d_send_partial.size() < partialFloats)
            CUDA_TRY(d, regrow(d->d_send_partial, partialFloats, d->stream));
        SM.chunks = chunks; SM.partial = d->d_send_partial;
        if(int rc = run_bus_mix(d, SM, numEntries, dd.max_slots, false)) return rc;
    }
    return B200MIX_OK;
}

// Phase B: run the effect slots on their Wet input, mix their output into Dry, post-process
// (alc/alu.cpp:2252-2256, 2439-2443).
static int render_phase_b(b200mix_device *d, uint32_t frames)
{
    const b200mix_device_desc &dd = d->desc;
    stage_mark(d, 6);
    SlotTable &T = d->slots;
    if(T.active)
    {
        bool upload = false;
        for(uint32_t sl = 0;sl < T.size();++sl)
        {
            const SlotTable::Due due = T.advance(sl, frames);
            if(due.clear >= 0)
                if(int rc = reverb_clear_pipeline(d, sl, due.clear)) return rc;
            if(due.silence >= 0)
                CUDA_TRY(d, cudaMemsetAsync(T[sl].rec.gtgt + size_t(due.silence)*8*32, 0, size_t(8)*32*sizeof(float),
                    d->stream));
            upload |= due.upload;
        }
        if(upload)
            if(int rc = refresh_slots(d)) return rc;
        ConvParams CP{};
        CP.slots = d->d_slots; CP.wet = d->d_wet; CP.twiddle = d->d_twiddle;
        CP.frames = frames; CP.cw = dd.wet_channels; CP.num_slots = dd.max_slots; CP.chunks = T.conv_chunks;
        SlotMixParams SP{};
        SP.slots = d->d_slots; SP.dry = d->d_dry; SP.frames = frames; SP.cd = dd.dry_channels;
        SP.num_slots = dd.max_slots; SP.wet = d->d_wet; SP.cw = dd.wet_channels;
        // one pass per stage of the slot graph (a single pass unless slots target other slots)
        for(uint32_t st = 0;st < T.stages;++st)
        {
            if(T.reverb)
            {
                ReverbParamsK RP{};
                RP.slots = d->d_slots; RP.wet = d->d_wet; RP.cubic = d->d_cubic_filter;
                RP.frames = frames; RP.cw = dd.wet_channels; RP.stage = st;
                RP.seq = ++d->reverb_seq;
                k_reverb_process<<<dim3(dd.max_slots, 2, 2), 128, 0, d->stream>>>(RP);
                k_reverb_commit<<<dd.max_slots, 2, 0, d->stream>>>(RP);
                d->launches += 2;
                if(T.upmix)
                {
                    k_reverb_upmix<<<dim3(dd.max_slots, 2), 256, 8*kLine*sizeof(float), d->stream>>>(RP);
                    ++d->launches;
                }
            }
            CP.stage = st; SP.stage = st;
            if(T.efx)
            {
                EfxRunParams EQ{d->d_slots, d->d_wet, frames, dd.wet_channels, st, d->d_cubic_filter};
                CUDA_TRY(d, launch_efx_process(EQ, dd.max_slots, d->stream));
                ++d->launches;
                if(T.pshift)
                {
                    CUDA_TRY(d, launch_efx_pshift(EQ, dd.max_slots, d->stream));
                    ++d->launches;
                }
            }
            if(T.conv)
            {
                k_conv_input<<<dd.max_slots, 128, 0, d->stream>>>(CP);
                k_conv_mac<<<dim3(dd.max_slots, T.conv_ch, CP.chunks), 128, sizeof(ConvMacSmem), d->stream>>>(CP);
                k_conv_ifft<<<dim3(dd.max_slots, T.conv_ch, kConvMaxBlocks), 128, 0, d->stream>>>(CP);
                k_conv_output<<<dim3(dd.max_slots, T.conv_ch), 128, 0, d->stream>>>(CP);
                d->launches += 4;
            }
            k_slot_output_mix<<<dim3((frames + 127)/128, dd.dry_channels), 128, 0, d->stream>>>(SP);
            ++d->launches;
            if(T.targets)
            {
                k_slot_target_mix<<<dim3((frames + 127)/128, dd.max_slots), 128, 0, d->stream>>>(SP);
                ++d->launches;
            }
        }
        k_slot_gains_commit<<<dd.max_slots, 64, 0, d->stream>>>(SP);
        ++d->launches;
        CUDA_TRY(d, cudaGetLastError());
    }

    stage_mark(d, 7);
    if(int rc = d->out.post(d->d_dry, d->d_real, d->d_partial, d->fir_rows, d->book.dry_active, d->real_mixed,
        d->fir_done, frames, d->launches)) return rc;
    stage_mark(d, 8);
    if(d->profile_level >= 2) d->stage_valid = true;
    CUDA_TRY(d, cudaGetLastError());
    return B200MIX_OK;
}

// ---- voice-sharded device sets: the two exchanges of an update (SURVEY §8e) -------------
// Wet reduce-scatter: every owner ends up with the summed send input of its slots.
static int shard_wet_exchange(b200mix_device *d)
{
    b200mix_device::Shard &S = d->shard;
    const b200mix_device_desc &dd = d->desc;
    if(!S.transport || !d->d_wet) return B200MIX_OK;
    if(d->profile) { cudaEventRecord(S.ev[0], d->stream); }
    const size_t wetFloats = size_t(dd.max_slots)*dd.wet_channels*kLine;
    if(S.transport == 2)
    {
        if(S.allreduce(d->d_wet, d->d_wet, wetFloats, 7 /*ncclFloat*/, 0 /*ncclSum*/, S.comm, d->stream) != 0)
        { d->error = "ncclAllReduce of the wet buffers failed"; return B200MIX_ERR_CUDA; }
        d->fir_done = 0;            // a kernel that `launches` does not count
    }
    else
    {
        const uint32_t slotFloats = dd.wet_channels*uint32_t(kLine);
        ShardPushParams P{};
        P.src = d->d_wet; P.rank = S.rank; P.world = S.world; P.epoch = S.epoch;
        P.wet = 1u; P.num_slots = dd.max_slots; P.slot_floats = slotFloats; P.owned_max = S.owned_max;
        P.own = reinterpret_cast<ShardCtl*>(S.own.get());
        for(uint32_t r = 0;r < S.world;++r) P.peer[r] = S.peer[r];
        P.off_data = S.off_wet; P.per_src_floats = S.wet_src_floats;
        P.counters = S.d_counters + 4;
        const uint32_t chunks = std::max(1u, std::min(32u, slotFloats*S.owned_max/(4u*256u*4u)));
        k_shard_push<<<dim3(chunks, S.world), 256, 0, d->stream>>>(P);
        ShardSumParams Q{};
        Q.dst = d->d_wet; Q.rank = S.rank; Q.world = S.world; Q.epoch = S.epoch;
        Q.wet = 1u; Q.num_slots = dd.max_slots; Q.slot_floats = slotFloats; Q.owned_max = S.owned_max;
        Q.own = P.own; for(uint32_t r = 0;r < S.world;++r) Q.peer[r] = S.peer[r];
        Q.off_data = S.off_wet; Q.per_src_floats = S.wet_src_floats; Q.counter = S.d_counters + 2;
        k_shard_sum<<<std::max(1u, std::min(64u, slotFloats*S.owned_max/(4u*256u*2u))), 256, 0, d->stream>>>(Q);
        d->launches += 2;
        CUDA_TRY(d, cudaGetLastError());
    }
    if(d->profile) { cudaEventRecord(S.ev[1], d->stream); S.ev_wet = true; }
    return B200MIX_OK;
}

// RealOut reduce onto rank 0.
static int shard_real_reduce(b200mix_device *d)
{
    b200mix_device::Shard &S = d->shard;
    const b200mix_device_desc &dd = d->desc;
    if(!S.transport) return B200MIX_OK;
    if(d->profile) { cudaEventRecord(S.ev[2], d->stream); }
    const uint32_t floats = dd.real_channels*uint32_t(kLine);
    if(S.transport == 2)
    {
        if(S.reduce(d->d_real, d->d_real, floats, 7, 0, 0, S.comm, d->stream) != 0)
        { d->error = "ncclReduce of RealOut failed"; return B200MIX_ERR_CUDA; }
    }
    else if(S.rank != 0u)
    {
        ShardPushParams P{};
        P.src = d->d_real; P.rank = S.rank; P.world = S.world; P.epoch = S.epoch; P.floats = floats;
        P.own = reinterpret_cast<ShardCtl*>(S.own.get());
        for(uint32_t r = 0;r < S.world;++r) P.peer[r] = S.peer[r];
        P.off_data = S.off_real; P.per_src_floats = S.real_floats; P.counters = S.d_counters;
        k_shard_push<<<dim3(std::max(1u, floats/(4u*256u*2u)), 1), 256, 0, d->stream>>>(P);
        ++d->launches;
    }
    else
    {
        ShardSumParams Q{};
        Q.dst = d->d_real; Q.rank = 0u; Q.world = S.world; Q.epoch = S.epoch; Q.floats = floats;
        Q.own = reinterpret_cast<ShardCtl*>(S.own.get());
        for(uint32_t r = 0;r < S.world;++r) Q.peer[r] = S.peer[r];
        Q.off_data = S.off_real; Q.per_src_floats = S.real_floats; Q.counter = S.d_counters + 1;
        k_shard_sum<<<std::max(1u, floats/(4u*256u*2u)), 256, 0, d->stream>>>(Q);
        ++d->launches;
    }
    CUDA_TRY(d, cudaGetLastError());
    if(d->profile) { cudaEventRecord(S.ev[3], d->stream); S.ev_real = true; }
    return B200MIX_OK;
}

// The limiter and distance compensation, after a sharded set's RealOut reduce on its root only (alc/alu.cpp:2446-2450).
static int render_finish(b200mix_device *d, uint32_t frames)
{
    return d->shard.transport && d->shard.rank != 0u ? B200MIX_OK : d->out.finish(d->d_real, frames, d->launches);
}

static int render_launch(b200mix_device *d, uint32_t frames, bool want_results)
{
    if(d->mid_render) { d->error = "render: a render_begin is pending"; return B200MIX_ERR_INVALID; }
    const bool sharded = d->shard.transport != 0;
    if(sharded) ++d->shard.epoch;
    // a sharded set always finishes its sends: another rank may own the slots they feed
    if(int rc = render_phase_a(d, frames, want_results, sharded)) return rc;
    if(sharded) if(int rc = shard_wet_exchange(d)) return rc;
    if(int rc = render_phase_b(d, frames)) return rc;
    if(sharded) if(int rc = shard_real_reduce(d)) return rc;
    return render_finish(d, frames);
}

static int render_collect(b200mix_device *d, uint32_t frames, float *const *real_out,
    b200mix_voice_result *results)
{
    const b200mix_device_desc &dd = d->desc;
    const uint32_t nv = std::max(d->book.voice_hi, 1u);
    const bool contiguous = d->d_real == reinterpret_cast<float*>(d->d_outblock.get());
    if(real_out && results && contiguous)
        CUDA_TRY(d, cudaMemcpyAsync(d->h_outblock, d->d_outblock, d->out_real_bytes + size_t(nv)*sizeof(VoiceResult),
            cudaMemcpyDeviceToHost, d->stream));
    else
    {
        if(real_out)
            CUDA_TRY(d, cudaMemcpyAsync(d->h_real, d->d_real, size_t(dd.real_channels)*kLine*sizeof(float),
                cudaMemcpyDeviceToHost, d->stream));
        if(results)
            CUDA_TRY(d, cudaMemcpyAsync(d->h_results, d->d_results, size_t(nv)*sizeof(VoiceResult),
                cudaMemcpyDeviceToHost, d->stream));
    }
    if(d->shard.transport == 1)
        CUDA_TRY(d, cudaMemcpyAsync(d->shard.h_status, d->shard.own + offsetof(ShardCtl, status),
            sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    if(d->shard.transport == 1 && *d->shard.h_status)
    { d->error = "render: a peer of the sharded device set did not answer in time"; return B200MIX_ERR_CUDA; }
    if(real_out)
        for(uint32_t c = 0;c < dd.real_channels;++c)
            if(real_out[c]) std::memcpy(real_out[c], d->h_real + size_t(c)*kLine, frames*sizeof(float));
    if(results)
    {
        std::memcpy(results, d->h_results, size_t(nv)*sizeof(b200mix_voice_result));
        for(uint32_t v = nv;v < dd.max_voices;++v)
            results[v] = b200mix_voice_result{0, 0u, B200MIX_VF_STOPPED, 0u};
    }
    return B200MIX_OK;
}

int b200mix_render(b200mix_device *d, uint32_t frames, float *const *real_out,
    b200mix_voice_result *results)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(int rc = render_launch(d, frames, results != nullptr)) return rc;
    return render_collect(d, frames, real_out, results);
}

int b200mix_set_uhj_encoder(b200mix_device *d, uint32_t filter_length, uint32_t *delay)
{
    return set_output(d, "set_uhj_encoder", &OutputStage::set_uhj_encoder, filter_length, delay);
}

int b200mix_set_front_stabilizer(b200mix_device *d, uint32_t center_channel, float splitter_coeff)
{
    if(d && center_channel != B200MIX_NO_SLOT && d->book.has_direct())
    { d->error = "set_front_stabilizer: not with active direct-channel voices"; return B200MIX_ERR_UNSUPPORTED; }
    return set_output(d, "set_front_stabilizer", &OutputStage::set_front_stabilizer, center_channel, splitter_coeff);
}

int b200mix_set_bs2b(b200mix_device *d, uint32_t level)
{
    return set_output(d, "set_bs2b", &OutputStage::set_bs2b, level);
}

int b200mix_set_distance_comp(b200mix_device *d, uint32_t channels, const uint32_t *delays, const float *gains)
{
    return set_output(d, "set_distance_comp", &OutputStage::set_distance_comp, channels, delays, gains);
}

int b200mix_set_limiter(b200mix_device *d, const b200mix_limiter_desc *p, uint32_t *look_ahead)
{
    if(d && look_ahead) *look_ahead = 0;
    return set_output(d, "set_limiter", &OutputStage::set_limiter, p, look_ahead);
}

int b200mix_render_interleaved(b200mix_device *d, uint32_t frames, void *out, uint32_t out_type,
    uint32_t frame_step, float dither_depth, uint32_t *dither_seed, b200mix_voice_result *results)
{
    if(!d) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    if(!out || out_type > B200MIX_OUT_F32 || frame_step < dd.real_channels || frame_step > 64u
        || (dither_depth > 0.0f && !dither_seed))
    { d->error = "render_interleaved: bad arguments"; return B200MIX_ERR_INVALID; }
    if(int rc = render_launch(d, frames, results != nullptr)) return rc;
    if(int rc = d->out.interleave(d->d_real, frames, frame_step, out_type, dither_depth,
        dither_seed ? *dither_seed : 0u, d->launches)) return rc;
    if(int rc = render_collect(d, frames, nullptr, results)) return rc;     // synchronises the stream
    d->out.copy_interleaved(out);
    if(dither_depth > 0.0f) *dither_seed = lcg_skip(*dither_seed, uint64_t(2)*dd.real_channels*frames);
    return B200MIX_OK;
}

int b200mix_render_begin(b200mix_device *d, uint32_t frames, float **wet_dev, size_t *wet_floats)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(d->mid_render) { d->error = "render_begin: already begun"; return B200MIX_ERR_INVALID; }
    if(d->shard.transport)
    { d->error = "render_begin: a sharded device set exchanges its wet buffers itself — use b200mix_render"; return B200MIX_ERR_INVALID; }
    if(int rc = render_phase_a(d, frames, true, true)) return rc;
    d->mid_render = true; d->mid_frames = frames;
    d->fir_done = 0;                // the caller may use the stream before render_end
    if(wet_dev) *wet_dev = d->d_wet;
    if(wet_floats) *wet_floats = d->d_wet ? size_t(d->desc.max_slots)*d->desc.wet_channels*kLine : 0;
    return B200MIX_OK;
}

int b200mix_render_end(b200mix_device *d, float *const *real_out, b200mix_voice_result *results,
    const float **real_out_dev)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(!d->mid_render) { d->error = "render_end: no render_begin pending"; return B200MIX_ERR_INVALID; }
    d->mid_render = false;
    if(int rc = render_phase_b(d, d->mid_frames)) return rc;
    if(int rc = render_finish(d, d->mid_frames)) return rc;
    if(real_out_dev) *real_out_dev = d->d_real;
    if(!real_out && !results) return B200MIX_OK;
    return render_collect(d, d->mid_frames, real_out, results);
}

int b200mix_render_device(b200mix_device *d, uint32_t frames, const float **real_out_dev)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(int rc = render_launch(d, frames, false)) return rc;
    if(real_out_dev) *real_out_dev = d->d_real;
    return B200MIX_OK;
}

// ---- voice-sharded device sets ---------------------------------------------------------
static void shard_release(b200mix_device *d)
{
    b200mix_device::Shard &S = d->shard;
    if(S.transport == 1)
        for(uint32_t r = 0;r < S.world;++r)
            if(r != S.rank && S.peer[r]) cudaIpcCloseMemHandle(S.peer[r]);
    if(S.comm && S.comm_destroy) S.comm_destroy(S.comm);
    if(S.nccl_lib) dlclose(S.nccl_lib);
    S = b200mix_device::Shard{};
}

static int shard_common(b200mix_device *d, uint32_t rank, uint32_t world)
{
    if(world < 1u || world > kShardMaxWorld || rank >= world)
    { d->error = "shard: rank/world out of range (world <= 16)"; return B200MIX_ERR_INVALID; }
    if(d->mid_render) { d->error = "shard: a render_begin is pending"; return B200MIX_ERR_INVALID; }
    // a sharded set has no RealOut bus (b200mix_voices_update_direct refuses it)
    if(world > 1u && d->book.has_direct())
    { d->error = "shard: not with active direct-channel voices"; return B200MIX_ERR_UNSUPPORTED; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    shard_release(d);
    d->shard.rank = rank; d->shard.world = world;
    for(Event &e : d->shard.ev) CUDA_TRY(d, e.create());
    return B200MIX_OK;
}

int b200mix_shard_init(b200mix_device *d, uint32_t rank, uint32_t world, void *handle_out)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(!handle_out) { d->error = "shard_init: null handle"; return B200MIX_ERR_INVALID; }
    static_assert(sizeof(cudaIpcMemHandle_t) == B200MIX_SHARD_HANDLE_BYTES, "IPC handle size");
    if(int rc = shard_common(d, rank, world)) return rc;
    b200mix_device::Shard &S = d->shard;
    const b200mix_device_desc &dd = d->desc;
    S.real_floats = size_t(std::max(dd.real_channels, 1u))*kLine;
    S.owned_max = dd.max_slots ? (dd.max_slots + world - 1u)/world : 0u;
    S.wet_src_floats = size_t(S.owned_max)*dd.wet_channels*kLine;
    S.off_real = sizeof(ShardCtl);
    S.off_wet = S.off_real + size_t(2)*world*S.real_floats*sizeof(float);
    CUDA_TRY(d, S.own.alloc(S.off_wet + size_t(2)*world*S.wet_src_floats*sizeof(float)));
    CUDA_TRY(d, cudaMemset(S.own, 0, S.own.bytes()));
    CUDA_TRY(d, S.d_counters.alloc(4 + kShardMaxWorld, d->stream));
    CUDA_TRY(d, S.h_status.alloc(1));
    *S.h_status = 0u;
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    cudaIpcMemHandle_t h;
    CUDA_TRY(d, cudaIpcGetMemHandle(&h, S.own));
    std::memcpy(handle_out, &h, sizeof(h));
    return B200MIX_OK;
}

int b200mix_shard_connect(b200mix_device *d, const void *handles)
{
    if(!d) return B200MIX_ERR_INVALID;
    b200mix_device::Shard &S = d->shard;
    if(!handles || !S.own || S.transport)
    { d->error = "shard_connect: call b200mix_shard_init first (once)"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    for(uint32_t r = 0;r < S.world;++r)
    {
        if(r == S.rank) { S.peer[r] = S.own.get(); continue; }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, static_cast<const char*>(handles) + size_t(r)*sizeof(h), sizeof(h));
        void *p = nullptr;
        CUDA_TRY(d, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        S.peer[r] = static_cast<char*>(p);
    }
    S.transport = 1; S.epoch = 0;
    return B200MIX_OK;
}

namespace { struct NcclId { char internal[128]; }; }

static void *nccl_open(std::string &err)
{
    void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if(!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if(!lib) err = std::string("NCCL not found: ") + dlerror();
    return lib;
}

int b200mix_shard_nccl_id(void *id_out)
{
    if(!id_out) return B200MIX_ERR_INVALID;
    std::string err;
    void *lib = nccl_open(err);
    if(!lib) { g_create_error = err; return B200MIX_ERR_UNSUPPORTED; }
    auto get = reinterpret_cast<int(*)(NcclId*)>(dlsym(lib, "ncclGetUniqueId"));
    NcclId id{};
    const int rc = get ? get(&id) : 1;
    if(rc == 0) std::memcpy(id_out, &id, sizeof(id));
    dlclose(lib);
    return rc == 0 ? B200MIX_OK : B200MIX_ERR_CUDA;
}

int b200mix_shard_nccl(b200mix_device *d, uint32_t rank, uint32_t world, const void *nccl_id)
{
    if(!d) return B200MIX_ERR_INVALID;
    if(!nccl_id) { d->error = "shard_nccl: null id"; return B200MIX_ERR_INVALID; }
    if(int rc = shard_common(d, rank, world)) return rc;
    b200mix_device::Shard &S = d->shard;
    S.nccl_lib = nccl_open(d->error);
    if(!S.nccl_lib) return B200MIX_ERR_UNSUPPORTED;
    auto init = reinterpret_cast<int(*)(void**, int, NcclId, int)>(dlsym(S.nccl_lib, "ncclCommInitRank"));
    S.reduce = reinterpret_cast<decltype(S.reduce)>(dlsym(S.nccl_lib, "ncclReduce"));
    S.allreduce = reinterpret_cast<decltype(S.allreduce)>(dlsym(S.nccl_lib, "ncclAllReduce"));
    S.comm_destroy = reinterpret_cast<decltype(S.comm_destroy)>(dlsym(S.nccl_lib, "ncclCommDestroy"));
    if(!init || !S.reduce || !S.allreduce || !S.comm_destroy)
    { d->error = "shard_nccl: NCCL symbols missing"; return B200MIX_ERR_UNSUPPORTED; }
    NcclId id; std::memcpy(&id, nccl_id, sizeof(id));
    if(init(&S.comm, int(world), id, int(rank)) != 0)
    { d->error = "ncclCommInitRank failed"; S.comm = nullptr; return B200MIX_ERR_CUDA; }
    S.transport = 2; S.epoch = 0;
    return B200MIX_OK;
}

int b200mix_shard_last_us(b200mix_device *d, float *wet_us, float *real_us)
{
    if(!d || !d->shard.transport) return B200MIX_ERR_INVALID;
    b200mix_device::Shard &S = d->shard;
    float ms = 0.0f;
    if(wet_us)
    {
        *wet_us = -1.0f;
        if(S.ev_wet && cudaEventSynchronize(S.ev[1]) == cudaSuccess
            && cudaEventElapsedTime(&ms, S.ev[0], S.ev[1]) == cudaSuccess) *wet_us = ms*1000.0f;
    }
    if(real_us)
    {
        *real_us = -1.0f;
        if(S.ev_real && cudaEventSynchronize(S.ev[3]) == cudaSuccess
            && cudaEventElapsedTime(&ms, S.ev[2], S.ev[3]) == cudaSuccess) *real_us = ms*1000.0f;
    }
    return B200MIX_OK;
}

int b200mix_get_dry(b200mix_device *d, float *dry)
{
    if(!d || !dry) return B200MIX_ERR_INVALID;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d, cudaStreamSynchronize(d->stream));
    CUDA_TRY(d, cudaMemcpy(dry, d->d_dry, size_t(d->desc.dry_channels)*kLine*sizeof(float),
        cudaMemcpyDeviceToHost));
    return B200MIX_OK;
}

int64_t b200mix_get_resampler_table(b200mix_device *d, uint32_t which, float *out, size_t max_floats)
{
    if(!d) return -1;
    if(cudaSetDevice(d->cuda_dev) != cudaSuccess) return -1;
    const float *src = nullptr; size_t n = 0;
    if(which == B200MIX_RESAMPLER_SPLINE) { src = d->d_cubic[0]; n = 256; }
    else if(which == B200MIX_RESAMPLER_GAUSSIAN) { src = d->d_cubic[1]; n = 256; }
    else if(bsinc_for(d, which))
    {
        const int i = int(which - B200MIX_RESAMPLER_FAST_BSINC12) >> 1;
        src = d->d_bsinc[i]; n = d->bsinc[i].tab.size();
    }
    else return -1;
    if(out)
    {
        cudaStreamSynchronize(d->stream);
        if(cudaMemcpy(out, src, std::min(n, max_floats)*sizeof(float), cudaMemcpyDeviceToHost)
            != cudaSuccess) return -1;
    }
    return int64_t(n);
}

// Taps per output sample the resampler of a voice with this step runs (BsincPrepare's m for
// the bsinc family, alc/alu.cpp:140-165; 4 for the cubic family, 2 linear, 1 point; 0 for the
// pitch-1.0 copy) and whether it is the full BSinc form (scale interpolation, mixer_c.cpp:84-105).
int b200mix_resampler_taps(b200mix_device *d, uint32_t resampler, uint32_t step, uint32_t *full)
{
    if(!d || resampler > B200MIX_RESAMPLER_BSINC48) return B200MIX_ERR_INVALID;
    if(full) *full = 0u;
    if(const BsincTable *t = bsinc_for(d, resampler))
    {
        const BsincState st = PrepareBsinc(*t, step);
        if(full) *full = (step > 65536u && (resampler & 1u)) ? 1u : 0u;
        return int(st.m);
    }
    return resampler >= 2u ? 4 : (resampler == 1u ? 2 : 1);
}

int b200mix_profile(b200mix_device *d, int enable)
{
    if(!d) return B200MIX_ERR_INVALID;
    CUDA_TRY(d, cudaSetDevice(d->cuda_dev));
    if(enable && !d->ev_mix1)
    {
        CUDA_TRY(d, d->ev_mix0.create());
        CUDA_TRY(d, d->ev_mix1.create());
    }
    if(enable >= 2 && !d->ev_stage[b200mix_device::kStages])
        for(Event &e : d->ev_stage) CUDA_TRY(d, e.create());
    d->profile = enable != 0;
    d->profile_level = enable;
    d->ev_valid = false; d->stage_valid = false;
    return B200MIX_OK;
}

int b200mix_last_stage_ms(b200mix_device *d, float *ms, uint32_t count)
{
    if(!d || !ms || !d->stage_valid) return B200MIX_ERR_INVALID;
    if(cudaEventSynchronize(d->ev_stage[b200mix_device::kStages]) != cudaSuccess) return B200MIX_ERR_CUDA;
    for(uint32_t i = 0;i < count && i < uint32_t(b200mix_device::kStages);++i)
        if(cudaEventElapsedTime(&ms[i], d->ev_stage[i], d->ev_stage[i+1]) != cudaSuccess) return B200MIX_ERR_CUDA;
    return int(b200mix_device::kStages);
}

float b200mix_last_mix_kernel_ms(b200mix_device *d)
{
    if(!d || !d->ev_valid) return -1.0f;
    if(cudaEventSynchronize(d->ev_mix1) != cudaSuccess) return -1.0f;
    float ms = -1.0f;
    if(cudaEventElapsedTime(&ms, d->ev_mix0, d->ev_mix1) != cudaSuccess) return -1.0f;
    return ms;
}

uint64_t b200mix_launch_count(const b200mix_device *d) { return d ? d->launches : 0; }
void *b200mix_stream(b200mix_device *d) { return d ? static_cast<void*>(d->stream) : nullptr; }

} // extern "C"
