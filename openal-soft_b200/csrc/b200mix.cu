// b200mix.cu — host side of the C ABI in include/b200mix.h.
//
// Owns the device-resident mirrors of the reference's mixer state (voices, gain targets, mix
// buffers) and the parts that keep the rest: BufferTable (buffers), VoiceBook (per-voice
// bookkeeping), VoiceLoop (resample kernel to complete Dry / RealOut / Wet), SlotTable (effect
// slots), OutputStage (post-process to the interleaved output).  An update runs on one CUDA stream:
//   [k_apply_updates]  voice loop  effect slots  post-process  (D2H)
// No CPU mixing path exists: every entry point fails with B200MIX_ERR_CUDA when the CUDA
// runtime/device is unusable.
#include "../../include/b200mix.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include <dlfcn.h>

#include "mixer_kernels.cuh"
#include "shard_kernels.cuh"
#include "param_kernels.hpp"
#include "resampler_tables.hpp"
#include "hrtf_store.hpp"
#include "adpcm.hpp"
#include "device_memory.hpp"
#include "voice_book.hpp"
#include "slot_table.hpp"
#include "output_stage.hpp"
#include "buffer_table.hpp"
#include "voice_loop.hpp"

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
    DevArray<VoiceRec> d_voices;
    BufferTable buffers;                          // buffers and callback buffers, source of the device's records
    VoiceBook book;                               // host mirror of the voices, source of the loop's lists
    DevArray<float2> d_hrtf_tgt, d_hrtf_old;
    DevArray<float> d_dry_cur, d_dry_tgt, d_send_cur, d_send_tgt;
    VoiceResult *d_results{nullptr};              // inside d_outblock
    b200mix_voice_result *h_results{nullptr};     // inside h_outblock (pinned)
    DevArray<char> d_outblock; PinnedArray<char> h_outblock; size_t out_real_bytes{0};

    // mix buffers
    uint32_t dry_alloc_ch{0};
    DevArray<float> d_dry, d_wet;
    float *d_real{nullptr};                       // d_dry, or inside d_outblock
    float *h_real{nullptr};                       // pinned [real][1024]
    VoiceLoop loop;                               // resample kernel to complete Dry / RealOut / Wet
    OutputStage out;                              // post-process, limiter, distance comp, interleaved output

    UploadArena stage;                            // b200mix_voices_update's inputs (see ensure_stage)

    SlotTable slots;                              // effect slots, from install to launch

    // attached HRTF data set (device-side HrtfStore::getCoeffs)
    DevArray<float2> d_st_fields; DevArray<uint2> d_st_elevs; DevArray<float2> d_st_coeffs;
    DevArray<uint8_t> d_st_delays; uint32_t st_num_fields{0}, st_ir{0};
    bool mid_render{false}; uint32_t mid_frames{0};   // between render_begin and render_end
    bool profile{false};
    Event ev_mix0, ev_mix1;
    bool ev_valid{false};
    // stage marks of the last update (profile >= 2): see b200mix_last_stage_ms
    static constexpr int kStages = 8;
    Event ev_stage[kStages + 1];
    bool stage_valid{false}; int profile_level{0};

    // GPU parameter stage (b200mix_sources_update): pinned input staging + device scratch
    UploadArena src;

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

    ~b200mix_device() { if(stream) cudaStreamDestroy(stream); }
};

namespace {

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
    CUDA_TRY(d->error, d->stage.reserve(n, cap, bytes, bytes, d->stream));
    return B200MIX_OK;
}

const BsincTable *bsinc_for(const b200mix_device *d, uint32_t resampler)
{
    if(resampler < B200MIX_RESAMPLER_FAST_BSINC12 || resampler > B200MIX_RESAMPLER_BSINC48)
        return nullptr;
    return &d->bsinc[(resampler - B200MIX_RESAMPLER_FAST_BSINC12) >> 1];
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
    if(!stopped && !nobuf && d->buffers.cb_slot(p.flags, p.buffer) < 0)
    {
        if(p.flags & B200MIX_VF_STATIC)
        { if(const char *why = d->buffers.unplayable_static(p.buffer, (p.flags & B200MIX_VF_LOOPING) ? p.loop_end : 0u)) return bad(why); }
        // a streaming voice reads its queue: make sure the (empty) queue table exists
        else if(int rc = d->loop.ensure_queues()) return rc;
    }
    for(uint32_t s = 0;s < dd.num_sends;++s)
        if(p.send_slot[s] != B200MIX_NO_SLOT && p.send_slot[s] >= dd.max_slots)
            return bad("send slot out of range");
    if(!stopped && !hrtf && d->loop.parks_dry())
        if(int rc = d->loop.ensure_dry_bus()) return rc;
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
    d->loop.fill(A);
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    return (d->out.*set)(args...);
}

// Every buffer setter: on the mixer's GPU, the table checks the call against the buffers the voices
// hold, then builds and commits the new state (BufferTable).
template<typename... Params, typename... Args>
int set_buffer(b200mix_device *d, int (BufferTable::*set)(Params...), Args... args)
{
    if(!d) return B200MIX_ERR_INVALID;
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    return (d->buffers.*set)(args..., d->book.bufrefs);
}

// Every slot setter: on the mixer's GPU, the table checks the call, then builds and commits the new
// state (SlotTable).  A host allocation that fails is reported, not thrown across the C ABI.
template<typename... Params, typename... Args>
int set_slot(b200mix_device *d, int (SlotTable::*set)(Params...), Args... args)
{
    if(!d) return B200MIX_ERR_INVALID;
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    try { return (d->slots.*set)(args...); }
    catch(const std::bad_alloc &) { d->error = "out of memory"; return B200MIX_ERR_NOMEM; }
}

} // namespace

extern "C" {

static void shard_release(b200mix_device *d);

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
            CUDA_TRY(d->error, d->d_bsinc[i].alloc(d->bsinc[i].tab.size()));
            CUDA_TRY(d->error, upload(d->d_bsinc[i], d->bsinc[i].tab, d->stream));
        }
        const std::vector<float> cubic[2] = {BuildSplineTable(), BuildGaussianTable()};
        for(int i = 0;i < 2;++i)
        {
            CUDA_TRY(d->error, d->d_cubic[i].alloc(cubic[i].size()));
            CUDA_TRY(d->error, upload(d->d_cubic[i], cubic[i], d->stream));
        }

        const b200mix_device_desc &dd = d->desc;
        d->ir_pad = (dd.ir_size + 7u) & ~7u;
        CUDA_TRY(d->error, d->d_voices.alloc(dd.max_voices, d->stream));
        if(int rc = d->buffers.init(dd.max_buffers, dd.max_voices, d->stream, d->error)) return rc;
        d->book.init(dd.max_voices, dd.max_buffers, dd.num_sends, dd.max_slots);
        if(dd.ir_size)
        {
            CUDA_TRY(d->error, d->d_hrtf_tgt.alloc(size_t(dd.max_voices)*d->ir_pad, d->stream));
            CUDA_TRY(d->error, d->d_hrtf_old.alloc(size_t(dd.max_voices)*d->ir_pad, d->stream));
        }
        CUDA_TRY(d->error, d->d_dry_cur.alloc(size_t(dd.max_voices)*std::max(dd.dry_channels, 1u), d->stream));
        CUDA_TRY(d->error, d->d_dry_tgt.alloc(size_t(dd.max_voices)*std::max(dd.dry_channels, 1u), d->stream));
        if(dd.num_sends && dd.wet_channels)
        {
            const size_t per = size_t(dd.num_sends)*dd.wet_channels;
            CUDA_TRY(d->error, d->d_send_cur.alloc(dd.max_voices*per, d->stream));
            CUDA_TRY(d->error, d->d_send_tgt.alloc(dd.max_voices*per, d->stream));
        }
        if(int rc = d->loop.init(dd, d->num_sms, d->stream, d->error, d->d_dry_cur, d->d_dry_tgt, d->d_send_cur,
            d->d_send_tgt)) return rc;
        d->dry_alloc_ch = d->loop.dry_rows();
        CUDA_TRY(d->error, d->d_dry.alloc(size_t(d->dry_alloc_ch)*kLine, d->stream));
        // RealOut and the voice results share one block (and one pinned mirror): a render that
        // returns both needs ONE device-to-host copy
        {
            const size_t realFloats = size_t(std::max(dd.real_channels, 1u))*kLine;
            static_assert(sizeof(VoiceResult) == 16 && sizeof(b200mix_voice_result) == 16, "result layout");
            const size_t blockBytes = realFloats*sizeof(float) + size_t(dd.max_voices)*sizeof(VoiceResult);
            CUDA_TRY(d->error, d->d_outblock.alloc(blockBytes, d->stream));
            char *blk = d->d_outblock;
            d->d_results = reinterpret_cast<VoiceResult*>(blk + realFloats*sizeof(float));
            CUDA_TRY(d->error, d->h_outblock.alloc(blockBytes));
            d->h_real = reinterpret_cast<float*>(d->h_outblock.get());
            d->h_results = reinterpret_cast<b200mix_voice_result*>(d->h_outblock + realFloats*sizeof(float));
            d->out_real_bytes = realFloats*sizeof(float);
            if(dd.post_process == B200MIX_POST_NONE) d->d_real = d->d_dry;
            else d->d_real = reinterpret_cast<float*>(blk);
        }
        if(dd.max_slots && dd.wet_channels)
            CUDA_TRY(d->error, d->d_wet.alloc(size_t(dd.max_slots)*dd.wet_channels*kLine, d->stream));
        if(int rc = d->out.init(dd, d->stream, d->error)) return rc;
        if(int rc = d->slots.init(dd, uint32_t(d->num_sms), d->stream, d->error)) return rc;
        if(int rc = ensure_stage(d, std::min(dd.max_voices, 4096u))) return rc;
        CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
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

int b200mix_buffer_callback(b200mix_device *d, uint32_t buffer, const b200mix_callback_buffer *cb)
{ return set_buffer(d, &BufferTable::set_callback, buffer, cb); }

int b200mix_buffer_callback_state(b200mix_device *d, uint32_t buffer, uint32_t *num_blocks,
    uint32_t *block_offset, uint32_t *stopped)
{ return d ? d->buffers.callback_state(buffer, num_blocks, block_offset, stopped) : B200MIX_ERR_INVALID; }

int b200mix_buffer_data(b200mix_device *d, uint32_t buffer, uint32_t sample_type, uint32_t channels,
    uint32_t frames, const void *data, size_t bytes)
{ return set_buffer(d, &BufferTable::set_data, buffer, sample_type, channels, frames, data, bytes); }

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
    return b200mix_buffer_data(d, buffer, B200MIX_FMT_I16, channels, blocks*samples_per_block,
        pcm.data(), pcm.size()*sizeof(int16_t));
}

int b200mix_buffer_free(b200mix_device *d, uint32_t buffer)
{ return set_buffer(d, &BufferTable::free, buffer); }

int b200mix_slot_disable(b200mix_device *d, uint32_t slot)
{ return set_slot(d, &SlotTable::disable, slot); }

int b200mix_slot_convolution(b200mix_device *d, uint32_t slot, uint32_t ir_channels,
    uint32_t ir_frames, const float *ir)
{ return set_slot(d, &SlotTable::convolution, slot, ir_channels, ir_frames, ir); }

int b200mix_slot_reverb(b200mix_device *d, uint32_t slot, const b200mix_reverb_params *p)
{ return set_slot(d, &SlotTable::reverb, slot, p); }

int b200mix_slot_efx(b200mix_device *d, uint32_t slot, const b200mix_efx_props *props,
    const b200mix_efx_target *target)
{ return set_slot(d, &SlotTable::efx, slot, props, target); }

int b200mix_slot_target(b200mix_device *d, uint32_t slot, uint32_t target)
{ return set_slot(d, &SlotTable::target, slot, target); }

int b200mix_slot_reverb_update(b200mix_device *d, uint32_t slot, const b200mix_reverb_params *p,
    uint32_t full_update)
{ return set_slot(d, &SlotTable::reverb_update, slot, p, full_update); }

int b200mix_slot_output_gains(b200mix_device *d, uint32_t slot, uint32_t lines, const float *gains)
{ return set_slot(d, &SlotTable::output_gains, slot, lines, gains); }

int b200mix_hrtf_attach(b200mix_device *d, const b200mix_hrtf *h)
{
    if(!d || !h) return B200MIX_ERR_INVALID;
    if(h->ir_size > d->desc.ir_size)
    { d->error = "hrtf_attach: data set HRIRs are longer than the device's ir_size"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
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
    CUDA_TRY(d->error, d->d_st_fields.alloc(fields.size()));
    CUDA_TRY(d->error, d->d_st_elevs.alloc(elevs.size()));
    CUDA_TRY(d->error, d->d_st_coeffs.alloc(h->coeffs.size()/2));
    CUDA_TRY(d->error, d->d_st_delays.alloc(h->delays.size()));
    CUDA_TRY(d->error, cudaMemcpy(d->d_st_fields, fields.data(), fields.size()*sizeof(float2), cudaMemcpyHostToDevice));
    CUDA_TRY(d->error, cudaMemcpy(d->d_st_elevs, elevs.data(), elevs.size()*sizeof(uint2), cudaMemcpyHostToDevice));
    CUDA_TRY(d->error, cudaMemcpy(d->d_st_coeffs, h->coeffs.data(), h->coeffs.size()*sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(d->error, cudaMemcpy(d->d_st_delays, h->delays.data(), h->delays.size(), cudaMemcpyHostToDevice));
    d->st_num_fields = uint32_t(fields.size()); d->st_ir = h->ir_size;
    return B200MIX_OK;
}

static int voices_update_impl(b200mix_device *d, uint32_t n, const b200mix_voice_params *params,
    const float *hrtf_coeffs, const float *dirs, const float *dry_gains, const float *send_gains,
    bool direct);

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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
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
    }
    if(int rc = d->buffers.check_voices(n, params)) return rc;

    if(direct)
        if(int rc = d->loop.ensure_real_bus()) return rc;
    CUDA_TRY(d->error, d->stage.wait());
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
        d->buffers.apply_voice(p);
    }
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
    CUDA_TRY(d->error, d->stage.ship(d->stream));
    k_apply_updates<<<n, 64, 0, d->stream>>>(A);
    ++d->launches;
    CUDA_TRY(d->error, cudaGetLastError());
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));

    bool mayFilter = d->loop.filt() != nullptr;
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
        if(d->buffers.cb_slot(p.flags, p.buffer) >= 0)
        { d->error = "sources_update: callback buffers play through b200mix_voices_update"; return B200MIX_ERR_UNSUPPORTED; }
        if(!mayFilter && source_may_filter(P, dd.num_sends)) mayFilter = true;
    }
    if(mayFilter)
        if(int rc = d->loop.ensure_filters(d->launches)) return rc;
    // staging: [voices n][props n] in, [VoiceUpdate n][dirs n][dry][send][hf/lf][FilterUpdate] scratch
    const uint32_t paths = 1u + dd.num_sends;
    CUDA_TRY(d->error, d->src.wait());
    {
        const uint32_t cap = std::max<uint32_t>(n, 2u*uint32_t(d->src.capacity()));
        const size_t in = align16(size_t(cap)*sizeof(b200mix_source_voice)) + align16(size_t(cap)*sizeof(b200mix_source_props));
        const size_t out = align16(size_t(cap)*sizeof(VoiceUpdate)) + align16(size_t(cap)*16)
            + align16(size_t(cap)*std::max(dd.dry_channels, 1u)*4) + align16(size_t(cap)*std::max(dd.num_sends*dd.wet_channels, 1u)*4)
            + align16(size_t(cap)*(1u + B200MIX_MAX_SENDS)*8) + align16(size_t(cap)*paths*sizeof(FilterUpdate));
        CUDA_TRY(d->error, d->src.reserve(n, cap, in, in + out + 64, d->stream));
    }

    if(mayFilter) d->book.set_device_filters();
    for(uint32_t i = 0;i < n;++i)
    {
        const b200mix_source_voice &p = voices[i];
        const bool act = !(p.flags & B200MIX_VF_STOPPED);
        d->buffers.unbind(p.voice);           // it no longer plays a callback buffer
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
    CUDA_TRY(d->error, U.ship(d->stream));
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
    const bool filters = d->loop.filt() != nullptr;
    CUDA_TRY(d->error, launch_calc_voices(Q, filters, d->stream));
    d->launches += filters ? 2 : 1;

    ApplyParams A = apply_params(d, Q.updates);
    if(hrtfMode) apply_dirs(d, A, Q.dirs);
    else A.dry = Q.dry;
    A.send = Q.send;
    k_apply_updates<<<n, 64, 0, d->stream>>>(A);
    ++d->launches;
    if(filters)
    {
        k_apply_filter_updates<<<(2u*n*paths + 127u)/128u, 128, 0, d->stream>>>(d->loop.filt(), paths, Q.fupd, n*paths);
        ++d->launches;
    }
    CUDA_TRY(d->error, cudaGetLastError());
    return B200MIX_OK;
}

int b200mix_get_voice_targets(b200mix_device *d, uint32_t voice, uint32_t *step, float bsinc[4],
    float *hrtf_gain, uint32_t hrtf_delay[2], float *hrtf_coeffs, float *dry_gains, float *send_gains,
    float *filters)
{
    if(!d || voice >= d->desc.max_voices) return B200MIX_ERR_INVALID;
    const b200mix_device_desc &dd = d->desc;
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
    VoiceRec rec;
    CUDA_TRY(d->error, cudaMemcpy(&rec, d->d_voices + voice, offsetof(VoiceRec, prev), cudaMemcpyDeviceToHost));
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
        CUDA_TRY(d->error, cudaMemcpy(hrtf_coeffs, d->d_hrtf_tgt + size_t(voice)*d->ir_pad, size_t(dd.ir_size)*8, cudaMemcpyDeviceToHost));
    if(dry_gains && dd.dry_channels)
        CUDA_TRY(d->error, cudaMemcpy(dry_gains, d->d_dry_tgt + size_t(voice)*dd.dry_channels, size_t(dd.dry_channels)*4, cudaMemcpyDeviceToHost));
    if(send_gains && d->d_send_tgt)
        CUDA_TRY(d->error, cudaMemcpy(send_gains, d->d_send_tgt + size_t(voice)*dd.num_sends*dd.wet_channels,
            size_t(dd.num_sends)*dd.wet_channels*4, cudaMemcpyDeviceToHost));
    if(filters)
    {
        const uint32_t paths = 1u + dd.num_sends;
        for(uint32_t pth = 0;pth < paths;++pth)
        {
            float *o = filters + size_t(pth)*11;
            for(int k = 0;k < 11;++k) o[k] = k == 1 ? 1.0f : (k == 6 ? 1.0f : 0.0f);
            if(!d->loop.filt()) continue;
            FilterRec fr;
            CUDA_TRY(d->error, cudaMemcpy(&fr, d->loop.filt() + size_t(voice)*paths + pth, sizeof(fr), cudaMemcpyDeviceToHost));
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
        if(!d->buffers.queueable(buffers[i]))
        { d->error = "voice_queue: buffer id without data"; return B200MIX_ERR_INVALID; }
        Q.items[i] = buffers[i];
    }
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    return d->loop.set_queue(d->d_voices, Q, d->launches);
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    if(int rc = d->loop.ensure_filters(d->launches)) return rc;
    for(uint32_t i = 0;i < n;++i)
        if(filters[i].path == 0) d->book.set_direct_filter(filters[i].voice, filters[i].active != 0);
    return d->loop.set_filters(n, reinterpret_cast<const FilterUpdate*>(filters), d->launches);
}

// Stage mark i of an update (profile >= 2); marks 1 and 3 also bound the voice kernels (profile >= 1).
static inline void stage_mark(b200mix_device *d, int i)
{
    if(i == 3 && d->profile) { cudaEventRecord(d->ev_mix1, d->stream); d->ev_valid = true; }
    if(d->profile_level >= 2) cudaEventRecord(d->ev_stage[i], d->stream);
    if(i == 1 && d->profile) cudaEventRecord(d->ev_mix0, d->stream);
}

// Phase A of an update: clear the mix buffers, mix every voice, reduce the partial rows and
// finish the aux sends -> the slots' Wet buffers are complete (alc/alu.cpp:2196-2206).
static int render_phase_a(b200mix_device *d, uint32_t frames, bool want_results, bool force_sends)
{
    const b200mix_device_desc &dd = d->desc;
    if(frames < 1 || frames > B200MIX_LINE_SIZE)
    { d->error = "render: frames out of range"; return B200MIX_ERR_INVALID; }
    if(const char *why = d->out.missing()) { d->error = std::string("render: ") + why; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    // all the update allocates, before anything of it is on the stream
    if(int rc = d->loop.prepare(d->book, frames, d->slots.active() || force_sends)) return rc;
    // callback buffers: their callbacks run here, before anything of the update is launched
    const BufferRec *cbplan = nullptr;
    if(int rc = d->buffers.plan(frames, cbplan)) return rc;

    stage_mark(d, 0);
    // clear MixBuffer (alc/alu.cpp:2417) and the wet buffers (alc/alu.cpp:2196-2198)
    // (the dry mix is left alone while nothing can write or read it: HRTF-only scenes; an
    // HRTF post-process whose RealOut is just L/R overwrites it instead of accumulating, unless
    // the RealOut bus has mixed direct-channel voices into it)
    if(d->book.dry_active || d->slots.ever_installed() || dd.post_process != B200MIX_POST_HRTF)
        CUDA_TRY(d->error, cudaMemsetAsync(d->d_dry, 0, size_t(d->dry_alloc_ch)*kLine*sizeof(float), d->stream));
    if(d->d_real != d->d_dry && (!d->out.overwrites_real() || d->loop.real_mixed()))
        CUDA_TRY(d->error, cudaMemsetAsync(d->d_real, 0, size_t(dd.real_channels)*kLine*sizeof(float), d->stream));
    if(d->d_wet)
        CUDA_TRY(d->error, cudaMemsetAsync(d->d_wet, 0, size_t(dd.max_slots)*dd.wet_channels*kLine*sizeof(float), d->stream));

    const MixParams P{.voices = d->d_voices, .buffers = d->buffers.device(), .hrtf_tgt = d->d_hrtf_tgt,
        .hrtf_old = d->d_hrtf_old, .dry_cur = d->d_dry_cur, .dry_tgt = d->d_dry_tgt,
        .results = want_results ? d->d_results : nullptr, .bsinc_tab = {d->d_bsinc[0], d->d_bsinc[1], d->d_bsinc[2]},
        .cubic_tab = {d->d_cubic[0], d->d_cubic[1]}, .ir_pad = d->ir_pad, .cbplan = cbplan};
    return d->loop.launch(P, d->book, d->d_dry, d->d_real, d->d_wet, d->launches, [d](int i) { stage_mark(d, i); });
}

// Phase B: run the effect slots on their Wet input, mix their output into Dry, post-process
// (alc/alu.cpp:2252-2256, 2439-2443).
static int render_phase_b(b200mix_device *d, uint32_t frames)
{
    stage_mark(d, 6);
    if(int rc = d->slots.run(frames, d->d_wet, d->d_dry, d->launches)) return rc;
    stage_mark(d, 7);
    if(int rc = d->out.post(d->d_dry, d->d_real, d->loop.partial(), d->loop.fir_rows(),
        d->book.dry_active || d->slots.ever_installed(), d->loop.real_mixed(), d->loop.fir_done(), frames,
        d->launches)) return rc;
    stage_mark(d, 8);
    if(d->profile_level >= 2) d->stage_valid = true;
    CUDA_TRY(d->error, cudaGetLastError());
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
        d->loop.fir_done() = 0;     // a kernel that `launches` does not count
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
        CUDA_TRY(d->error, cudaGetLastError());
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
    CUDA_TRY(d->error, cudaGetLastError());
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
        CUDA_TRY(d->error, cudaMemcpyAsync(d->h_outblock, d->d_outblock, d->out_real_bytes + size_t(nv)*sizeof(VoiceResult),
            cudaMemcpyDeviceToHost, d->stream));
    else
    {
        if(real_out)
            CUDA_TRY(d->error, cudaMemcpyAsync(d->h_real, d->d_real, size_t(dd.real_channels)*kLine*sizeof(float),
                cudaMemcpyDeviceToHost, d->stream));
        if(results)
            CUDA_TRY(d->error, cudaMemcpyAsync(d->h_results, d->d_results, size_t(nv)*sizeof(VoiceResult),
                cudaMemcpyDeviceToHost, d->stream));
    }
    if(d->shard.transport == 1)
        CUDA_TRY(d->error, cudaMemcpyAsync(d->shard.h_status, d->shard.own + offsetof(ShardCtl, status),
            sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
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
    d->loop.fir_done() = 0;         // the caller may use the stream before render_end
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
    shard_release(d);
    d->shard.rank = rank; d->shard.world = world;
    for(Event &e : d->shard.ev) CUDA_TRY(d->error, e.create());
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
    CUDA_TRY(d->error, S.own.alloc(S.off_wet + size_t(2)*world*S.wet_src_floats*sizeof(float)));
    CUDA_TRY(d->error, cudaMemset(S.own, 0, S.own.bytes()));
    CUDA_TRY(d->error, S.d_counters.alloc(4 + kShardMaxWorld, d->stream));
    CUDA_TRY(d->error, S.h_status.alloc(1));
    *S.h_status = 0u;
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
    cudaIpcMemHandle_t h;
    CUDA_TRY(d->error, cudaIpcGetMemHandle(&h, S.own));
    std::memcpy(handle_out, &h, sizeof(h));
    return B200MIX_OK;
}

int b200mix_shard_connect(b200mix_device *d, const void *handles)
{
    if(!d) return B200MIX_ERR_INVALID;
    b200mix_device::Shard &S = d->shard;
    if(!handles || !S.own || S.transport)
    { d->error = "shard_connect: call b200mix_shard_init first (once)"; return B200MIX_ERR_INVALID; }
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    for(uint32_t r = 0;r < S.world;++r)
    {
        if(r == S.rank) { S.peer[r] = S.own.get(); continue; }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, static_cast<const char*>(handles) + size_t(r)*sizeof(h), sizeof(h));
        void *p = nullptr;
        CUDA_TRY(d->error, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    CUDA_TRY(d->error, cudaStreamSynchronize(d->stream));
    CUDA_TRY(d->error, cudaMemcpy(dry, d->d_dry, size_t(d->desc.dry_channels)*kLine*sizeof(float),
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
    CUDA_TRY(d->error, cudaSetDevice(d->cuda_dev));
    if(enable && !d->ev_mix1)
    {
        CUDA_TRY(d->error, d->ev_mix0.create());
        CUDA_TRY(d->error, d->ev_mix1.create());
    }
    if(enable >= 2 && !d->ev_stage[b200mix_device::kStages])
        for(Event &e : d->ev_stage) CUDA_TRY(d->error, e.create());
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
