// buffer_table.hpp — the host's state of every buffer: the record the device's copy is uploaded
// from and the samples it views, the callback registrations (AL_SOFT_callback_buffer), the
// planner's mirror of the voices that play them, and the pinned arenas a callback update's samples
// travel in.  It is the only code that writes a buffer record to the device.  Host code only.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200mix.h"
#include "mixer_kernels.cuh"
#include "device_memory.hpp"
#include "callback_plan.hpp"
#include "adpcm.hpp"

namespace b200mix {

// Every call below returns a B200MIX_* code and, when it fails, sets the device's error string.
#define BUF_TRY(expr) do { const cudaError_t e_ = (expr); if(e_ != cudaSuccess) return fail(#expr, e_); } while(0)

class BufferTable {
public:
    // `err`: the device's error string, which outlives the table.
    int init(uint32_t max_buffers, uint32_t max_voices, cudaStream_t stream, std::string &err)
    {
        n_ = max_buffers; s_ = stream; err_ = &err;
        bufs_.resize(std::max(max_buffers, 1u));
        voices_.assign(max_voices, CbVoice{});
        BUF_TRY(d_buffers_.alloc(bufs_.size(), s_));
        BUF_TRY(zero_.alloc(kCbPad, s_));
        return B200MIX_OK;
    }
    const BufferRec *device() const { return d_buffers_; }

    // ---- setters: each checks its arguments, refuses a buffer that an active voice holds (`bufrefs`: the
    // voice book's active static voices per buffer), builds the new state in a local and commits it once
    // the stream is idle, so a refused or failed call changes nothing.  set_data and free end a registration.
    int set_data(uint32_t buffer, uint32_t sample_type, uint32_t channels, uint32_t frames, const void *data,
        size_t bytes, const std::vector<uint32_t> &bufrefs)
    {
        if(buffer >= n_ || sample_type > B200MIX_FMT_ALAW || channels < 1 || !data)
            return refuse("buffer_data: bad arguments");
        const size_t need = size_t(frames)*channels*kSampleBytes[sample_type];
        if(bytes < need) return refuse("buffer_data: short data");
        if(int rc = releasable(buffer, bufrefs, "buffer_data", kHeld)) return rc;
        Buf next;
        BUF_TRY(next.store.alloc(need + 16));   // +16 bytes: vector/tail reads past the last frame stay inside
        BUF_TRY(cudaMemcpyAsync(next.store.get(), data, need, cudaMemcpyHostToDevice, s_));
        next.rec = BufferRec{next.store.get(), frames, sample_type, channels, 0u};
        return commit(buffer, std::move(next));
    }

    // A new callback buffer, or a registered one's new callback and state.
    int set_callback(uint32_t buffer, const b200mix_callback_buffer *cb, const std::vector<uint32_t> &bufrefs)
    {
        if(buffer >= n_ || !cb || cb->struct_size != sizeof(b200mix_callback_buffer) || !cb->callback
            || cb->sample_type > B200MIX_FMT_MSADPCM || cb->channels < 1 || !cb->storage
            || cb->samples_per_block < 1 || cb->bytes_per_block < 1)
            return refuse("buffer_callback: bad arguments");
        const bool adpcm = cb->sample_type >= B200MIX_FMT_IMA4;
        const bool ms = cb->sample_type == B200MIX_FMT_MSADPCM;
        if(adpcm ? (cb->channels > 2 || !AdpcmBlockValid(ms, cb->samples_per_block)
                    || cb->bytes_per_block != AdpcmBlockBytes(ms, cb->channels, cb->samples_per_block))
                 : (cb->samples_per_block != 1u || cb->bytes_per_block != cb->channels*kSampleBytes[cb->sample_type]))
            return refuse("buffer_callback: block size does not match the format");
        if(cb->channels > 16u)
        { *err_ = "buffer_callback: more than 16 channels"; return B200MIX_ERR_UNSUPPORTED; }
        // PrepareCallback's size (al/buffer.cpp:468-473): MixerLineSize*MaxPitch + MaxResamplerEdge
        // samples in whole blocks.  No request of the reference's chunk loop passes it, so the
        // callbacks of an update never stop half way.
        const uint64_t lineBlocks = ((1024u + 256u)*10u + 24u + cb->samples_per_block - 1u) / cb->samples_per_block;
        if(cb->storage_bytes < lineBlocks*cb->bytes_per_block)
            return refuse("buffer_callback: storage smaller than the reference's callback storage");
        if(uint64_t(cb->num_blocks)*cb->bytes_per_block > cb->storage_bytes || cb->stopped > 1u)
            return refuse("buffer_callback: state outside the storage");
        int32_t s = bufs_[buffer].slot;    // a registered buffer keeps its slot, and its voices play on
        if(int rc = s < 0 ? releasable(buffer, bufrefs, "buffer_callback", kHeld) : B200MIX_OK) return rc;
        if(s < 0) s = int32_t(std::find(slots_.begin(), slots_.end(), B200MIX_NO_BUFFER) - slots_.begin());
        // the kernel reads the samples from the update's arena: the record carries the format, and
        // zeros to read should a voice ever meet it without a plan
        return commit(buffer, Buf{BufferRec{zero_.get(), 0u, adpcm ? uint32_t(B200MIX_FMT_I16) : cb->sample_type,
            cb->channels, uint32_t(s) + 1u}, {}, s, *cb, cbplan::State{cb->num_blocks, cb->block_offset, cb->stopped},
            cb->channels*(adpcm ? 2u : kSampleBytes[cb->sample_type])});
    }

    int free(uint32_t buffer, const std::vector<uint32_t> &bufrefs)
    {
        if(buffer >= n_) return B200MIX_ERR_INVALID;
        if(int rc = releasable(buffer, bufrefs, "buffer_free",
            "the buffer is attached to an active voice; stop the voice first")) return rc;
        return bufs_[buffer].rec.data ? commit(buffer, Buf{}) : B200MIX_OK;
    }

    // The state of a callback buffer after the last update (b200mix_buffer_callback_state).
    int callback_state(uint32_t buffer, uint32_t *num_blocks, uint32_t *block_offset, uint32_t *stopped)
    {
        if(buffer >= n_ || bufs_[buffer].slot < 0) return refuse("buffer_callback_state: not a callback buffer");
        const cbplan::State &st = bufs_[buffer].st;
        if(num_blocks) *num_blocks = st.num_blocks;
        if(block_offset) *block_offset = st.block_offset;
        if(stopped) *stopped = st.stopped;
        return B200MIX_OK;
    }

    // Plan slot of the callback buffer an entry plays (-1: none).
    int32_t cb_slot(uint32_t flags, uint32_t buffer) const
    { return !(flags & B200MIX_VF_STOPPED) && buffer != B200MIX_NO_BUFFER ? bufs_[buffer].slot : -1; }

    // Why a static voice cannot play `buffer` up to `loop_end` (0: not looping), or null.
    const char *unplayable_static(uint32_t buffer, uint32_t loop_end) const
    {
        const BufferRec &r = bufs_[buffer].rec;
        return !r.data || !r.frames ? "static voice on a buffer without data" : loop_end > r.frames ? "loop end beyond the buffer" : nullptr;
    }

    // A streaming voice may queue `buffer`: it holds samples of its own.
    bool queueable(uint32_t buffer) const { return buffer < n_ && bufs_[buffer].rec.data && !bufs_[buffer].rec.pad; }

    // The callback checks of one b200mix_voices_update call, on a copy of the mirror as the call leaves it: a
    // callback voice is not static, joins with RESET, and agrees with its buffer's other voices (group).
    int check_voices(uint32_t n, const b200mix_voice_params *params)
    {
        if(idle()) return B200MIX_OK;
        next_.assign(voices_.begin(), voices_.begin() + hi_);     // voices from hi_ on are unbound
        for(uint32_t i = 0;i < n;++i)
        {
            const b200mix_voice_params &p = params[i];
            const int32_t s = cb_slot(p.flags, p.buffer);
            const CbVoice cur = p.voice < next_.size() ? next_[p.voice] : CbVoice{};
            if(s >= 0 && (p.flags & B200MIX_VF_STATIC))
                return refuse("voices_update: a callback buffer is not static (IsCallback)");
            if(s >= 0 && cur.slot != s && !(p.flags & B200MIX_VF_RESET))
                return refuse("voices_update: a voice starts a callback buffer with B200MIX_VF_RESET");
            const CbVoice nx = next_voice(cur, p);
            if(nx.slot >= 0 && p.voice >= next_.size()) next_.resize(p.voice + 1u);
            if(p.voice < next_.size()) next_[p.voice] = nx;
        }
        return group(next_, uint32_t(next_.size())) ? B200MIX_OK
            : refuse("voices_update: voices sharing a callback buffer disagree on step, position or state");
    }

    // What a checked entry does to the mirror (what k_apply_updates does to the voice's record).
    void apply_voice(const b200mix_voice_params &p)
    {
        if(idle()) return;
        CbVoice &cv = voices_[p.voice];
        const CbVoice nx = next_voice(cv, p);
        bound_ = bound_ + (nx.slot >= 0) - (cv.slot >= 0);
        if(nx.slot >= 0) hi_ = std::max(hi_, p.voice + 1u);
        if(nx.slot >= 0 && (p.flags & B200MIX_VF_RESET)) bufs_[slots_[size_t(nx.slot)]].st = cbplan::State{};
        cv = nx;
    }

    // The voice no longer plays a callback buffer (b200mix_sources_update).
    void unbind(uint32_t voice) { if(voices_[voice].slot >= 0) { voices_[voice].slot = -1; --bound_; } }

    // The callback buffers' part of an update (callback_plan.hpp).  First every callback buffer's
    // callbacks run on this thread; then, straight into the pinned arena, each buffer's plan record and
    // the blocks it has stored (ADPCM decoded to int16) are packed, its storage is compacted as the
    // reference does after the mix, and its voices' mirror advances; table and samples go to the GPU
    // with one copy on the mixer stream.  *plan stays null when no callback voice mixes this update.
    int plan(uint32_t frames, const BufferRec *&plan)
    {
        plan = nullptr;
        if(!bound_) return B200MIX_OK;
        group(voices_, hi_);             // true: check_voices keeps them so, and they advance together below
        if(std::none_of(reps_.begin(), reps_.end(), [](int32_t r) { return r >= 0; })) return B200MIX_OK;
        work_.resize(slots_.size());
        // 1. the callbacks.  Registration guarantees the reference's storage size, which no request of
        //    its chunk loop passes: plan_loads cannot stop half way through the buffers.
        size_t size = UploadArena::align(slots_.size()*sizeof(BufferRec));
        for(size_t s = 0;s < slots_.size();++s)
        {
            if(reps_[s] < 0) continue;
            Buf &c = bufs_[slots_[s]];
            CbWork &w = work_[s];
            const b200mix_callback_buffer &cb = c.cb;
            auto request = [&cb](uint64_t offset, uint32_t bytes) -> int64_t {
                return cb.callback(cb.userptr, static_cast<char*>(cb.storage) + offset, int(bytes));
            };
            w.start = c.st;
            if(!cbplan::plan_loads(c.st, cb.samples_per_block, cb.bytes_per_block, voices_[size_t(reps_[s])].v,
                frames, cb.storage_bytes, request, w.loads))
                return refuse("render: a callback request passes the callback buffer's storage");
            // [pad | the stored blocks as the kernel reads them | pad], a pad holding one frame and
            // 16 bytes: a load held at the last stored sample may address the frame before the first
            // (none stored) or the first (empty span); the bulk copies round their runs up to 16 bytes
            const size_t pad = UploadArena::align(c.frame_bytes) + 16u;
            w.bytes = w.loads.chunks ? size_t(c.st.num_blocks)*cb.samples_per_block*c.frame_bytes : 0u;
            w.region = size + pad;
            size = w.region + UploadArena::align(w.bytes) + pad;
        }
        // 2. the arena (two alternate: the other one's copy may still be in flight)
        UploadArena &U = arena_[idx_];
        BUF_TRY(U.wait());
        BUF_TRY(U.reserve(size, size*2, size*2, size*2, s_));
        U.begin();
        uint8_t *arena = U.host_part<uint8_t>(size);
        const uintptr_t devArena = reinterpret_cast<uintptr_t>(U.dev_of(arena));
        // 3. pack, then what the reference does after the mix
        std::memset(arena, 0, size);
        for(size_t s = 0;s < slots_.size();++s)
        {
            if(reps_[s] < 0) continue;
            Buf &c = bufs_[slots_[s]];
            const CbWork &w = work_[s];
            const b200mix_callback_buffer &cb = c.cb;
            cbplan::Voice &vm = voices_[size_t(reps_[s])].v;
            const cbplan::Span span = cbplan::span_of(w.start, vm, cb.samples_per_block, c.st);
            BufferRec rec = c.rec;
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
            for(uint32_t v : members_[s]) voices_[v].v = vm;
        }
        BUF_TRY(U.ship(s_));
        idx_ ^= 1;
        plan = reinterpret_cast<const BufferRec*>(devArena);
        return B200MIX_OK;
    }

private:
    static constexpr uint32_t kSampleBytes[] = {1, 2, 4, 4, 8, 1, 1};   // per PCM b200mix_sample_type
    static constexpr const char *kHeld = "the buffer is attached to an active voice (AL_INVALID_OPERATION)";
    static constexpr size_t kCbPad = 256;               // zeros that cover a callback buffer's frame (16*8 bytes)

    // A buffer: its device record and the samples that views.  A callback buffer views zeros; its plan slot
    // is rec.pad - 1 (else -1), with its registration, state and bytes per arena frame (int16 for ADPCM).
    struct Buf { BufferRec rec{}; DevArray<char> store; int32_t slot{-1};
        b200mix_callback_buffer cb{}; cbplan::State st{}; uint32_t frame_bytes{0}; };
    // A voice as the planner sees it: the plan slot it is bound to (-1: none) and its position and
    // state, which advance by the same arithmetic as on the device, so planning needs no read-back
    struct CbVoice { int32_t slot{-1}; cbplan::Voice v{}; };
    struct CbWork { cbplan::State start; cbplan::Loads loads; size_t region{0}, bytes{0}; };

    int refuse(const std::string &why) { *err_ = why; return B200MIX_ERR_INVALID; }
    int fail(const char *what, cudaError_t e) { *err_ = std::string(what) + ": " + cudaGetErrorString(e); return B200MIX_ERR_CUDA; }

    // No callback buffer is registered or played: the mirror has nothing to follow.
    bool idle() const { return !bound_ && std::all_of(slots_.begin(), slots_.end(), [](uint32_t b) { return b == B200MIX_NO_BUFFER; }); }

    // Refused while a voice plays `buffer` as a callback buffer, or an active static voice holds it.
    int releasable(uint32_t buffer, const std::vector<uint32_t> &bufrefs, const char *what, const char *held)
    {
        const Buf &b = bufs_[buffer];
        if(b.slot >= 0 && std::any_of(voices_.begin(), voices_.begin() + hi_, [&b](const CbVoice &cv)
            { return cv.slot == b.slot && (cv.v.state == 1u || cv.v.state == 2u); }))
            return refuse(std::string(what) + ": the callback buffer is played by a voice; stop it first");
        return b.rec.data && bufrefs[buffer] ? refuse(std::string(what) + ": " + held) : B200MIX_OK;
    }

    // Once the stream is idle (queued kernels may still read what is replaced, and `next`'s copies
    // have landed), `next` replaces the buffer; a registration that ends unbinds its voices.
    int commit(uint32_t buffer, Buf &&next)
    {
        BUF_TRY(cudaMemcpyAsync(d_buffers_ + buffer, &next.rec, sizeof(BufferRec), cudaMemcpyHostToDevice, s_));
        BUF_TRY(cudaStreamSynchronize(s_));
        Buf &b = bufs_[buffer];
        if(b.slot >= 0 && b.slot != next.slot)
        {
            for(uint32_t v = 0;v < hi_;++v) if(voices_[v].slot == b.slot) unbind(v);
            slots_[size_t(b.slot)] = B200MIX_NO_BUFFER;
        }
        if(size_t(next.slot + 1) > slots_.size()) slots_.push_back(buffer);     // a new slot
        else if(next.slot >= 0) slots_[size_t(next.slot)] = buffer;
        b = std::move(next);
        return B200MIX_OK;
    }

    // What the checked entry `p` makes of the voice.
    CbVoice next_voice(CbVoice cv, const b200mix_voice_params &p) const
    {
        const bool nobuf = p.buffer == B200MIX_NO_BUFFER;
        if(!nobuf || (p.flags & B200MIX_VF_STOPPED)) cv.slot = cb_slot(p.flags, p.buffer);   // else it stays bound
        if(cv.slot < 0) return cv;
        cbplan::Voice &m = cv.v;
        if(p.flags & B200MIX_VF_RESET) { m.pos = p.position; m.frac = p.position_frac; m.have_buffer = true; }
        if(p.flags & B200MIX_VF_STOPPING) m.state = 2u;
        else if(p.flags & B200MIX_VF_PLAYING) m.state = 1u;
        m.step = p.step;
        if(nobuf) m.have_buffer = false;
        return cv;
    }

    // The voices of each callback buffer are the channels of one source: reps_[slot] = the first of vs[0, hi)
    // that mixes this update (-1: none), members_[slot] the others, which agree with it (else false).
    bool group(const std::vector<CbVoice> &vs, uint32_t hi)
    {
        reps_.assign(slots_.size(), -1);
        members_.resize(slots_.size());
        for(auto &m : members_) m.clear();
        for(uint32_t v = 0;v < hi;++v)
        {
            const CbVoice &cv = vs[v];
            if(cv.slot < 0 || (cv.v.state != 1u && cv.v.state != 2u)) continue;
            int32_t &r = reps_[size_t(cv.slot)];
            if(r < 0) { r = int32_t(v); continue; }
            const cbplan::Voice &a = vs[size_t(r)].v, &b = cv.v;
            if(a.pos != b.pos || a.frac != b.frac || a.step != b.step || a.state != b.state
                || a.have_buffer != b.have_buffer) return false;
            members_[size_t(cv.slot)].push_back(v);
        }
        return true;
    }

    uint32_t n_{0}; cudaStream_t s_{nullptr}; std::string *err_{nullptr};   // n_: max_buffers
    std::vector<Buf> bufs_; DevArray<BufferRec> d_buffers_;
    DevArray<char> zero_;                // zeros behind every callback buffer's own record
    std::vector<uint32_t> slots_;        // per plan slot: its callback buffer (B200MIX_NO_BUFFER: free)
    std::vector<CbVoice> voices_, next_; // per voice; check_voices' copy
    uint32_t bound_{0}, hi_{0};          // voices bound to a callback buffer; 1 + the highest ever bound
    UploadArena arena_[2]; int idx_{0};  // alternating: one is filled while the other's copy is in flight
    std::vector<int32_t> reps_;          // per slot: the voice the update is planned from (-1: none)
    std::vector<std::vector<uint32_t>> members_;   // per slot: its other mixing voices
    std::vector<CbWork> work_;           // per slot, for the update being planned
};

#undef BUF_TRY

} // namespace b200mix
