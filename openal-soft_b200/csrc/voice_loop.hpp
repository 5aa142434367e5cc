// voice_loop.hpp — the host's state of the voice loop, from the resample kernel up to complete Dry /
// RealOut / Wet buffers: the kernel variant, the device copies of the VoiceBook's lists, the parked
// lines, the filter state, the streaming queues and the three buses of parked lines (dry, RealOut,
// sends).  It decides in one place which kernels an update launches, on what grids.  Host code.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/b200mix.h"
#include "mixer_kernels.cuh"
#include "effect_kernels.cuh"
#include "panmix_tc.cuh"
#include "device_memory.hpp"
#include "launch.hpp"
#include "voice_book.hpp"

namespace b200mix {

class VoiceLoop {
public:
    // The kernels and their grids' limits, the partial rows, and what a parking device or one with
    // sends needs from its first update.  The dry and send gains are the device's (k_apply_updates
    // writes them).  `err`: the device's error string, which outlives the loop.
    int init(const b200mix_device_desc &dd, int num_sms, cudaStream_t stream, std::string &err,
        float *dry_cur, const float *dry_tgt, float *send_cur, const float *send_tgt)
    {
        dd_ = dd; num_sms_ = num_sms; s_ = stream; err_ = &err;
        CUDA_TRY(*err_, order_.alloc(dd.max_voices, s_));
        // non-HRTF devices with <= 4 dry channels mix the dry bus in registers; HRTF devices and
        // wider dry mixes resample + park (k_hrtf_fir mixes the HRTF voices, the parked dry bus
        // the others)
        const bool hrtfDev = dd.ir_size > 0;
        cdr_ = !hrtfDev && dd.dry_channels <= 4 ? 4 : 0;
        mix_fn_ = cdr_ ? k_mix_voices<kMixGS, kMixGroups, 4> : k_mix_voices<kMixGS, kMixGroups, 0>;
        mix_smem_ = (cdr_ ? sizeof(GroupSmem<4>) : sizeof(GroupSmem<0>))*kMixGroups;
        CUDA_TRY(*err_, cudaFuncSetAttribute(mix_fn_, cudaFuncAttributeMaxDynamicSharedMemorySize, int(mix_smem_)));
        int perSm = 0;
        CUDA_TRY(*err_, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, mix_fn_, kMixGS*kMixGroups, mix_smem_));
        mix_blocks_per_sm_ = std::max(perSm, 1);
        if(parks_dry())
        {
            // the parking variant writes every mixed voice's line and state bits
            if(int rc = ensure_park_lines()) return rc;
            CUDA_TRY(*err_, claim_.alloc(2, s_));
        }
        if(hrtfDev)
        {
            // 17 outputs per thread / 64 front pad for ir <= 64, 19 / 128 for ir <= 128
            fir_fn_ = dd.ir_size <= 64u ? k_hrtf_fir<17, 64> : k_hrtf_fir<19, 128>;
            fir_smem_ = (dd.ir_size <= 64u ? sizeof(FirSmem<kFirGS, 17, 64>) : sizeof(FirSmem<kFirGS, 19, 128>))*kFirGroups;
            CUDA_TRY(*err_, cudaFuncSetAttribute(fir_fn_, cudaFuncAttributeMaxDynamicSharedMemorySize, int(fir_smem_)));
            CUDA_TRY(*err_, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, fir_fn_, kFirGS*kFirGroups, fir_smem_));
            // the FIR grid sets the partial rows, hence the summation order: it is fixed at
            // kFirCtasPerSm per SM (the launch bounds), not at whatever more might fit
            fir_blocks_per_sm_ = std::max(std::min(perSm, kFirCtasPerSm), 1);
        }
        // partial rows: the FIR's HrtfAccumData rows (HRTF devices), or the register dry bus'
        // rows in two regions, k_mix_voices' and k_mix_deferred's (voices with direct filters)
        partial_floats_ = hrtfDev ? size_t(num_sms_)*fir_blocks_per_sm_*(2*kAccumLen)
            : size_t(num_sms_)*mix_blocks_per_sm_*size_t(cdr_)*kLine;
        CUDA_TRY(*err_, partial_.alloc(std::max<size_t>((hrtfDev ? 1 : 2)*partial_floats_, 4), s_));

        // a CTA's 8 warps share its entries evenly: chunks of 64 dry entries (128 per send slot) keep
        // the first (fading) tile's serial work per warp short
        dry_ = Bus{.cw = dd.dry_channels, .valid_bit = kSiDry, .per_chunk = 64, .max_chunks = 128, .cur = dry_cur, .tgt = dry_tgt};
        real_ = Bus{.cw = dd.real_channels, .valid_bit = kSiReal};
        sends_ = Bus{.cw = dd.wet_channels, .slots = dd.max_slots, .sends = dd.num_sends, .valid_bit = kSiSend,
            .per_chunk = 128, .max_chunks = 16, .cur = send_cur, .tgt = send_tgt};
        if(dd.max_slots && dd.wet_channels && dd.num_sends)
        {
            if(int rc = ensure_park_lines()) return rc;
            if(int rc = alloc(sends_, size_t(dd.max_voices)*dd.num_sends)) return rc;
        }
        return B200MIX_OK;
    }

    bool parks_dry() const { return cdr_ == 0; }       // no register dry bus: every mixed line is parked
    // Dry's rows the loop writes: the register dry bus sums 4 channels whatever the dry mix's width.
    uint32_t dry_rows() const { return std::max<uint32_t>(std::max(dd_.dry_channels, 1u), uint32_t(cdr_)); }
    // The partial rows and how many the last update's HRIR FIR stored (OutputStage::post sums them).
    const float *partial() const { return partial_; }
    uint32_t fir_rows() const { return fir_rows_; }
    // `launches` once the last update's k_hrtf_fir was launched; zeroed after work the count does not see.
    uint64_t &fir_done() { return fir_done_; }
    bool real_mixed() const { return real_mixed_; }   // the last update mixed the RealOut bus
    FilterRec *filt() const { return filt_; }

    // ---- parts allocated on first use: into locals, moved in once all succeeded (a failure changes nothing)

    // Storage of the parked dry bus (a parking device that meets a non-HRTF voice).
    int ensure_dry_bus()
    {
        if(dry_.entries) return B200MIX_OK;
        if(int rc = ensure_park_lines()) return rc;
        const bool wide = dd_.dry_channels > 4u && dd_.dry_channels <= uint32_t(kPmN);
        if(wide)
            CUDA_TRY(*err_, cudaFuncSetAttribute(k_panmix_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, kPmStages*kPmStageBytes + 1024));
        if(int rc = alloc(dry_, dd_.max_voices)) return rc;
        // B200MIX_PANMIX_SIMT=1 keeps the whole pan-mix on k_send_mix (A/B measurements only)
        const char *simt = std::getenv("B200MIX_PANMIX_SIMT");
        panmix_tc_ = wide && !(simt && simt[0] == '1');
        return B200MIX_OK;
    }

    // Storage of the RealOut bus (the first direct-channel voice), with the voices' RealOut gains.
    int ensure_real_bus()
    {
        if(real_.entries) return B200MIX_OK;
        if(int rc = ensure_park_lines()) return rc;
        const size_t gains = size_t(dd_.max_voices)*dd_.real_channels;
        DevArray<float> cur, tgt;
        CUDA_TRY(*err_, cur.alloc(gains, s_));
        CUDA_TRY(*err_, tgt.alloc(gains, s_));
        if(int rc = alloc(real_, dd_.max_voices)) return rc;
        real_.cur = cur; real_.tgt = tgt;
        real_cur_ = std::move(cur); real_tgt_ = std::move(tgt);
        return B200MIX_OK;
    }

    // Queue tables of the streaming voices (the first voice that reads a queue).
    int ensure_queues()
    {
        if(qhdr_) return B200MIX_OK;
        DevArray<uint4> qhdr; DevArray<uint32_t> queue;
        CUDA_TRY(*err_, qhdr.alloc(dd_.max_voices, s_));
        CUDA_TRY(*err_, queue.alloc(size_t(dd_.max_voices)*kMaxQueue, s_));
        qhdr_ = std::move(qhdr); queue_ = std::move(queue);
        return B200MIX_OK;
    }

    // Filter state of every voice path (the first filter a host or the GPU parameter stage sets).
    int ensure_filters(uint64_t &launches)
    {
        if(filt_) return B200MIX_OK;
        const size_t count = size_t(dd_.max_voices)*paths();
        if(int rc = ensure_park_lines()) return rc;
        DevArray<FilterRec> filt; DevArray<float> dline; DevArray<uint32_t> order2;
        CUDA_TRY(*err_, filt.alloc(count));
        CUDA_TRY(*err_, dline.alloc(size_t(dd_.max_voices)*kLine, s_));
        CUDA_TRY(*err_, order2.alloc(dd_.max_voices, s_));
        k_filter_init<<<unsigned((count*32u + 255u)/256u), 256, 0, s_>>>(filt, count);
        CUDA_TRY(*err_, cudaGetLastError());
        ++launches;
        filt_ = std::move(filt); dline_ = std::move(dline); order2_ = std::move(order2);
        return B200MIX_OK;
    }

    // k_apply_updates' pointers into the loop: filters, queues and the RealOut gains.
    void fill(ApplyParams &A) const
    {
        A.filt = filt_; A.filt_paths = paths(); A.qhdr = qhdr_;
        A.real_cur = real_cur_; A.real_tgt = real_tgt_; A.creal = dd_.real_channels;
    }

    // b200mix_voices_filters' updates, once ensure_filters has run.
    int set_filters(uint32_t n, const FilterUpdate *updates, uint64_t &launches)
    {
        CUDA_TRY(*err_, fstage_.wait());
        const size_t cap = std::max<size_t>(n, 2u*fstage_.capacity());
        CUDA_TRY(*err_, fstage_.reserve(n, cap, cap*sizeof(FilterUpdate), cap*sizeof(FilterUpdate), s_));
        fstage_.begin();
        const FilterUpdate *fupd = fstage_.pack(updates, n);
        CUDA_TRY(*err_, fstage_.ship(s_));
        k_apply_filter_updates<<<(2u*n + 127u)/128u, 128, 0, s_>>>(filt_, paths(), fupd, n);
        ++launches;
        CUDA_TRY(*err_, cudaGetLastError());
        return B200MIX_OK;
    }

    // b200mix_voice_queue's list of one voice.
    int set_queue(VoiceRec *voices, const QueueSet &Q, uint64_t &launches)
    {
        if(int rc = ensure_queues()) return rc;
        k_set_queue<<<1, 32, 0, s_>>>(voices, qhdr_, queue_, Q);
        ++launches;
        CUDA_TRY(*err_, cudaGetLastError());
        return B200MIX_OK;
    }

    // Step one of an update, before anything of it is on the stream: the book's lists are refreshed
    // and all the update needs is allocated.  A list the book rebuilt stays pending until launch()
    // has uploaded it, so an update that fails before then leaves it to the next.
    int prepare(VoiceBook &B, uint32_t frames, bool mix_sends)
    {
        mix_sends_ = mix_sends && sends_.entries;
        const VoiceBook::Rebuilt re = B.refresh(filt_ != nullptr, dry_.entries, mix_sends_);
        pending_ = {pending_.order || re.order, pending_.order2 || re.order2, pending_.dry || re.dry,
            pending_.sends || re.sends, pending_.real || re.real};
        real_mixed_ = !B.real_entries.empty();
        frames_ = frames;
        dry_.chunks = dry_.chunks_for(uint32_t(B.dry_entries.size()));
        sends_.chunks = sends_.chunks_for(B.max_slot_entries);
        const size_t numEntries = B.entries.size();
        if(dry_.entries && !B.dry_entries.empty())
            if(int rc = grow(dry_.partial, dry_.partial_floats())) return rc;
        if(mix_sends_ && filt_ && numEntries)
            if(int rc = grow(fscratch_, numEntries*kLine, std::max<size_t>(numEntries, 64)*kLine, true)) return rc;
        return mix_sends_ ? grow(sends_.partial, sends_.partial_floats()) : B200MIX_OK;
    }

    // Step two: the pending lists' uploads, then the launches.  P holds the caller's part (voice
    // records, buffers, tables, results, callback plan); mark(i) records stage mark i (1..5).
    template<typename Mark>
    int launch(MixParams P, const VoiceBook &B, float *dry, float *real, float *wet, uint64_t &launches,
        Mark &&mark)
    {
        if(pending_.order) { CUDA_TRY(*err_, b200mix::upload(order_, B.order, s_)); pending_.order = false; }
        if(pending_.order2) { CUDA_TRY(*err_, b200mix::upload(order2_, B.order2, s_)); pending_.order2 = false; }
        if(pending_.dry) { if(int rc = upload(dry_, B.dry_entries, nullptr)) return rc; pending_.dry = false; }
        if(pending_.sends) { if(int rc = upload(sends_, B.entries, &B.slot_start)) return rc; pending_.sends = false; }
        if(pending_.real && real_.entries)
        { if(int rc = upload(real_, B.real_entries, nullptr)) return rc; pending_.real = false; }

        const uint32_t numOrder = uint32_t(B.order.size()), numOrder2 = uint32_t(B.order2.size());
        const uint32_t maxBlocks = uint32_t(num_sms_*mix_blocks_per_sm_);
        const uint32_t blocks = std::max(1u, std::min(maxBlocks, (numOrder + kMixGroups - 1)/kMixGroups));
        P.partial = partial_; P.max_voices = std::max(B.voice_hi, 1u); P.frames = frames_;
        P.cd = dd_.dry_channels; P.num_sends = dd_.num_sends; P.order = order_; P.num_order = numOrder;
        P.xscratch = xscratch_; P.sendinfo = sendinfo_; P.filt = filt_; P.filt_paths = paths();
        P.qhdr = qhdr_; P.queue = queue_; P.claim = claim_; P.dline = dline_;
        mark(1);
        mix_fn_<<<blocks, kMixGS*kMixGroups, mix_smem_, s_>>>(P);
        ++launches;
        CUDA_TRY(*err_, cudaGetLastError());
        const uint64_t mixDone = launches;

        mark(2);
        // ---- voices with an active direct filter: filter the parked lines, then mix them ----
        uint32_t rows2 = 0;
        if(filt_ && numOrder2)
        {
            k_filters<<<(numOrder2 + 31u)/32u, 32, 0, s_>>>(FilterRunParams{.filt = filt_, .filt_paths = paths(),
                .sendinfo = sendinfo_, .direct_order = order2_, .num_direct = numOrder2, .xscratch = xscratch_,
                .dline = dline_, .frames = frames_});
            ++launches;
            if(!parks_dry())
            {
                // The grid is the number of partial rows, so it fixes the order in which the
                // deferred voices' sums are added: it follows the resample kernel's occupancy, as
                // the main pass's does, not this kernel's own.
                rows2 = std::max(1u, std::min(maxBlocks, (numOrder2 + kMixGroups - 1)/kMixGroups));
                MixParams P2 = P;
                P2.order = order2_; P2.num_order = numOrder2;
                P2.partial = partial_ + partial_floats_;
                P2.results = nullptr;
                k_mix_deferred<kMixGS, kMixGroups, 4><<<rows2, kMixGS*kMixGroups,
                    sizeof(DeferredSmem<kMixGroups, 4>), s_>>>(P2);
                ++launches;
            }
            CUDA_TRY(*err_, cudaGetLastError());
        }
        // the HRIR FIR's partial rows are summed by the HRTF post-process (OutputStage::post)
        fir_rows_ = 0;
        if(dd_.ir_size)
        {
            fir_rows_ = std::max(1u, std::min(uint32_t(num_sms_*fir_blocks_per_sm_), (numOrder + kFirGroups - 1)/kFirGroups));
            // straight behind the resample kernel (no direct filters in between), its set-up runs
            // under the resample kernel's last CTAs
            CUDA_TRY(*err_, launch_ex(s_, launches, launches == mixDone, fir_fn_, dim3(fir_rows_), dim3(kFirGS*kFirGroups),
                fir_smem_, P));
            fir_done_ = launches;
        }

        mark(3);
        // the register dry bus' two regions of rows
        const uint32_t len = uint32_t(cdr_)*kLine, rows[2] = {blocks, rows2};
        for(uint32_t r = 0;r < 2 && !parks_dry() && rows[r];++r, ++launches)
            k_reduce_rows<<<(len/4 + kReduceCols - 1)/kReduceCols, 1024, 0, s_>>>(partial_ + r*partial_floats_, rows[r],
                len, dry, 1);
        CUDA_TRY(*err_, cudaGetLastError());

        mark(4);
        // ---- parked dry bus: non-HRTF voices of the parking variant ----
        if(dry_.entries && !B.dry_entries.empty())
        {
            // Above 4 dry channels (third-order output) a full update's pan-mix past the gain fades
            // is a dense GEMM over the voices: samples 128..1023 go to the tensor cores
            // (k_panmix_tc), k_send_mix keeps the first tile with the fades
            const bool tc = panmix_tc_ && frames_ == uint32_t(kLine) && dry_.chunks > 1u;
            if(int rc = mix(dry_, dry, uint32_t(B.dry_entries.size()), tc, launches)) return rc;
        }
        // ---- RealOut bus: direct-channel voices (core/voice.cpp:947-963 with mDirect.Buffer = RealOut)
        // in index order, one pseudo slot of real_channels; RealOut is then (direct sum) + the
        // post-process' output, the reference's association ----
        if(real_mixed_)
            if(int rc = mix(real_, real, uint32_t(B.real_entries.size()), false, launches)) return rc;

        mark(5);
        // ---- aux sends (core/voice.cpp:967-980) ----
        if(mix_sends_)
        {
            const uint32_t numEntries = uint32_t(B.entries.size());
            if(filt_ && numEntries)
            {
                k_filters<<<(numEntries + 31u)/32u, 32, 0, s_>>>(FilterRunParams{.filt = filt_, .filt_paths = paths(),
                    .sendinfo = sendinfo_, .entries = sends_.entries, .num_entries = numEntries, .xscratch = xscratch_,
                    .fscratch = fscratch_, .frames = frames_});
                ++launches;
            }
            if(int rc = mix(sends_, wet, numEntries, false, launches)) return rc;
        }
        return B200MIX_OK;
    }

private:
    // A bus of parked lines into `slots` pseudo slots of `cw` channels, with Current / Target gains
    // [voice][sends][cw]; `valid_bit`: the sendinfo bit of a voice parked for it.
    struct Bus {
        uint32_t cw{0}, slots{1}, sends{1}, valid_bit{0};
        uint32_t per_chunk{1}, max_chunks{1};      // entries per chunk, chunks at most
        float *cur{nullptr}; const float *tgt{nullptr};
        DevArray<SendEntry> entries; DevArray<uint32_t> slot_start;   // [max entries], [slots + 1]
        DevArray<float> geff; DevArray<float4> gramp;                  // [max entries][cw]
        DevArray<float> partial;                                       // [chunks][slots][cw][1024]
        uint32_t chunks{1};                                            // this update's (prepare)

        // the chunks of a slot with `n` entries
        uint32_t chunks_for(uint32_t n) const { return std::max(1u, std::min(max_chunks, (n + per_chunk - 1u)/per_chunk)); }
        size_t partial_floats() const { return chunks > 1u ? size_t(chunks)*slots*cw*kLine : 0; }
    };

    uint32_t paths() const { return 1u + dd_.num_sends; }

    // Parked lines and state bits of every voice (the resample kernel writes them, buses and filters read them).
    int ensure_park_lines()
    {
        if(xscratch_) return B200MIX_OK;
        DevArray<float> xscratch; DevArray<uint32_t> sendinfo;
        CUDA_TRY(*err_, xscratch.alloc(size_t(dd_.max_voices)*kLine, s_));
        CUDA_TRY(*err_, sendinfo.alloc(dd_.max_voices, s_));
        xscratch_ = std::move(xscratch); sendinfo_ = std::move(sendinfo);
        return B200MIX_OK;
    }

    // The bus' entries, CSR and gain ramps for `count` entries (zeroed).
    int alloc(Bus &b, size_t count)
    {
        DevArray<SendEntry> entries; DevArray<uint32_t> slotStart; DevArray<float> geff; DevArray<float4> gramp;
        CUDA_TRY(*err_, entries.alloc(count, s_));
        CUDA_TRY(*err_, slotStart.alloc(b.slots + 1, s_));
        CUDA_TRY(*err_, geff.alloc(count*b.cw, s_));
        CUDA_TRY(*err_, gramp.alloc(count*b.cw, s_));
        b.entries = std::move(entries); b.slot_start = std::move(slotStart);
        b.geff = std::move(geff); b.gramp = std::move(gramp);
        return B200MIX_OK;
    }

    // Below `need` elements, `a` is replaced by max(count, need) (zeroed when `zero`) once they are
    // allocated and the stream is idle: the last update may still read the old array.
    template<typename T>
    int grow(DevArray<T> &a, size_t need, size_t count = 0, bool zero = false)
    {
        if(a.size() >= need) return B200MIX_OK;
        count = std::max(count, need);
        DevArray<T> next;
        CUDA_TRY(*err_, zero ? next.alloc(count, s_) : next.alloc(count));
        CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        a = std::move(next);
        return B200MIX_OK;
    }

    // A bus' entries and CSR: `slot_start`, or {0, entries} for a one-slot bus (pageable memory: the
    // entries' upload waits for its copy).
    int upload(Bus &b, const std::vector<SendEntry> &entries, const std::vector<uint32_t> *slot_start)
    {
        const uint32_t ss[2] = {0u, uint32_t(entries.size())};
        if(slot_start) CUDA_TRY(*err_, b200mix::upload(b.slot_start, *slot_start, s_));
        else CUDA_TRY(*err_, cudaMemcpyAsync(b.slot_start, ss, sizeof(ss), cudaMemcpyHostToDevice, s_));
        CUDA_TRY(*err_, b200mix::upload(b.entries, entries, s_));
        return B200MIX_OK;
    }

    // The bus' mix into `out`: gain ramps -> k_send_mix in b.chunks entry chunks (samples 128..1023 on
    // the tensor cores when `tc`) -> the chunks' rows summed -> Current gains advanced.  The dry and
    // RealOut buses read direct-filtered lines from dline, the sends send-filtered ones from fscratch.
    int mix(const Bus &b, float *out, uint32_t num_entries, bool tc, uint64_t &launches)
    {
        SendMixParams M{.slot_start = b.slot_start, .entries = b.entries, .sendinfo = sendinfo_, .xscratch = xscratch_,
            .send_cur = b.cur, .send_tgt = b.tgt, .wet = out, .frames = frames_, .cw = b.cw, .num_sends = b.sends,
            .valid_bit = b.valid_bit, .chunks = b.chunks, .partial = b.partial, .geff = b.geff, .gramp = b.gramp};
        if(b.valid_bit != kSiSend) M.dline = dline_ ? dline_.get() : xscratch_.get();
        else if(filt_ && num_entries) { M.filt = filt_; M.filt_paths = paths(); M.fscratch = fscratch_; }

        const uint32_t chunks = b.chunks, gainGrid = (num_entries*M.cw + 127)/128;
        if(num_entries) { k_send_gains_prepare<<<gainGrid, 128, 0, s_>>>(M, num_entries); ++launches; }
        const uint32_t tiles = tc ? 1u : (chunks > 1u ? uint32_t(kLine/128) : (M.frames + 127u)/128u);
        if(M.cw > 4u) k_send_mix<16><<<dim3(b.slots, tiles, chunks), 256, 0, s_>>>(M);
        else k_send_mix<4><<<dim3(b.slots, tiles, chunks), 256, 0, s_>>>(M);
        ++launches;
        // dline stays null until a direct filter is set: no sendinfo lookups per entry before then
        if(tc)
        {
            k_panmix_tc<<<chunks, 128, kPmStages*kPmStageBytes + 1024, s_>>>(PanMixTcParams{M.slot_start, M.entries,
                M.sendinfo, M.xscratch, dline_, M.geff, M.cw, chunks, M.partial});
            ++launches;
        }
        if(chunks > 1u)
        {
            const uint32_t len = b.slots*M.cw*kLine;
            if(chunks <= 16u)
                k_reduce_few<<<(len/4 + 255)/256, 256, 0, s_>>>(M.partial, chunks, len, M.wet, 1);
            else
                k_reduce_rows<<<(len/4 + kReduceCols - 1)/kReduceCols, 1024, 0, s_>>>(M.partial, chunks, len, M.wet, 1);
            ++launches;
        }
        if(num_entries) { k_send_gains_update<<<gainGrid, 128, 0, s_>>>(M, num_entries); ++launches; }
        CUDA_TRY(*err_, cudaGetLastError());
        return B200MIX_OK;
    }

    b200mix_device_desc dd_{};
    int num_sms_{0};
    cudaStream_t s_{nullptr};
    std::string *err_{nullptr};

    void (*mix_fn_)(const MixParams){nullptr};   // k_mix_voices<kMixGS, kMixGroups, cdr_>
    size_t mix_smem_{0}; int cdr_{0}; int mix_blocks_per_sm_{1};
    void (*fir_fn_)(const MixParams){nullptr};   // k_hrtf_fir of an HRTF device
    size_t fir_smem_{0}; int fir_blocks_per_sm_{0};
    DevArray<uint32_t> claim_;                   // voice claim counters of the parking k_mix_voices
    DevArray<float> partial_; size_t partial_floats_{0};
    uint32_t fir_rows_{0}; uint64_t fir_done_{0};

    DevArray<uint32_t> order_, order2_;          // book.order, book.order2
    DevArray<float> xscratch_; DevArray<uint32_t> sendinfo_;   // parked lines and state bits
    DevArray<FilterRec> filt_;                   // direct/send filters (the first filter set)
    UploadArena fstage_;                         // b200mix_voices_filters' inputs
    DevArray<float> dline_;                      // [max_voices][1024] filtered direct-path lines
    DevArray<float> fscratch_;                   // [send entries][1024] filtered send lines
    DevArray<uint4> qhdr_; DevArray<uint32_t> queue_;   // streaming queues
    Bus dry_, real_, sends_;                     // book.dry_entries, book.real_entries, book.entries
    DevArray<float> real_cur_, real_tgt_;        // [max_voices][real_channels] the RealOut bus' gains
    bool panmix_tc_{false};                      // wide dry buses: pan-mix past the fades on the tensor cores

    VoiceBook::Rebuilt pending_{};               // lists rebuilt and not uploaded yet
    uint32_t frames_{0}; bool mix_sends_{false}, real_mixed_{false};   // this update's (prepare)
};


} // namespace b200mix
