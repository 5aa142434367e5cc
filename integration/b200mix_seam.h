/* b200mix_seam.h — the seam a maintainer adds to OpenAL Soft to mix on an H100 through
 * libb200mix.so (include/b200mix.h).  Declared here, called from the patched places of
 * alc/alu.cpp (integration/alu_seam.patch), alc/effects/convolution.cpp
 * (integration/convolution_seam.patch) and core/device.cpp (integration/device_seam.patch),
 * implemented in b200mix_seam.cpp. */
#ifndef B200MIX_SEAM_H
#define B200MIX_SEAM_H

struct DeviceBase;
struct BufferStorage;

/* True when this device mixes on the GPU (ALSOFT_B200MIX=1 in the environment and
 * libb200mix.so could be loaded).  ProcessContexts then skips its voice loop and effect loop
 * (alc/alu.cpp:2201-2206, 2252-2256) — parameter updates still run on the host. */
bool b200seam_enabled(const DeviceBase *device /* may be null: the switch is process-wide */) noexcept;

/* Replaces the voice loop, the slot loop and DeviceBase::Process(mPostProcess) of
 * DeviceBase::renderSamples(unsigned) (alc/alu.cpp:2412-2443): snapshots the post-ALU voices
 * of the device's contexts into b200mix_voice_params, renders `samplesToDo` frames on the GPU
 * and leaves the result in RealOut.Buffer; positions and play states go back into the Voice
 * objects.  Limiter, distance compensation, dither and Write<T> stay the host's.  A failure
 * (CUDA error, unsupported configuration) disconnects the device (DeviceBase::handleDisconnect). */
void b200seam_render(DeviceBase *device, unsigned samplesToDo) noexcept;

/* Called at the top of ConvolutionState::deviceUpdate (alc/effects/convolution.cpp:318,
 * integration/convolution_seam.patch): the effect state objects are private to their source
 * files, so this is where the seam learns the impulse response a convolution slot was given.
 * No-op unless the seam is enabled. */
void b200seam_note_convolution(const void *state, const BufferStorage *buffer) noexcept;

/* Called from DeviceBase::~DeviceBase (core/device.cpp:18, integration/device_seam.patch): the
 * device's mixer, if it had one, is destroyed (b200mix_destroy) and its GPU memory released. */
void b200seam_device_closed(const DeviceBase *device) noexcept;

/* Called where UpdateDeviceParams has re-prepared every voice and re-initialized every effect
 * state (alc/alc.cpp:1908, integration/alc_seam.patch) — alcResetDeviceSOFT, or alcCreateContext
 * with an attribute list on a device that is already playing.  The next update builds a new mixer
 * from the reference's objects: positions are theirs, histories start clean like Voice::prepare's.
 * (Most resets also change something b200seam_render can see — channel counts, the decoder
 * objects — but one that re-creates the same configuration does not.) */
void b200seam_device_reset(const DeviceBase *device) noexcept;

#endif
