// TEST HARNESS ONLY — the per-instance kernels' frame and launch (ik_instance_launch.h) on the host. EmuFrame is one instance group's
// shared memory: the floats of the kernel's frame, carved by its own layout function, then a canary tail. A pass that writes past the
// frame changes the canary, and the emulator then fails instead of returning a result.
#pragma once
#include <cstring>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_instance_launch.h"
#include "emu_error.h"

// an InstanceLaunch as the emulator's launch entries return it: out = [W, groups per CTA, threads, smem bytes, staged point tables]
inline void launchWords(const mb2::InstanceLaunch& l, int64_t out[5]) {
  out[0] = l.warpsPerInstance; out[1] = l.groupsPerCta; out[2] = l.threads; out[3] = l.smemBytes; out[4] = l.stagedPoints;
}

struct EmuFrame {
  static constexpr size_t kCanaryFloats = 64;
  static constexpr uint32_t kCanaryBits = 0x7fc0c0deu; // a NaN payload no pass writes
  size_t floats;
  std::vector<float> buf = canaried(floats + kCanaryFloats);
  static std::vector<float> canaried(size_t n) {
    float c;
    std::memcpy(&c, &kCanaryBits, 4);
    return std::vector<float>(n, c);
  }
  float* at(size_t offset) { return buf.data() + offset; }
  // the region at `offset` after the kernel's copy of an instance's `count` input floats into it
  float* load(size_t offset, const float* src, size_t count) { return static_cast<float*>(std::memcpy(at(offset), src, count * 4)); }
  // MB2_OK when the canary is intact (compared bit for bit), else the emulator's error
  int check(const char* kernel) const {
    const std::vector<float> tail = canaried(kCanaryFloats);
    if (std::memcmp(buf.data() + floats, tail.data(), kCanaryFloats * 4) == 0) return MB2_OK;
    g_emuErr = std::string(kernel) + ": a pass wrote past the instance's shared-memory frame";
    return MB2_ERR_CUDA;
  }
};
