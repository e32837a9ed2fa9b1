// witness.cu — the device witness builder, one chip at a time: vgpu_witness_device builds all 14 + 2 traces with it, vgpu_diff_witness
// (diff.cu) builds and compares one chip at a time, so that it never holds a second whole witness.
#pragma once
#include "ctx.h"

struct VgVmLogs;
class VgWitnessBuilder {
  public:
    VgWitnessBuilder(vgpu_ctx* ctx, const VgVmLogs& L);
    ~VgWitnessBuilder();
    // uploads the logs (on the context's stream; the host logs must outlive the builder's last launch) and builds the short chips'
    // traces on the host (a few KB)
    int32_t start();
    // the global height of chip c's main trace (of its preprocessed trace too, for chips 1 and 12): known once start() returned
    uint64_t height(int c) const;
    // Chip c's main trace: of a chip whose rows are generated on the device (cpu, memory, add, sub, lt, bitwise), this rank's run of
    // rows (vg_trace_run: a row shard when split, vgpu_dmat_upload_rows' rule); of the others the whole trace, uploaded.
    int32_t main(int c, VgMat* out);
    // preprocessed trace w (0: program, 1: range), whole
    int32_t prep(int w, VgMat* out);

  private:
    struct Impl;
    std::unique_ptr<Impl> impl_;
};
