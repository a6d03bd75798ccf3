// Host API of the carried collectives (device side: carry.cuh).  One queue per process (one process drives one GPU).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tb {

struct CarryArgs;

// Enqueue an all-gather (kind 1) or reduce-scatter (kind 2) job.  Pointer arrays are host arrays of `world` device
// addresses.  Returns a job id (> 0).  Jobs are executed in FIFO order by the GEMM launches that follow.
//   kind 1: src[r] = peer r's shard (bytes each), dst = local gathered buffer (shard r lands at dst + r * bytes)
//   kind 2: src[r] = peer r's flat buffer (world * bytes, this rank's slice at + rank * bytes), dst = output shard
long long carry_push(int kind, const uint64_t* src, uint64_t dst, const uint64_t* pads, long long bytes, int rank,
                     int world, int channel, uint32_t epoch, uint64_t block_counter, float scale, int in_bf16,
                     int out_fp32, int accumulate, uint64_t stats, int background, int entry_channel,
                     uint32_t entry_epoch);

// Publish `epoch` in this rank's ENTRY slot of `channel` on every peer's signal pad, ordered after the work already
// queued on `stream` ("the buffers jobs with this entry epoch read from me are final").
cudaError_t symm_signal(const uint64_t* pad_ptrs, int rank, int world, int channel, uint32_t epoch, cudaStream_t stream);

// Called by the GEMM launcher: move up to `flops * bytes_per_flop` bytes worth of pending chunks into `out`.
// Returns the number of slices filled (0 = nothing to carry).
int carry_take(double flops, CarryArgs* out);

// Host-only view of carry_take for tests of the queue logic (no kernel is launched; the taken chunks are CONSUMED):
// out[4 i .. 4 i + 3] = kind, chunk_begin, chunk_end, chunk_bytes of slice i.  Returns the number of slices.
int carry_take_probe(double flops, long long* out);

// Chunks not yet handed to a kernel, for all jobs (job_id == 0) or up to and including job `job_id`, in queue
// `queue` (0 foreground, 1 background, -1 both).
long long carry_pending(long long job_id, int queue);

// Run everything still queued up to and including `job_id` (0 = all) of `queue` as a stand-alone kernel on `stream`.
cudaError_t carry_flush(long long job_id, int queue, int num_sms, cudaStream_t stream);

// Bytes of NVLink traffic a GEMM carries per FLOP it executes (default 1.2e-4, not re-tuned for H100; TORCHACC_B200_CARRY_BYTES_PER_FLOP).
double carry_bytes_per_flop(double v);

// One-warp kernel: wait until every rank published `epoch` in the exit slots of `channel` (see carry.cuh).
cudaError_t symm_wait_done(const uint64_t* pad_ptrs, int rank, int world, int channel, uint32_t epoch,
                           cudaStream_t stream);

// Timing records of carrying GEMM launches (CTA 0's copy warp, globaltimer ns; layout: CarryArgs::debug).  Pass a
// device buffer of `records` x 8 u64 (nullptr disables); returns how many records the previous buffer received.
long long carry_set_debug(unsigned long long* buf, long long records);

// statistics: [0] chunks carried by GEMMs, [1] chunks flushed stand-alone, [2] GEMM launches that carried, [3] flushes
void carry_stats(long long* out4, int reset);

}  // namespace tb
