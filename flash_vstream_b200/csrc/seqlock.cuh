// seqlock.cuh — the sequence-counter protocol between one device-side writer and readers that may live in other processes
// (CUDA IPC) or on other GPUs (peer access), written once.  The counter is the first 64-bit word of a publication's header:
// odd while a write is in progress, even otherwise, and it only ever grows.
//
//   writer:  write_begin (one thread) -> barrier -> writes -> every writer thread fences, barrier -> header fields ->
//            write_end (the same one thread)
//   reader:  read_open (one thread) -> barrier -> copy -> every reader thread fences, barrier -> read_close
// A reader accepts its copy iff read_open and read_close returned the same even value.  The barriers are the caller's
// (a grid sync, or a block-group barrier inside a cooperative kernel): they are what makes "every write" / "every read"
// complete before the counter moves or is read again.
// Users: consolidate_kernel / snapshot_kernel (stream_kernels.cu, the LLaVA bank) and publish_kernel / snapshot_kernel
// (qwen_serve.cu, the Qwen2-VL memory).
#pragma once

namespace fvs {
namespace seqlock {

// seq becomes odd; readers that open from here on reject their copy
__device__ __forceinline__ void write_begin(unsigned long long* seq) {
  atomicAdd_system(seq, 1ull);
  __threadfence_system();
}

// seq becomes even again: every write of the bracket (and the header fields written by this thread) is visible before it
__device__ __forceinline__ void write_end(unsigned long long* seq) {
  __threadfence_system();
  atomicAdd_system(seq, 1ull);
}

// the sequence number before the copy; the fence orders it before every header / data read that follows
__device__ __forceinline__ unsigned long long read_open(const unsigned long long* seq) {
  const unsigned long long s = *reinterpret_cast<const volatile unsigned long long*>(seq);
  __threadfence_system();
  return s;
}

// the sequence number after the copy (call it behind a fence and a barrier over every reading thread)
__device__ __forceinline__ unsigned long long read_close(const unsigned long long* seq) {
  return *reinterpret_cast<const volatile unsigned long long*>(seq);
}

}  // namespace seqlock
}  // namespace fvs
