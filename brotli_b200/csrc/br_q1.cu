// br_q1.cu -- kernels and host orchestration of the quality-1 path (br_q1.h): a BATCH of
// independent streams goes through four launches, whatever its size.
//
//   k_q1_parse   persistent warps pull fragments from a queue (one 2^table_bits-entry table per warp)
//   k_q1_prep    one CTA per 128 KiB block
//   k_q1_chain   one thread per stream
//   k_q1_emit    one CTA per block
//   k_q1_pack    dense packing of the compressed streams for one device->host copy
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <functional>
#include <thread>
#include <vector>
#include "br_q1.h"
#include "br_q1_host.h"
#include "br_q1_plan.h"

__global__ void __launch_bounds__(128, 16) k_q1_parse(BrQ1 q) {
  const u32 slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int* table = q.tables + (size_t)slot * q.table_slot;
  for (;;) {
    u32 f = 0;
    if ((threadIdx.x & 31u) == 0) f = atomicAdd(q.counters, 1u);
    f = __shfl_sync(0xffffffffu, f, 0);
    if (f >= q.nfrags) return;
    br_q1_parse_fragment(q, f, table);
  }
}
// ---- on-chip variant: fragments of at most 64 KiB (BASELINE config 5 is 10 000 of them)
// One warp per CTA, one CTA per SM.  Shared memory: the 2^16-entry hash table as u16 positions (128 KiB) and the
// fragment's input (<= 64 KiB + slack), fetched by ONE TMA bulk copy (cp.async.bulk, completion on an mbarrier) while
// the warp zeroes the table.  Every probe of the trawl loop -- input bytes, table slot, candidate bytes -- is then a
// shared-memory access: no DRAM sector per probe, no table memset in HBM.
#define BR_Q1_SHM_TABLE (1u << 16)
#define BR_Q1_SHM_INPUT (65536u + 64u)
#define BR_Q1_SHM_BYTES (BR_Q1_SHM_TABLE * 2u + BR_Q1_SHM_INPUT + 16u)
__device__ __forceinline__ u32 br_smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(32, 1) k_q1_parse_shm(BrQ1 q) {
  extern __shared__ __align__(128) u8 shm[];
  u16* table = (u16*)shm;
  u8* buf = shm + BR_Q1_SHM_TABLE * 2u;
  unsigned long long* bar = (unsigned long long*)(buf + BR_Q1_SHM_INPUT);
  const u32 lane = threadIdx.x;
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(br_smem_addr(bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  u32 phase = 0;
  for (;;) {
    u32 f = 0;
    if (lane == 0) f = atomicAdd(q.counters, 1u);
    f = __shfl_sync(0xffffffffu, f, 0);
    if (f >= q.nfrags) return;
    const BrQ1Frag fr = q.frags[f];
    const BrQ1Stream& st = q.streams[fr.stream];
    // input bytes [fr.start & ~15, fr.start + fr.size + 16) rounded up to 16: behind every stream lie >= 16 bytes of slack
    const u32 a0 = fr.start & ~15u;
    u32 nbytes = (fr.start - a0) + fr.size + 16u;
    nbytes = (nbytes + 15u) & ~15u;
    if (lane == 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the previous fragment's reads are done (generic proxy)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(br_smem_addr(bar)), "r"(nbytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"(br_smem_addr(buf)), "l"(q.in + st.in_off + a0), "r"(nbytes), "r"(br_smem_addr(bar)) : "memory");
    }
    // zero the table while the copy is in flight (encode.c:156 GetHashTable)
    {
      uint4* t4 = (uint4*)table;
      const u32 n4 = (2u << fr.table_bits) >> 4;
      for (u32 i = lane; i < n4; i += 32) t4[i] = make_uint4(0, 0, 0, 0);
      if (n4 == 0) for (u32 i = lane; i < (1u << fr.table_bits); i += 32) table[i] = 0;
    }
    {
      u32 ok = 0;
      do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(ok) : "r"(br_smem_addr(bar)), "r"(phase) : "memory");
      } while (!ok);
      phase ^= 1u;
    }
    __syncwarp();
    br_q1_parse_fragment_shm(q, f, table, buf);
    __syncwarp();
  }
}
__global__ void __launch_bounds__(128) k_q1_prep(BrQ1 q) {
  __shared__ BrQ1Smem sm;
  br_q1_prep_block(q, blockIdx.x, &sm);
}
__global__ void k_q1_chain(BrQ1 q) {
  const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < q.nstreams) br_q1_chain_stream(q, s);
}
__global__ void __launch_bounds__(128) k_q1_emit(BrQ1 q) {
  __shared__ u32 scratch[8];
  br_q1_emit_block(q, blockIdx.x, scratch);
}
// dense offsets (16-aligned) of the compressed streams: one CTA, each thread owns a contiguous run of streams
__global__ void __launch_bounds__(1024) k_q1_offsets(BrQ1 q, u64* dense_off) {
  __shared__ u64 part[1024];
  const u32 per = (q.nstreams + blockDim.x - 1) / blockDim.x;
  const u32 a = threadIdx.x * per, b = a + per < q.nstreams ? a + per : q.nstreams;
  u64 sum = 0;
  for (u32 s = a; s < b; ++s) sum += (q.streams[s].out_bytes + 15u) & ~15u;
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    u64 o = 0;
    for (u32 t = 0; t < blockDim.x; ++t) { const u64 v = part[t]; part[t] = o; o += v; }
    dense_off[q.nstreams] = o;
  }
  __syncthreads();
  u64 o = part[threadIdx.x];
  for (u32 s = a; s < b; ++s) { dense_off[s] = o; o += (q.streams[s].out_bytes + 15u) & ~15u; }
}
__global__ void __launch_bounds__(256) k_q1_pack(BrQ1 q, const u64* dense_off, uint4* dense) {
  const u32 s = blockIdx.x;
  const uint4* src = (const uint4*)((const u8*)q.out + q.streams[s].out_off);
  uint4* dst = dense + (dense_off[s] >> 4);
  const u32 n = (q.streams[s].out_bytes + 15u) >> 4;
  for (u32 i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// device-resident batch: copy stream s from the caller's packed buffer to the pipeline's layout (16-byte aligned starts)
__global__ void __launch_bounds__(256) k_q1_gather(BrQ1 q, const u8* __restrict__ src, const u64* __restrict__ src_off, u8* dst) {
  const u32 s = blockIdx.x;
  const u8* a = src + src_off[s];
  u8* b = dst + q.streams[s].in_off;
  const u32 n = q.streams[s].size;
  if ((((size_t)a) & 15u) == 0) {
    const u32 nv = n >> 4;
    for (u32 i = threadIdx.x; i < nv; i += blockDim.x) ((uint4*)b)[i] = ((const uint4*)a)[i];
    for (u32 i = (nv << 4) + threadIdx.x; i < n; i += blockDim.x) b[i] = a[i];
  } else {
    for (u32 i = threadIdx.x; i < n; i += blockDim.x) b[i] = a[i];
  }
}

// ------------------------------------------------------------------ host
namespace {
struct Arena {
  void* p = nullptr; size_t cap = 0;
  bool need(size_t n) {
    if (n <= cap) return true;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 4096;
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); return false; }
    cap = want; return true;
  }
  ~Arena() { if (p) cudaFree(p); }
};
struct Pinned {
  void* p = nullptr; size_t cap = 0;
  bool need(size_t n) {
    if (n <= cap) return true;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 4096;
    if (cudaMallocHost(&p, want) != cudaSuccess) { cudaGetLastError(); return false; }
    cap = want; return true;
  }
  ~Pinned() { if (p) cudaFreeHost(p); }
};
}  // namespace

struct BrQ1Job {
  cudaStream_t st = nullptr;
  cudaEvent_t ev[6] = {};
  Arena in, out, dense, cmds, lits, streams, frags, blocks, codes, hdr, tables, counters, dense_off, log2;
  Pinned h_in, h_out, h_off;
  u32 log2_n = 0;
  int sm_count = 0;
  u32 warps_per_sm = 16, first_width = 32;   // tuning knobs (env BR_Q1_WARPS_PER_SM, BR_Q1_FIRST_WIDTH); 16: best of a sweep of warps per SM
  bool shm_ok = false;        // the device grants k_q1_parse_shm its shared memory
  int kernel_choice = 0;      // 0 / 1 global-memory tables, 2 on-chip tables whenever the fragments fit (env BR_Q1_KERNEL)
  BrQ1Stats stats = {};
};

extern "C" const double* br_host_log2_table(u32* n);   // br_host.cc

extern "C" void br_q1_job_destroy(BrQ1Job* j);
extern "C" BrQ1Job* br_q1_job_create(void) {
  BrQ1Job* j = new BrQ1Job();
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaStreamCreateWithFlags(&j->st, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError(); delete j; return nullptr;
  }
  cudaDeviceGetAttribute(&j->sm_count, cudaDevAttrMultiProcessorCount, dev);
  for (auto& e : j->ev) cudaEventCreate(&e);
  j->shm_ok = cudaFuncSetAttribute(k_q1_parse_shm, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BR_Q1_SHM_BYTES) == cudaSuccess;
  if (!j->shm_ok) cudaGetLastError();
  if (const char* e = getenv("BR_Q1_KERNEL")) j->kernel_choice = atoi(e);
  if (const char* e = getenv("BR_Q1_WARPS_PER_SM")) { int v = atoi(e); if (v >= 4 && v <= 64) j->warps_per_sm = (u32)v; }
  if (const char* e = getenv("BR_Q1_FIRST_WIDTH")) { int v = atoi(e); if (v >= 1 && v <= 32) j->first_width = (u32)v; }
  // bit_cost.c:18 needs FastLog2 of sampled counts only (<= 2^17 / 43): the first 4096 entries
  u32 n = 0; const double* h = br_host_log2_table(&n);
  j->log2_n = n < 4096 ? n : 4096;
  if (!j->log2.need((size_t)j->log2_n * 8)) { delete j; return nullptr; }
  // (a pageable-source cudaMemcpy may return before the DMA lands; the job's stream is non-blocking, so wait here)
  if (cudaMemcpy(j->log2.p, h, (size_t)j->log2_n * 8, cudaMemcpyHostToDevice) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    cudaGetLastError(); br_q1_job_destroy(j); return nullptr;
  }
  return j;
}
extern "C" void br_q1_job_destroy(BrQ1Job* j) {
  if (!j) return;
  for (auto& e : j->ev) if (e) cudaEventDestroy(e);
  if (j->st) cudaStreamDestroy(j->st);
  delete j;
}
extern "C" const BrQ1Stats* br_q1_job_stats(const BrQ1Job* j) { return &j->stats; }

static void run_threads(int threads, size_t count, const std::function<void(size_t, size_t)>& fn) {
  if (threads <= 1 || count < 64) { fn(0, count); return; }
  std::vector<std::thread> th;
  size_t per = (count + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    size_t a = (size_t)t * per, b = a + per < count ? a + per : count;
    if (a >= b) break;
    th.emplace_back([=, &fn] { fn(a, b); });
  }
  for (auto& t : th) t.join();
}

extern "C" int br_q1_compress_batch(BrQ1Job* j, int lgwin, size_t count, const uint8_t* const* in, const size_t* in_n,
                                    const size_t* const* calls, const size_t* ncalls, const BrQ1Packed* packed,
                                    uint8_t* const* out, size_t* out_n, int* ok, int threads, int with_header, int end_op,
                                    const uint32_t* start_bits, uint32_t* end_bit) {
  const bool inputs_on_device = packed != nullptr;
  if (!j || lgwin < 10 || lgwin > 24 || count == 0 || count > (1u << 24)) return 0;
  std::vector<BrQ1Stream> streams; std::vector<BrQ1Frag> frags; std::vector<BrQ1Block> blocks;
  streams.reserve(count);
  u64 in_off = 0, out_off = 0;
  u32 max_tb = 8;
  for (size_t s = 0; s < count; ++s) {
    if (in_n[s] > (1u << 28)) return 0;         // bit offsets of a stream are 32-bit
    br_q1_plan_stream(lgwin, (u32)s, in_off, out_off, in_n[s], calls ? calls[s] : nullptr, calls ? ncalls[s] : 0, streams, frags, blocks, with_header, end_op, start_bits ? start_bits[s] : 0u);
    in_off += (in_n[s] + 15 + 16) & ~(u64)15;   // >= 16 bytes of slack behind every stream (unaligned 8-byte loads)
    out_off += br_q1_stream_bound(frags, streams.back());
  }
  for (auto& f : frags) if (f.table_bits > max_tb) max_tb = f.table_bits;
  const u64 total_in = in_off, total_out = out_off;
  const u32 nfr = (u32)frags.size(), nbl = (u32)blocks.size();
  const u32 table_slot = 1u << max_tb;
  u32 nwarps = (u32)j->sm_count * j->warps_per_sm;
  if (nwarps > nfr) nwarps = nfr ? nfr : 1;
  nwarps = (nwarps + 3u) & ~3u;

  if (!j->in.need(total_in + 64) || !j->out.need(total_out + 64) || !j->dense.need(total_out + 64) ||
      !j->lits.need(total_in + 64) || !j->cmds.need(4 * total_in + 64) ||
      !j->streams.need(streams.size() * sizeof(BrQ1Stream)) || !j->frags.need((size_t)nfr * sizeof(BrQ1Frag) + 16) ||
      !j->blocks.need((size_t)nbl * sizeof(BrQ1Block) + 16) || !j->codes.need((size_t)nbl * sizeof(BrQ1Codes) + 16) ||
      !j->hdr.need((size_t)nbl * BR_Q1_HDR_WORDS * 4 + 16) || !j->tables.need((size_t)nwarps * table_slot * 4) ||
      !j->counters.need(64) || !j->dense_off.need((count + 1) * 8))
    return 0;
  cudaStream_t st = j->st;
  cudaEventRecord(j->ev[0], st);
  // ---- inputs
  if (inputs_on_device) {
    // the packed offsets ride in dense_off (rewritten by k_q1_offsets later, after the gather)
    cudaMemcpyAsync(j->dense_off.p, packed->in_off, count * 8, cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(j->in.p, 0, total_in + 64, st);
  } else {
    if (!j->h_in.need(total_in + 64)) return 0;
    u8* hp = (u8*)j->h_in.p;
    run_threads(threads, count, [&](size_t a, size_t b) {
      for (size_t s = a; s < b; ++s) if (in_n[s]) memcpy(hp + streams[s].in_off, in[s], in_n[s]);
    });
    cudaMemcpyAsync(j->in.p, hp, total_in, cudaMemcpyHostToDevice, st);
  }
  cudaMemcpyAsync(j->streams.p, streams.data(), streams.size() * sizeof(BrQ1Stream), cudaMemcpyHostToDevice, st);
  if (nfr) cudaMemcpyAsync(j->frags.p, frags.data(), (size_t)nfr * sizeof(BrQ1Frag), cudaMemcpyHostToDevice, st);
  if (nbl) cudaMemcpyAsync(j->blocks.p, blocks.data(), (size_t)nbl * sizeof(BrQ1Block), cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(j->counters.p, 0, 64, st);
  cudaMemsetAsync(j->out.p, 0, total_out + 64, st);

  BrQ1 q; memset(&q, 0, sizeof(q));
  q.in = (const u8*)j->in.p; q.out = (u32*)j->out.p; q.cmds = (u32*)j->cmds.p; q.lits = (u8*)j->lits.p;
  q.streams = (BrQ1Stream*)j->streams.p; q.frags = (BrQ1Frag*)j->frags.p; q.blocks = (BrQ1Block*)j->blocks.p;
  q.codes = (BrQ1Codes*)j->codes.p; q.hdr = (u32*)j->hdr.p; q.tables = (int*)j->tables.p; q.table_slot = table_slot;
  q.nstreams = (u32)count; q.nfrags = nfr; q.nblocks = nbl; q.counters = (u32*)j->counters.p;
  q.log2tab = (const double*)j->log2.p; q.log2tab_n = j->log2_n;
  q.first_width = j->first_width;

  if (inputs_on_device) k_q1_gather<<<(unsigned)count, 256, 0, st>>>(q, packed->d_in, (const u64*)j->dense_off.p, (u8*)j->in.p);
  cudaEventRecord(j->ev[1], st);
  u32 max_frag = 0;
  for (auto& f : frags) if (f.size > max_frag) max_frag = f.size;
  // table and input on chip when every fragment fits (<= 64 KiB) and there are enough of them to fill the SMs
  // The on-chip variant is bit-exact but slower on BASELINE config 5: with the 128 KiB table only ONE warp fits an SM,
  // every instruction latency of its dependent probe chain is exposed, and one latency-bound warp per SM loses to 16
  // warps per SM that hide each other's HBM round trips.  It stays selectable (BR_Q1_KERNEL=2); the default is the
  // global-table kernel.
  const bool on_chip = j->shm_ok && max_frag <= 65536u && j->kernel_choice == 2;
  if (nfr) {
    if (on_chip) {
      u32 ctas = nfr < (u32)j->sm_count ? nfr : (u32)j->sm_count;
      k_q1_parse_shm<<<ctas, 32, BR_Q1_SHM_BYTES, st>>>(q);
    } else k_q1_parse<<<nwarps / 4, 128, 0, st>>>(q);
  }
  cudaEventRecord(j->ev[2], st);
  if (nbl) k_q1_prep<<<nbl, 128, 0, st>>>(q);
  k_q1_chain<<<(unsigned)((count + 127) / 128), 128, 0, st>>>(q);
  if (nbl) k_q1_emit<<<nbl, 128, 0, st>>>(q);
  cudaEventRecord(j->ev[3], st);
  k_q1_offsets<<<1, 1024, 0, st>>>(q, (u64*)j->dense_off.p);
  k_q1_pack<<<(unsigned)count, 256, 0, st>>>(q, (const u64*)j->dense_off.p, (uint4*)j->dense.p);
  cudaEventRecord(j->ev[4], st);
  // ---- results
  if (!j->h_off.need((count + 1) * 8 + streams.size() * sizeof(BrQ1Stream))) return 0;
  u64* h_off = (u64*)j->h_off.p;
  BrQ1Stream* h_streams = (BrQ1Stream*)(h_off + count + 1);
  cudaMemcpyAsync(h_off, j->dense_off.p, (count + 1) * 8, cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(h_streams, j->streams.p, streams.size() * sizeof(BrQ1Stream), cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) { fprintf(stderr, "brotli_b200 q1: %s\n", cudaGetErrorString(cudaGetLastError())); return 0; }
  const u64 dense_bytes = h_off[count];
  size_t good = 0;
  if (inputs_on_device) {
    // device-resident variant: the dense packing goes to the caller's device buffer, offsets and sizes to the host
    if (dense_bytes > packed->out_cap) return 0;
    cudaMemcpyAsync(packed->d_out, j->dense.p, dense_bytes, cudaMemcpyDeviceToDevice, st);
    cudaEventRecord(j->ev[5], st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return 0;
    for (size_t s = 0; s < count; ++s) { packed->out_off[s] = h_off[s]; out_n[s] = h_streams[s].out_bytes; ok[s] = 1; ++good; }
    packed->out_off[count] = dense_bytes;
  } else {
    if (!j->h_out.need(dense_bytes + 64)) return 0;
    cudaMemcpyAsync(j->h_out.p, j->dense.p, dense_bytes, cudaMemcpyDeviceToHost, st);
    cudaEventRecord(j->ev[5], st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return 0;
    const u8* hp = (const u8*)j->h_out.p;
    std::vector<int> okv(count, 0);
    run_threads(threads, count, [&](size_t a, size_t b) {
      for (size_t s = a; s < b; ++s) {
        const size_t sz = h_streams[s].out_bytes;
        if (sz <= out_n[s]) { memcpy(out[s], hp + h_off[s], sz); out_n[s] = sz; okv[s] = 1; }
      }
    });
    for (size_t s = 0; s < count; ++s) { ok[s] = okv[s]; good += okv[s]; }
  }
  if (end_bit) for (size_t s = 0; s < count; ++s) end_bit[s] = h_streams[s].end_bit;
  BrQ1Stats& S = j->stats;
  cudaEventElapsedTime(&S.ms_h2d, j->ev[0], j->ev[1]);
  cudaEventElapsedTime(&S.ms_parse, j->ev[1], j->ev[2]);
  cudaEventElapsedTime(&S.ms_code, j->ev[2], j->ev[3]);
  cudaEventElapsedTime(&S.ms_pack, j->ev[3], j->ev[4]);
  cudaEventElapsedTime(&S.ms_d2h, j->ev[4], j->ev[5]);
  cudaEventElapsedTime(&S.ms_total, j->ev[0], j->ev[5]);
  S.streams = count; S.fragments = nfr; S.blocks = nbl; S.in_bytes = total_in; S.out_bytes = dense_bytes; S.launches = 6;
  return (int)(good == count);
}
