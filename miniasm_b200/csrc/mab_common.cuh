// mab_common.cuh -- shared device-side types and the per-GPU runtime object of miniasm_b200.
//
// Data layouts are byte-compatible with the reference's host structs so that one 128-bit load
// fetches an arc and two fetch a hit (SURVEY.md section 8a, rows a0-a3):
//   DHit  = ma_hit_t   (miniasm.h:29-34)   32 B: qns | qe tn | ts te | ml:31,rev:1 | bl:31,del:1
//   DSub  = ma_sub_t   (miniasm.h:38-40)    8 B: s:31,del:1 | e
//   DArc  = asg_arc_t  (asg.h:7-11)        16 B: ul = u<<32|len | v | ol:31,del:1
//   seq   = asg_seq_t  (asg.h:13-15)        4 B: len:31,del:1
//   idx   = asg_t::idx (asg.c:27-36)        8 B: first<<32 | count, one per oriented vertex
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <vector>

#define MAB_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
	fprintf(stderr, "[E::miniasm_b200] %s failed at %s:%d: %s\n", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); \
	exit(70); } } while (0)

struct __align__(16) DHit4 { uint32_t x, y, z, w; };

struct __align__(16) DHit {
	uint64_t qns;            // qid<<32 | qs
	uint32_t qe, tn;
	uint32_t ts, te;
	uint32_t ml_rev;         // ml:31 (low), rev:1 (bit 31)
	uint32_t bl_del;         // bl:31 (low), del:1 (bit 31)
};
static_assert(sizeof(DHit) == 32, "ma_hit_t layout");

struct __align__(8) DSub { uint32_t s_del; uint32_t e; }; // s:31 (low), del:1 (bit 31)
static_assert(sizeof(DSub) == 8, "ma_sub_t layout");

struct __align__(16) DArc {
	uint64_t ul;             // u<<32 | len
	uint32_t v;
	uint32_t ol_del;         // ol:31 (low), del:1 (bit 31)
};
static_assert(sizeof(DArc) == 16, "asg_arc_t layout");

#define MAB_DEL_BIT 0x80000000u

// ---------------------------------------------------------------------------------------------
// Per-GPU runtime: one stream, a stream-ordered allocator, a scratch area for CUB and a pinned
// mailbox for the few scalars (element counts) the host must see between passes.
// ---------------------------------------------------------------------------------------------
// Device memory arena: a few large cudaMalloc'd segments carved by a host-side first-fit free list with
// coalescing.  All work of a context runs on ONE stream, so a block can be handed out again as soon as it is
// freed on the host: any kernel that still uses it was launched earlier on the same stream.  After the first
// pass over a workload no driver allocation happens any more (cudaMallocAsync showed 100s of ms of jitter on
// multi-GB requests, see DESIGN.md "memory").
struct MabArena {
	struct Seg { char *base; size_t size; };
	std::vector<Seg> segs;
	std::map<char*, size_t> free_blk;    // start -> size, coalesced
	std::map<char*, size_t> live;        // start -> size
	size_t reserved = 0, in_use = 0, peak = 0;
	void *alloc(size_t bytes);
	void free(void *p);
	void release_all();
	bool segment_of(const void *p, char **base, size_t *offset) const // the cudaMalloc'd segment holding p (for CUDA IPC handles)
	{
		for (const Seg &s : segs)
			if ((const char*)p >= s.base && (const char*)p < s.base + s.size) { *base = s.base; *offset = (size_t)((const char*)p - s.base); return true; }
		return false;
	}
};

struct MabDev {
	int device = 0;
	MabArena arena;
	cudaStream_t stream = nullptr;
	cudaStream_t copy_stream = nullptr;     // created on first use: H2D chunks of mab_load_ingest_text overlap the kernels on `stream`
	void *cub_tmp = nullptr;
	size_t cub_tmp_bytes = 0;
	unsigned long long *d_scal = nullptr;   // 64 device scalars
	unsigned long long *h_scal = nullptr;   // pinned mirror
	uint64_t n_launch = 0;                  // our own kernels launched
	uint64_t n_lib = 0;                     // CUB device-wide calls issued
	// per-kernel timing registry (cudaEvent based, optional)
	bool profile = false;

	void init(int dev);
	void destroy();
	void *alloc(size_t bytes);
	void free(void *p);
	void *tmp(size_t bytes);                // grow-only scratch for CUB
	void zero_scal(int i, int n = 1);
	unsigned long long get_scal(int i);     // synchronises the stream
	void sync();
	void trace(const char *label);          // MAB_TRACE=1: synchronise and print the wall time since the previous trace point
	int trace_on = -1;
	double trace_t = 0;
};

// Streaming multiprocessors of the H100 SXM: the grid caps of the grid-stride kernels are multiples of it.
constexpr unsigned MAB_SMS = 132u;

template <typename T> static inline T *mab_alloc(MabDev &d, size_t n) { return (T*)d.alloc((n ? n : 1) * sizeof(T)); }

static inline unsigned mab_grid(size_t n, unsigned block, unsigned max_blocks = MAB_SMS * 32u)
{
	size_t g = (n + block - 1) / block;
	if (g < 1) g = 1;
	return (unsigned)(g < max_blocks ? g : max_blocks);
}

#define MAB_LAUNCH(dev, kern, grid, block, smem, ...) do { \
	kern<<<(grid), (block), (smem), (dev).stream>>>(__VA_ARGS__); \
	++(dev).n_launch; \
	MAB_CUDA(cudaGetLastError()); } while (0)

// scalar slots in MabDev::d_scal
enum { SC_COUNT = 0, SC_NSEL = 1, SC_BIG = 2, SC_AUX = 3, SC_AUX2 = 4, SC_MIN = 5, SC_TMP0 = 8 };
