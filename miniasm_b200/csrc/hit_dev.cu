// hit_dev.cu -- stage (i) on the GPU: ma_hit_sort / ma_hit_sub / ma_hit_cut / ma_hit_flt / ma_sub_merge /
// ma_hit_contained / ma_sg_gen (hit.c:19-36,109-256; asm.c:9-39).  Hits are 32-byte records moved with
// two 128-bit accesses; the per-read interval tables (8 B/read) are gathered through L2.
#include "hit_dev.cuh"
#include "hit2arc.cuh"
#include <cub/cub.cuh>
#include <functional>

extern "C" int ma_verbose;              // hit.c prints its [M::fn::timestamp] lines only when ma_verbose >= 3
extern "C" const char *sys_timestamp(void);
#define ma_verbose_dev (mab_mute ? 0 : ma_verbose)

// Sharded runs: the counts in the [M::...] lines are per rank; the caller installs a hook that sums them over the ranks (a collective:
// every rank reaches every print site, muted or not).  Unset = single GPU, nothing to do.
thread_local MabCountHook mab_count_hook = nullptr;
thread_local void *mab_count_hook_ctx = nullptr;
static inline void sum_ranks(unsigned long long *v, int n) { if (mab_count_hook) mab_count_hook(mab_count_hook_ctx, v, n); }

__device__ __forceinline__ DHit ld_hit(const DHit *p)
{
	const uint4 *q = reinterpret_cast<const uint4*>(p);
	uint4 a = __ldg(q), b = __ldg(q + 1);
	DHit h;
	h.qns = (uint64_t)a.y << 32 | a.x; h.qe = a.z; h.tn = a.w;
	h.ts = b.x; h.te = b.y; h.ml_rev = b.z; h.bl_del = b.w;
	return h;
}
__device__ __forceinline__ DHit ld_hit_rw(const DHit *p) // for kernels that also store to the array
{
	const uint4 *q = reinterpret_cast<const uint4*>(p);
	uint4 a = q[0], b = q[1];
	DHit h;
	h.qns = (uint64_t)a.y << 32 | a.x; h.qe = a.z; h.tn = a.w;
	h.ts = b.x; h.te = b.y; h.ml_rev = b.z; h.bl_del = b.w;
	return h;
}
__device__ __forceinline__ void st_hit(DHit *p, const DHit &h)
{
	uint4 *q = reinterpret_cast<uint4*>(p);
	q[0] = make_uint4((uint32_t)h.qns, (uint32_t)(h.qns >> 32), h.qe, h.tn);
	q[1] = make_uint4(h.ts, h.te, h.ml_rev, h.bl_del);
}

static inline uint32_t bits_for(uint64_t x) { uint32_t b = 0; while (x) ++b, x >>= 1; return b ? b : 1; }

static void drop_bounds(MabDev &d, DHits &h) { d.free(h.grp); h.grp = nullptr; }
static void drop_selected(MabDev &d, DHits &h) { d.free(h.map); d.free(h.off); h.map = nullptr, h.off = nullptr; }

void dh_reserve(MabDev &d, DHits &h, size_t m)
{
	drop_bounds(d, h);                  // the caller refills the hits
	drop_selected(d, h);
	if (m <= h.m) return;
	DHit *na = mab_alloc<DHit>(d, m), *nb = mab_alloc<DHit>(d, m);
	if (h.n) MAB_CUDA(cudaMemcpyAsync(na, h.a, h.n * sizeof(DHit), cudaMemcpyDeviceToDevice, d.stream));
	d.free(h.a); d.free(h.a2);
	h.a = na, h.a2 = nb, h.m = m;
}

void dh_free(MabDev &d, DHits &h)
{
	d.free(h.a); d.free(h.a2); d.free(h.grp);
	drop_selected(d, h);
	h = DHits();
}

// ---------------------------------------------------------------------------------------------
// Stable compaction of hits by a byte flag array.  32-byte records move well below the copy bandwidth through the
// generic library selection, so the hit path has its own three-step compaction -- per-tile keep counts
// (flags only), a scan of the ~n/2048 tile counts, and a scatter in which every warp row reads 1 KB of contiguous
// records and writes them behind the tile's offset.  Order of the kept hits is the input order.
// ---------------------------------------------------------------------------------------------
constexpr int SEL_ROWS = 8, SEL_THREADS = 256, SEL_TILE = SEL_ROWS * SEL_THREADS;
static_assert(SEL_ROWS * (SEL_THREADS / 32) == 64, "k_sel_scatter scans exactly two counts per lane of one warp");

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_count(const uint8_t *__restrict__ flag, size_t n, uint32_t *__restrict__ tile_cnt, unsigned long long *__restrict__ total)
{
	__shared__ unsigned s_w[SEL_THREADS / 32];
	const size_t base = (size_t)blockIdx.x * SEL_TILE;
	unsigned c = 0;
	#pragma unroll
	for (int k = 0; k < SEL_ROWS; ++k) {
		const size_t i = base + (size_t)k * SEL_THREADS + threadIdx.x;
		c += (i < n && flag[i] != 0) ? 1u : 0u;
	}
	c = __reduce_add_sync(0xffffffffu, c);
	if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
	__syncthreads();
	if (threadIdx.x == 0) {
		unsigned t = 0;
		#pragma unroll
		for (int w = 0; w < SEL_THREADS / 32; ++w) t += s_w[w];
		tile_cnt[blockIdx.x] = t;
		if (t) atomicAdd(total, (unsigned long long)t);
	}
}

__global__ void __launch_bounds__(SEL_THREADS)
k_sel_scatter(const DHit *__restrict__ in, const uint8_t *__restrict__ flag, size_t n, const uint32_t *__restrict__ tile_off,
              DHit *__restrict__ out, unsigned long long *__restrict__ n_out)
{
	constexpr int NW = SEL_THREADS / 32;
	__shared__ uint32_t s_off[SEL_ROWS * NW];   // (row, warp) -> kept records of the tile before that warp row
	__shared__ uint32_t s_total;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const size_t base = (size_t)blockIdx.x * SEL_TILE;
	unsigned bal[SEL_ROWS];
	#pragma unroll
	for (int k = 0; k < SEL_ROWS; ++k) {
		const size_t i = base + (size_t)k * SEL_THREADS + tid;
		const bool f = i < n && flag[i] != 0;
		bal[k] = __ballot_sync(0xffffffffu, f);
		if (lane == 0) s_off[k * NW + warp] = __popc(bal[k]);
	}
	__syncthreads();
	if (warp == 0) { // exclusive scan of the SEL_ROWS * NW = 64 counts in record order, two per lane
		const uint32_t c0 = s_off[2 * lane], c1 = s_off[2 * lane + 1];
		uint32_t inc = c0 + c1;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
		const uint32_t exc = inc - (c0 + c1);
		s_off[2 * lane] = exc, s_off[2 * lane + 1] = exc + c0;
		if (lane == 31) s_total = inc;
	}
	__syncthreads();
	const uint32_t tbase = tile_off[blockIdx.x];
	#pragma unroll
	for (int k = 0; k < SEL_ROWS; ++k) {
		if (bal[k] >> lane & 1u) {
			const size_t i = base + (size_t)k * SEL_THREADS + tid;
			const uint32_t pos = tbase + s_off[k * NW + warp] + __popc(bal[k] & ((1u << lane) - 1u));
			st_hit(out + pos, ld_hit(in + i));
		}
	}
	if (blockIdx.x == gridDim.x - 1 && tid == 0) *n_out = (unsigned long long)tbase + s_total;
}

static size_t select_hits(MabDev &d, DHits &h, const uint8_t *flag)
{
	if (h.n == 0) return 0;
	if (h.n >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^32 hits on one GPU\n"); exit(73); }
	unsigned long long *d_n = d.d_scal + SC_NSEL;
	const uint32_t n_tile = (uint32_t)((h.n + SEL_TILE - 1) / SEL_TILE);
	uint32_t *cnt = mab_alloc<uint32_t>(d, n_tile), *off = mab_alloc<uint32_t>(d, n_tile);
	d.zero_scal(SC_NSEL);
	MAB_LAUNCH(d, k_sel_count, n_tile, SEL_THREADS, 0, flag, h.n, cnt, d_n);
	if ((size_t)d.get_scal(SC_NSEL) == h.n) { // every record stays (clean data: the common case of ma_hit_cut/flt): nothing to move
		d.free(cnt); d.free(off);
		return h.n;
	}
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, (int)n_tile, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, off, (int)n_tile, d.stream);
	++d.n_lib;
	MAB_LAUNCH(d, k_sel_scatter, n_tile, SEL_THREADS, 0, h.a, flag, h.n, off, h.a2, d_n);
	d.free(cnt); d.free(off);   // stream-ordered arena: reuse is ordered behind the kernels above
	size_t n = (size_t)d.get_scal(SC_NSEL);
	DHit *t = h.a; h.a = h.a2; h.a2 = t;
	h.n = n;
	drop_bounds(d, h);
	return n;
}

// Bitonic network over 32*M keys held in registers, element e = 32*m + lane: exchanges at distance j < 32 are lane
// shuffles, distances >= 32 pair two registers of the same lane -- no shared-memory traffic and none of the 2-way bank
// conflicts the strided pair indexing has in the shared-memory version.
template <int M, typename T>
__device__ __forceinline__ void warp_bitonic_regs(T (&v)[M], const int lane)
{
	#pragma unroll
	for (int k = 2; k <= 32 * M; k <<= 1) {
		#pragma unroll
		for (int j = k >> 1; j > 0; j >>= 1) {
			if (j >= 32) {
				#pragma unroll
				for (int m = 0; m < M; ++m) {
					const int pm = m ^ (j >> 5);
					if (pm > m) {
						const bool asc = ((32 * m) & k) == 0; // k >= 64 here: the lane bits do not reach it
						const T x = v[m], y = v[pm];
						const T lo = x < y ? x : y, hi = x < y ? y : x;
						v[m] = asc ? lo : hi, v[pm] = asc ? hi : lo;
					}
				}
			} else {
				const bool low = (lane & j) == 0;
				#pragma unroll
				for (int m = 0; m < M; ++m) {
					const T y = __shfl_xor_sync(0xffffffffu, v[m], j);
					const bool asc = ((32 * m + lane) & k) == 0;
					v[m] = (asc == low) == (v[m] < y) ? v[m] : y;
				}
			}
		}
	}
}

// ---------------------------------------------------------------------------------------------
// ma_hit_sort as a per-read bucket sort.  The number of reads is known and each read has ~100 hits, so the query-id part of
// the key is a counting sort (per-read counts -> exclusive scan -> every record scattered into its read's bucket with an
// atomic cursor) and the query-start part a small sort per bucket.  Inside a bucket every record has the same query id, so that
// half of qns carries an ordinal instead: a number that grows with the hit's input position (the position itself, or
// 2 * line + 1 for a mirrored hit in the fused ingest).  key = qs << 32 | ordinal is unique in its bucket, so sorting by it gives
// exactly the stable order by (qid, qs); the query id is written back when the sorted record is stored.
// Three tiers by bucket size, all reading h.a2's buckets and writing the sorted records to the same positions of h.a: a warp
// stages up to BKW_HITS records in shared memory and sorts (key, slot) pairs in registers; a CTA sorts up to BKC_HITS keys with
// a block merge sort (skewed sets: ~10 000 hits on each read of a hot locus) and stores every record at its key's rank; larger
// buckets go to a segmented device sort of their (key, slot) pairs, then a gather inside each bucket.  The bucket bounds become
// h.grp for ma_hit_sub.
// ---------------------------------------------------------------------------------------------
constexpr int BKW_WARPS = 4, BKW_HITS = 256;
constexpr int BKC_THREADS = 512, BKC_ITEMS = 32, BKC_HITS = BKC_THREADS * BKC_ITEMS;
typedef unsigned long long BKey;

// first 8 bytes of a bucket slot: qs, ordinal
__device__ __forceinline__ BKey bucket_key(uint2 w) { return (BKey)w.x << 32 | w.y; }

// the record of a bucket slot stored at dst as a hit of read q
__device__ __forceinline__ void bucket_put(DHit *dst, uint4 x, uint4 y, uint32_t q)
{
	x.y = q;
	uint4 *o = reinterpret_cast<uint4*>(dst);
	o[0] = x, o[1] = y;
}
__device__ __forceinline__ void bucket_put(DHit *dst, const DHit *src, uint32_t q)
{
	const uint4 *s = reinterpret_cast<const uint4*>(src);
	bucket_put(dst, __ldg(s), __ldg(s + 1), q);
}

__global__ void k_bucket_count(const DHit *a, size_t n, uint32_t *cnt)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		atomicAdd(&cnt[a[i].qns >> 32], 1u);
}

// every record into its read's bucket, with its input position as the ordinal
__global__ void k_bucket_fill(const DHit *__restrict__ a, size_t n, const uint32_t *__restrict__ first, uint32_t *cur, DHit *__restrict__ out)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		const uint4 *p = reinterpret_cast<const uint4*>(a + i);
		uint4 x = __ldg(p);
		const uint4 y = __ldg(p + 1);
		const uint32_t q = x.y;
		x.y = (uint32_t)i;
		uint4 *o = reinterpret_cast<uint4*>(out + first[q] + atomicAdd(&cur[q], 1u));
		o[0] = x, o[1] = y;
	}
}

// warp_bitonic_regs with a payload carried along each key.  The keys are distinct except the padding (~0), whose payloads
// may be duplicated and are never read.
template <int M>
__device__ __forceinline__ void warp_bitonic_pairs(BKey (&v)[M], uint32_t (&p)[M], const int lane)
{
	#pragma unroll
	for (int k = 2; k <= 32 * M; k <<= 1) {
		#pragma unroll
		for (int j = k >> 1; j > 0; j >>= 1) {
			if (j >= 32) {
				#pragma unroll
				for (int m = 0; m < M; ++m) {
					const int pm = m ^ (j >> 5);
					if (pm > m) {
						const bool asc = ((32 * m) & k) == 0; // k >= 64 here: the lane bits do not reach it
						if ((v[pm] < v[m]) == asc) {
							const BKey t = v[m]; v[m] = v[pm], v[pm] = t;
							const uint32_t u = p[m]; p[m] = p[pm], p[pm] = u;
						}
					}
				}
			} else {
				const bool low = (lane & j) == 0;
				#pragma unroll
				for (int m = 0; m < M; ++m) {
					const BKey y = __shfl_xor_sync(0xffffffffu, v[m], j);
					const uint32_t py = __shfl_xor_sync(0xffffffffu, p[m], j);
					const bool asc = ((32 * m + lane) & k) == 0;
					if ((asc == low) != (v[m] < y)) v[m] = y, p[m] = py;
				}
			}
		}
	}
}

// s = the bucket's cnt records staged in shared memory (two uint4 per record)
template <int M>
__device__ __forceinline__ void bucket_sort_regs(const uint4 *s, uint32_t cnt, uint32_t q, DHit *__restrict__ out, int lane)
{
	BKey v[M];
	uint32_t p[M];
	#pragma unroll
	for (int m = 0; m < M; ++m) {
		const uint32_t j = 32u * m + lane;
		v[m] = j < cnt ? bucket_key(*reinterpret_cast<const uint2*>(s + 2 * j)) : ~0ull, p[m] = j;
	}
	warp_bitonic_pairs<M>(v, p, lane);
	#pragma unroll
	for (int m = 0; m < M; ++m) {
		const uint32_t j = 32u * m + lane;
		if (j < cnt) bucket_put(out + j, s[2 * p[m]], s[2 * p[m] + 1], q);
	}
}

__global__ void __launch_bounds__(BKW_WARPS * 32)
k_bucket_warp(const DHit *__restrict__ a, const uint32_t *__restrict__ first, uint32_t n_seq,
              DHit *__restrict__ out, uint64_t *grp, uint32_t *big_list, unsigned long long *scal)
{
	__shared__ uint4 s_rec[BKW_WARPS][2 * BKW_HITS]; // one bucket's records per warp
	const int lane = threadIdx.x & 31;
	uint4 *s = s_rec[threadIdx.x >> 5];
	for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_seq; r += (gridDim.x * blockDim.x) >> 5) {
		const uint32_t f = first[r], e = first[r + 1], cnt = e - f;
		if (lane == 0) grp[r] = cnt ? (uint64_t)f << 32 | e : 0;
		if (cnt == 0) continue;
		if (cnt > BKW_HITS) { if (lane == 0) big_list[atomicAdd(scal + SC_BIG, 1ull)] = r; continue; }
		const uint4 *src = reinterpret_cast<const uint4*>(a + f);
		for (uint32_t u = lane; u < 2 * cnt; u += 32) s[u] = __ldg(src + u);
		__syncwarp();
		if (cnt <= 32) bucket_sort_regs<1>(s, cnt, r, out + f, lane);
		else if (cnt <= 64) bucket_sort_regs<2>(s, cnt, r, out + f, lane);
		else if (cnt <= 128) bucket_sort_regs<4>(s, cnt, r, out + f, lane);
		else bucket_sort_regs<8>(s, cnt, r, out + f, lane);
		__syncwarp(); // the next bucket overwrites the staged records
	}
}

struct BKeyLess { __device__ __forceinline__ bool operator()(const BKey &x, const BKey &y) const { return x < y; } };
typedef cub::BlockMergeSort<BKey, BKC_THREADS, BKC_ITEMS> BkcSort;
static_assert(sizeof(typename BkcSort::TempStorage) >= BKC_HITS * sizeof(BKey), "the sorted keys reuse the sort's storage");

// The keys are sorted alone (a slot payload would not fit the registers of 16 384 keys per CTA); the sorted keys then go to
// shared memory and every record finds its rank there by binary search: the keys are unique, so it finds exactly its own.
__global__ void __launch_bounds__(BKC_THREADS, 1)
k_bucket_cta(const DHit *__restrict__ a, const uint32_t *__restrict__ first, const uint32_t *__restrict__ big_list,
             uint32_t n_big, DHit *__restrict__ out, uint32_t *huge_list, unsigned long long *scal)
{
	extern __shared__ __align__(16) unsigned char bk_smem[];
	typename BkcSort::TempStorage &ts = *reinterpret_cast<typename BkcSort::TempStorage*>(bk_smem);
	BKey *s_key = reinterpret_cast<BKey*>(bk_smem);
	const uint32_t tid = threadIdx.x;
	for (uint32_t b = blockIdx.x; b < n_big; b += gridDim.x) {
		const uint32_t r = big_list[b], f = first[r], cnt = first[r + 1] - f;
		if (cnt > BKC_HITS) { if (tid == 0) huge_list[atomicAdd(scal + SC_AUX2, 1ull)] = r; continue; }
		BKey v[BKC_ITEMS];
		#pragma unroll
		for (int k = 0; k < BKC_ITEMS; ++k) { // padding sorts last
			const uint32_t j = k * BKC_THREADS + tid;
			v[k] = j < cnt ? bucket_key(__ldg(reinterpret_cast<const uint2*>(a + f + j))) : ~0ull;
		}
		BkcSort(ts).Sort(v, BKeyLess());
		__syncthreads(); // the sort's storage becomes the sorted key array
		#pragma unroll
		for (int k = 0; k < BKC_ITEMS; ++k) s_key[tid * BKC_ITEMS + k] = v[k]; // blocked: thread tid holds ranks tid * BKC_ITEMS + k
		__syncthreads();
		for (uint32_t j = tid; j < cnt; j += BKC_THREADS) {
			const uint4 *src = reinterpret_cast<const uint4*>(a + f + j);
			const uint4 x = __ldg(src), y = __ldg(src + 1);
			const BKey key = bucket_key(make_uint2(x.x, x.y));
			uint32_t lo = 0, n = cnt; // last rank whose key is <= key
			while (n > 1) { const uint32_t half = n >> 1; lo = s_key[lo + half] <= key ? lo + half : lo; n -= half; }
			bucket_put(out + f + lo, x, y, r);
		}
		__syncthreads(); // the storage is reused by the next bucket
	}
}

// Buckets beyond a CTA: their (key, slot) pairs are laid out bucket after bucket at off[b] (exclusive scan of the sizes).
__global__ void k_bucket_sizes(const uint32_t *list, uint32_t n, const uint32_t *first, uint32_t *sz)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x)
		sz[i] = i < n ? first[list[i] + 1] - first[list[i]] : 0;
}

__global__ void k_bucket_pairs(const DHit *__restrict__ a, const uint32_t *__restrict__ first, const uint32_t *list, uint32_t n,
                               const uint32_t *__restrict__ off, BKey *key, uint32_t *slot)
{
	for (uint32_t b = blockIdx.x; b < n; b += gridDim.x) {
		const uint32_t f = first[list[b]], cnt = first[list[b] + 1] - f, o = off[b];
		for (uint32_t j = threadIdx.x; j < cnt; j += blockDim.x)
			key[o + j] = bucket_key(__ldg(reinterpret_cast<const uint2*>(a + f + j))), slot[o + j] = j;
	}
}

__global__ void k_bucket_gather(const DHit *__restrict__ a, const uint32_t *__restrict__ first, const uint32_t *list, uint32_t n,
                                const uint32_t *__restrict__ off, const uint32_t *__restrict__ slot, DHit *__restrict__ out)
{
	for (uint32_t b = blockIdx.x; b < n; b += gridDim.x) {
		const uint32_t r = list[b], f = first[r], cnt = first[r + 1] - f, o = off[b];
		for (uint32_t j = threadIdx.x; j < cnt; j += blockDim.x) bucket_put(out + f + j, a + f + slot[o + j], r);
	}
}

void dh_bucket_first(MabDev &d, const uint32_t *cnt, uint32_t n_seq, uint32_t *first)
{
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, first, (int64_t)n_seq + 1, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, first, (int64_t)n_seq + 1, d.stream);
	++d.n_lib;
}

void dh_sort_buckets(MabDev &d, DHits &h, const uint32_t *first)
{
	drop_bounds(d, h);
	const uint32_t n_seq = h.n_seq;
	if (h.n == 0 || n_seq == 0) return;
	h.grp = mab_alloc<uint64_t>(d, n_seq);
	uint32_t *big = mab_alloc<uint32_t>(d, n_seq);
	d.zero_scal(SC_BIG);
	unsigned grid = (n_seq + BKW_WARPS - 1) / BKW_WARPS;
	if (grid > MAB_SMS * 32u) grid = MAB_SMS * 32u;
	MAB_LAUNCH(d, k_bucket_warp, grid, BKW_WARPS * 32, 0, h.a2, first, n_seq, h.a, h.grp, big, d.d_scal);
	const uint32_t n_big = (uint32_t)d.get_scal(SC_BIG);
	if (n_big) {
		const size_t smem = sizeof(typename BkcSort::TempStorage);
		MAB_CUDA(cudaFuncSetAttribute(k_bucket_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); // per device: set on every use
		uint32_t *huge = mab_alloc<uint32_t>(d, n_big);
		d.zero_scal(SC_AUX2);
		MAB_LAUNCH(d, k_bucket_cta, n_big < MAB_SMS ? n_big : MAB_SMS, BKC_THREADS, smem, h.a2, first, big, n_big, h.a, huge, d.d_scal);
		const uint32_t n_huge = (uint32_t)d.get_scal(SC_AUX2);
		if (n_huge) {
			uint32_t *sz = mab_alloc<uint32_t>(d, (size_t)n_huge + 1), *off = mab_alloc<uint32_t>(d, (size_t)n_huge + 1);
			MAB_LAUNCH(d, k_bucket_sizes, mab_grid((size_t)n_huge + 1, 128), 128, 0, huge, n_huge, first, sz);
			dh_bucket_first(d, sz, n_huge, off);
			uint32_t n_pair;
			MAB_CUDA(cudaMemcpyAsync(&n_pair, off + n_huge, 4, cudaMemcpyDeviceToHost, d.stream));
			d.sync();
			if (n_pair >= (1u << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 hits in reads of more than %d hits on one GPU\n", BKC_HITS); exit(73); }
			BKey *k0 = mab_alloc<BKey>(d, n_pair), *k1 = mab_alloc<BKey>(d, n_pair);
			uint32_t *s0 = mab_alloc<uint32_t>(d, n_pair), *s1 = mab_alloc<uint32_t>(d, n_pair);
			const unsigned g = n_huge < MAB_SMS * 4 ? n_huge : MAB_SMS * 4;
			MAB_LAUNCH(d, k_bucket_pairs, g, 256, 0, h.a2, first, huge, n_huge, off, k0, s0);
			size_t tb = 0;
			cub::DeviceSegmentedSort::SortPairs(nullptr, tb, k0, k1, s0, s1, (int)n_pair, (int)n_huge, off, off + 1, d.stream);
			void *tmp = d.tmp(tb);
			cub::DeviceSegmentedSort::SortPairs(tmp, tb, k0, k1, s0, s1, (int)n_pair, (int)n_huge, off, off + 1, d.stream);
			++d.n_lib;
			MAB_LAUNCH(d, k_bucket_gather, g, 256, 0, h.a2, first, huge, n_huge, off, s1, h.a);
			d.free(sz); d.free(off); d.free(k0); d.free(k1); d.free(s0); d.free(s1);
		}
		d.free(huge);
	}
	d.free(big);
}

void dh_sort(MabDev &d, DHits &h)
{
	drop_bounds(d, h);
	const uint32_t n_seq = h.n_seq;
	if (h.n == 0 || n_seq == 0) return;
	if (h.n >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^32 hits on one GPU\n"); exit(73); }
	uint32_t *cnt = mab_alloc<uint32_t>(d, (size_t)n_seq + 1), *first = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
	MAB_CUDA(cudaMemsetAsync(cnt, 0, ((size_t)n_seq + 1) * 4, d.stream));
	MAB_LAUNCH(d, k_bucket_count, mab_grid(h.n, 256), 256, 0, h.a, h.n, cnt);
	dh_bucket_first(d, cnt, n_seq, first);
	MAB_CUDA(cudaMemsetAsync(cnt, 0, (size_t)n_seq * 4, d.stream));   // the counts become the buckets' fill cursors
	MAB_LAUNCH(d, k_bucket_fill, mab_grid(h.n, 256), 256, 0, h.a, h.n, first, cnt, h.a2);
	dh_sort_buckets(d, h, first);
	d.free(cnt); d.free(first);
}

// ---------------------------------------------------------------------------------------------
// ma_hit_sub (hit.c:109-160)
//   group = maximal run of equal query id;  per group collect (qs+clip)<<1 and (qe-clip)<<1|1 of the hits
//   with tn != qid and ml >= bl*min_iden (float32) and qe > qs;  sort;  sweep the depth;  keep the FIRST
//   longest stretch with depth >= min_dp;  sub = {start-clip, end+clip} or del.
// GPU shape: every hit emits two 64-bit keys  qid<<33 | invalid<<32 | endpoint  (invalid keys sink to the
// end of their group), one device-wide radix sort orders all groups at once, then one warp per group
// sweeps its 2*count keys with a warp scan.
// ---------------------------------------------------------------------------------------------
// unsorted != null: set when the query ids do not ascend (the bounds are then meaningless)
__global__ void k_group_bounds(const DHit *a, size_t n, uint32_t *g32, unsigned long long *unsorted)
{
	bool bad = false;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		uint32_t q = (uint32_t)(a[i].qns >> 32), prev = i ? (uint32_t)(a[i - 1].qns >> 32) : 0;
		if (i == 0 || prev != q) g32[2 * (size_t)q + 1] = (uint32_t)i;
		if (i == n - 1 || (uint32_t)(a[i + 1].qns >> 32) != q) g32[2 * (size_t)q] = (uint32_t)(i + 1);
		bad |= i && prev > q;
	}
	if (bad && unsorted) *unsorted = 1ull;
}

// Slots at or past their read's bound (grp) are dead: dh_select leaves them behind the live hits of each bucket, still under
// the read's id, so they only turn into invalid keys.
__global__ void k_sub_keys(const DHit *a, size_t n, const uint64_t *__restrict__ grp, float min_iden, uint32_t clip, uint64_t *key)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		DHit h = ld_hit(a + i);
		uint32_t qid = (uint32_t)(h.qns >> 32);
		int ml = (int)(h.ml_rev & 0x7fffffffu), bl = (int)(h.bl_del & 0x7fffffffu);
		bool skip = i >= (uint32_t)grp[qid] || h.tn == qid || (float)ml < __fmul_rn((float)bl, min_iden);
		uint32_t qs = (uint32_t)h.qns + clip, qe = h.qe - clip;
		uint64_t base = (uint64_t)qid << 33;
		if (!skip && qe > qs) {
			key[2 * i] = base | (uint32_t)(qs << 1);
			key[2 * i + 1] = base | (uint32_t)(qe << 1 | 1);
		} else {
			key[2 * i] = key[2 * i + 1] = base | 1ull << 32;
		}
	}
}

__global__ void __launch_bounds__(256)
k_sub_sweep(const uint64_t *key, const uint64_t *grp, uint32_t n_seq, int min_dp, uint32_t clip, DSub *sub, unsigned long long *n_remained)
{
	const int lane = threadIdx.x & 31;
	const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
	unsigned remained = 0;
	for (uint32_t r = wid; r < n_seq; r += nw) {
		const uint64_t g = grp[r];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		if (end == 0) continue;                      // read heads no group: stays {0,0,del=0}
		const size_t k0 = 2 * (size_t)first;
		const uint32_t nk = 2 * (end - first);
		int depth = 0;
		uint32_t carry_start = 0;
		unsigned long long best = 0;                 // len<<32 | ~index  (max = longest, earliest on ties)
		uint32_t best_end = 0;
		for (uint32_t c = 0; c < nk; c += 32) {
			const uint32_t i = c + lane;
			uint64_t k = i < nk ? key[k0 + i] : (1ull << 32);
			const bool valid = !(k >> 32 & 1);
			const uint32_t pos = (uint32_t)k >> 1;
			int delta = valid ? ((k & 1) ? -1 : 1) : 0, dp = delta;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, dp, o); if (lane >= o) dp += t; }
			dp += depth;
			const int old = dp - delta;
			const bool up = valid && old < min_dp && dp >= min_dp;
			const bool down = valid && old >= min_dp && dp < min_dp;
			const unsigned upm = __ballot_sync(0xffffffffu, up);
			const unsigned below = upm & ((1u << lane) - 1);
			const int src = below ? 31 - __clz(below) : 0;
			uint32_t st = __shfl_sync(0xffffffffu, pos, src);
			if (!below) st = carry_start;
			unsigned long long cand = 0;
			if (down) cand = (unsigned long long)(pos - st) << 32 | (0xffffffffu - i);
			unsigned long long m = cand;
			#pragma unroll
			for (int o = 16; o; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, m, o); m = t > m ? t : m; }
			if (m > best && (m >> 32) != 0) {
				const unsigned who = __ballot_sync(0xffffffffu, down && cand == m);
				best = m;
				best_end = __shfl_sync(0xffffffffu, pos, __ffs(who) - 1);
			}
			if (upm) carry_start = __shfl_sync(0xffffffffu, pos, 31 - __clz(upm));
			depth = __shfl_sync(0xffffffffu, dp, 31);
		}
		if (lane == 0) {
			DSub s;
			uint32_t len = (uint32_t)(best >> 32);
			if (len > 0) {
				s.s_del = ((best_end - len) - clip) & 0x7fffffffu;
				s.e = best_end + clip;
				++remained;
			} else s.s_del = MAB_DEL_BIT, s.e = 0;
			sub[r] = s;
		}
	}
	if (lane == 0 && remained) atomicAdd(n_remained, (unsigned long long)remained);
}

// ---- shared-memory variant: one warp (<= SUBW_HITS hits) or one CTA (<= SUBC_HITS hits) per read ------------
// The endpoints of one read never leave the SM: load the group's hits (two 128-bit loads each), emit the keys into
// shared memory, sort them (the warp in registers), sweep the depth with the same warp scan as k_sub_sweep.  Only reads
// with more hits than a CTA can hold go through the device-wide sort above.
constexpr int SUBW_WARPS = 8;
constexpr int SUBW_HITS = 256;               // per warp: 512 keys = 2 KB
constexpr int SUBC_HITS = 16384;             // per CTA: 32768 keys = 128 KB of dynamic shared memory (a power of two: the bitonic network pads up to it)

// depth sweep over n sorted keys in shared memory by one warp; returns the interval through *out (lane 0 writes)
__device__ __forceinline__ bool sub_sweep_smem(const uint32_t *key, uint32_t n, int min_dp, uint32_t clip, DSub *out, int lane)
{
	int depth = 0;
	uint32_t carry_start = 0, best_end = 0;
	unsigned long long best = 0;
	for (uint32_t c = 0; c < n; c += 32) {
		const uint32_t i = c + lane;
		const bool valid = i < n;
		const uint32_t k = valid ? key[i] : 0, pos = k >> 1;
		int delta = valid ? ((k & 1) ? -1 : 1) : 0, dp = delta;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, dp, o); if (lane >= o) dp += t; }
		dp += depth;
		const int old = dp - delta;
		const bool up = valid && old < min_dp && dp >= min_dp;
		const bool down = valid && old >= min_dp && dp < min_dp;
		const unsigned upm = __ballot_sync(0xffffffffu, up);
		const unsigned below = upm & ((1u << lane) - 1);
		const int src = below ? 31 - __clz(below) : 0;
		uint32_t st = __shfl_sync(0xffffffffu, pos, src);
		if (!below) st = carry_start;
		if (__any_sync(0xffffffffu, down)) { // an interval closes in this chunk (a handful per read): longest, earliest on ties
			unsigned long long cand = 0;
			if (down) cand = (unsigned long long)(pos - st) << 32 | (0xffffffffu - i);
			unsigned long long m = cand;
			#pragma unroll
			for (int o = 16; o; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, m, o); m = t > m ? t : m; }
			if (m > best && (m >> 32) != 0) {
				const unsigned who = __ballot_sync(0xffffffffu, down && cand == m);
				best = m;
				best_end = __shfl_sync(0xffffffffu, pos, __ffs(who) - 1);
			}
		}
		if (upm) carry_start = __shfl_sync(0xffffffffu, pos, 31 - __clz(upm));
		depth = __shfl_sync(0xffffffffu, dp, 31);
	}
	const uint32_t len = (uint32_t)(best >> 32);
	if (lane == 0) {
		DSub s;
		if (len > 0) s.s_del = ((best_end - len) - clip) & 0x7fffffffu, s.e = best_end + clip;
		else s.s_del = MAB_DEL_BIT, s.e = 0;
		*out = s;
	}
	return len > 0;
}

__device__ __forceinline__ bool sub_hit_keys(const DHit &h, uint32_t qid, float min_iden, uint32_t clip, uint32_t *ks, uint32_t *ke)
{
	const int ml = (int)(h.ml_rev & 0x7fffffffu), bl = (int)(h.bl_del & 0x7fffffffu);
	if (h.tn == qid || (float)ml < __fmul_rn((float)bl, min_iden)) return false;
	const uint32_t qs = (uint32_t)h.qns + clip, qe = h.qe - clip;
	if (!(qe > qs)) return false;
	*ks = qs << 1, *ke = qe << 1 | 1;
	return true;
}

template <int M>
__device__ __forceinline__ void sub_sort_regs(uint32_t *key, const uint32_t n, const int lane)
{
	uint32_t v[M];
	#pragma unroll
	for (int m = 0; m < M; ++m) v[m] = 32u * m + lane < n ? key[32 * m + lane] : 0xffffffffu;
	warp_bitonic_regs<M>(v, lane);
	#pragma unroll
	for (int m = 0; m < M; ++m) key[32 * m + lane] = v[m];
}

__global__ void __launch_bounds__(SUBW_WARPS * 32)
k_sub_warp(const DHit *__restrict__ a, const uint64_t *__restrict__ grp, uint32_t n_seq, int min_dp, float min_iden, uint32_t clip,
           DSub *sub, uint32_t *big_list, unsigned long long *scal)
{
	__shared__ uint32_t s_key[SUBW_WARPS][2 * SUBW_HITS];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	uint32_t *key = s_key[warp];
	unsigned remained = 0;
	for (uint32_t r = blockIdx.x * SUBW_WARPS + warp; r < n_seq; r += gridDim.x * SUBW_WARPS) {
		const uint64_t g = grp[r];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		if (end == 0) continue;
		const uint32_t cnt = end - first;
		if (cnt > SUBW_HITS) { if (lane == 0) big_list[atomicAdd(scal + SC_BIG, 1ull)] = r; continue; }
		uint32_t n = 0; // keys emitted so far (uniform)
		for (uint32_t c = 0; c < cnt; c += 32) {
			uint32_t ks = 0, ke = 0;
			bool ok = false;
			if (c + lane < cnt) ok = sub_hit_keys(ld_hit(a + first + c + lane), r, min_iden, clip, &ks, &ke);
			const unsigned m = __ballot_sync(0xffffffffu, ok);
			if (ok) { const uint32_t p = n + 2 * __popc(m & ((1u << lane) - 1)); key[p] = ks, key[p + 1] = ke; }
			n += 2 * __popc(m);
		}
		uint32_t np = 32; while (np < n) np <<= 1;
		__syncwarp();
		switch (np) { // keys of the read sorted in registers (np is uniform across the warp)
			case 32: sub_sort_regs<1>(key, n, lane); break;
			case 64: sub_sort_regs<2>(key, n, lane); break;
			case 128: sub_sort_regs<4>(key, n, lane); break;
			case 256: sub_sort_regs<8>(key, n, lane); break;
			default: sub_sort_regs<16>(key, n, lane); break;
		}
		__syncwarp();
		remained += sub_sweep_smem(key, n, min_dp, clip, sub + r, lane);
		__syncwarp();
	}
	if (lane == 0 && remained) atomicAdd(scal + SC_COUNT, (unsigned long long)remained);
}

// Large groups (hot spots: thousands of hits on one read).  The depth sweep only depends on HOW MANY intervals start and end at
// every coordinate, so a read whose coordinates fit the counter array is not sorted at all: one pass counts starts / ends per
// coordinate (16 + 16 bits in one shared-memory word; a group has <= 16 384 hits), a block scan turns the counts into depths, and the
// up / down crossings of min_dp are read off per coordinate -- starts before ends at a coordinate, exactly the order of the sorted keys
// (hit.c:137-149).  O(hits + coordinates) instead of the 120-stage bitonic network over 32 768 keys, which is kept for reads whose
// coordinates reach 32 768 or beyond.
constexpr uint32_t SUBC_COORDS = 2 * SUBC_HITS;      // counters that fit the CTA's 128 KB

__device__ __forceinline__ bool sub_count_sweep(uint32_t *cnt, uint32_t n_coord, int min_dp, uint32_t clip, DSub *out)
{	// cnt[p] = starts(p) | ends(p) << 16; all 512 threads of the CTA; returns (to every thread) whether an interval was kept
	__shared__ int s_part[512];
	__shared__ uint32_t s_up[512];
	__shared__ unsigned long long s_best[512];
	const int tid = threadIdx.x;
	const uint32_t per = (n_coord + 511) / 512, p0 = tid * per, p1 = p0 + per < n_coord ? p0 + per : n_coord;
	int delta = 0;
	for (uint32_t p = p0; p < p1; ++p) { const uint32_t c = cnt[p]; delta += (int)(c & 0xffffu) - (int)(c >> 16); }
	s_part[tid] = delta;
	__syncthreads();
	for (int o = 1; o < 512; o <<= 1) { // inclusive scan of the per-thread depth changes
		const int t = tid >= o ? s_part[tid - o] : 0;
		__syncthreads();
		s_part[tid] += t;
		__syncthreads();
	}
	const int depth0 = s_part[tid] - delta;            // depth before coordinate p0
	uint32_t last_up = 0xffffffffu;                    // pass 1: the last coordinate of my range where the depth rises through min_dp
	{
		int dp = depth0;
		for (uint32_t p = p0; p < p1; ++p) {
			const uint32_t c = cnt[p];
			const int mid = dp + (int)(c & 0xffffu);
			if (dp < min_dp && mid >= min_dp) last_up = p;
			dp = mid - (int)(c >> 16);
		}
	}
	s_up[tid] = last_up;
	__syncthreads();
	for (int o = 1; o < 512; o <<= 1) { // "latest crossing at or before my range": positions ascend with the thread index, NONE = 0xffffffff
		const uint32_t t = tid >= o ? s_up[tid - o] : 0xffffffffu;
		__syncthreads();
		if (s_up[tid] == 0xffffffffu) s_up[tid] = t;
		__syncthreads();
	}
	uint32_t start = tid ? s_up[tid - 1] : 0xffffffffu; // the interval that is open when my range begins started here
	if (start == 0xffffffffu) start = 0;               // (the reference's `start` is 0 until the first crossing)
	unsigned long long best = 0;                       // pass 2: intervals closing in my range: longest, earliest on ties
	{
		int dp = depth0;
		for (uint32_t p = p0; p < p1; ++p) {
			const uint32_t c = cnt[p];
			const int mid = dp + (int)(c & 0xffffu);
			if (dp < min_dp && mid >= min_dp) start = p;
			dp = mid - (int)(c >> 16);
			if (mid >= min_dp && dp < min_dp) {
				const unsigned long long cand = (unsigned long long)(p - start) << 32 | (0xffffffffu - p);
				if ((cand >> 32) != 0 && cand > best) best = cand;
			}
		}
	}
	s_best[tid] = best;
	__syncthreads();
	for (int o = 256; o; o >>= 1) {
		if (tid < o && s_best[tid + o] > s_best[tid]) s_best[tid] = s_best[tid + o];
		__syncthreads();
	}
	best = s_best[0];
	const uint32_t len = (uint32_t)(best >> 32), end = 0xffffffffu - (uint32_t)best;
	if (tid == 0) {
		DSub sres;
		if (len > 0) sres.s_del = ((end - len) - clip) & 0x7fffffffu, sres.e = end + clip;
		else sres.s_del = MAB_DEL_BIT, sres.e = 0;
		*out = sres;
	}
	__syncthreads();
	return len > 0;
}

__global__ void __launch_bounds__(512)
k_sub_cta(const DHit *__restrict__ a, const uint64_t *__restrict__ grp, const uint32_t *__restrict__ big_list, uint32_t n_big,
          int min_dp, float min_iden, uint32_t clip, DSub *sub, uint32_t *huge_list, unsigned long long *scal)
{
	extern __shared__ uint32_t c_key[];
	__shared__ uint32_t s_n, s_max;
	const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
	for (uint32_t b = blockIdx.x; b < n_big; b += gridDim.x) {
		const uint32_t r = big_list[b];
		const uint64_t g = grp[r];
		const uint32_t first = (uint32_t)(g >> 32), cnt = (uint32_t)g - first;
		if (cnt > SUBC_HITS) { if (tid == 0) huge_list[atomicAdd(scal + SC_AUX2, 1ull)] = r; continue; }
		if (tid == 0) s_n = 0, s_max = 0;
		__syncthreads();
		{ // largest coordinate any kept hit of the group touches
			uint32_t mx = 0;
			for (uint32_t c = tid; c < cnt; c += nt) {
				uint32_t ks, ke;
				if (sub_hit_keys(ld_hit(a + first + c), r, min_iden, clip, &ks, &ke)) mx = (ke >> 1) > mx ? (ke >> 1) : mx;
			}
			mx = __reduce_max_sync(0xffffffffu, mx);
			if (lane == 0 && mx) atomicMax(&s_max, mx);
		}
		__syncthreads();
		if (s_max < SUBC_COORDS) { // counting sweep
			const uint32_t n_coord = s_max + 1;
			for (uint32_t i = tid; i < n_coord; i += nt) c_key[i] = 0;
			__syncthreads();
			for (uint32_t c = tid; c < cnt; c += nt) {
				uint32_t ks, ke;
				if (sub_hit_keys(ld_hit(a + first + c), r, min_iden, clip, &ks, &ke)) { atomicAdd(&c_key[ks >> 1], 1u); atomicAdd(&c_key[ke >> 1], 1u << 16); }
			}
			__syncthreads();
			const bool kept = sub_count_sweep(c_key, n_coord, min_dp, clip, sub + r);
			if (tid == 0 && kept) atomicAdd(scal + SC_COUNT, 1ull);
			__syncthreads();
			continue;
		}
		for (uint32_t c = tid; c < cnt; c += nt) {
			uint32_t ks, ke;
			if (sub_hit_keys(ld_hit(a + first + c), r, min_iden, clip, &ks, &ke)) { const uint32_t p = atomicAdd(&s_n, 2u); c_key[p] = ks, c_key[p + 1] = ke; }
		}
		__syncthreads();
		const uint32_t n = s_n;
		uint32_t np = 32; while (np < n) np <<= 1;
		for (uint32_t i = n + tid; i < np; i += nt) c_key[i] = 0xffffffffu;
		__syncthreads();
		for (uint32_t k = 2, lk = 1; k <= np; k <<= 1, ++lk)
			for (uint32_t lj = lk; lj-- > 0;) {
				const uint32_t j = 1u << lj;
				for (uint32_t t = tid; t < np / 2; t += nt) {
					const uint32_t lo = ((t >> lj) << (lj + 1)) | (t & (j - 1)), hi = lo + j;
					const uint32_t x = c_key[lo], y = c_key[hi];
					const bool asc = (lo & k) == 0;
					if ((x > y) == asc) c_key[lo] = y, c_key[hi] = x;
				}
				__syncthreads();
			}
		if (tid < 32) {
			const bool kept = sub_sweep_smem(c_key, n, min_dp, clip, sub + r, lane);
			if (lane == 0 && kept) atomicAdd(scal + SC_COUNT, 1ull);
		}
		__syncthreads();
	}
}

__global__ void k_sub_copy_listed(const uint32_t *list, uint32_t n, const DSub *from, DSub *to, unsigned long long *n_remained)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		to[list[i]] = from[list[i]];
		if (!(from[list[i]].s_del & MAB_DEL_BIT)) atomicAdd(n_remained, 1ull);
	}
}

static uint64_t dh_sub_global(MabDev &d, const DHits &h, int min_dp, float min_iden, int end_clip, DSub *sub_out, const uint64_t *grp);

// ma_hit_sub of the reads the warp tier listed (more than SUBW_HITS hits): a CTA each up to SUBC_HITS hits, the device-wide key
// sort beyond.  Adds the reads that keep an interval to d_scal[SC_COUNT]; d_scal[SC_AUX2] must be zero on entry.
static void sub_big_reads(MabDev &d, const DHits &h, const uint64_t *grp, const uint32_t *big, uint32_t n_big, int min_dp, float min_iden,
                          int end_clip, DSub *sub_out)
{
	const size_t smem = (size_t)SUBC_HITS * 2 * 4;
	MAB_CUDA(cudaFuncSetAttribute(k_sub_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); // per device: set on every use
	uint32_t *huge = mab_alloc<uint32_t>(d, n_big);
	MAB_LAUNCH(d, k_sub_cta, n_big < MAB_SMS * 2 ? n_big : MAB_SMS * 2, 512, smem, h.a, grp, big, n_big, min_dp, min_iden, (uint32_t)end_clip, sub_out, huge, d.d_scal);
	uint32_t n_huge = (uint32_t)d.get_scal(SC_AUX2);
	if (n_huge) { // reads with more hits than a CTA can sort: device-wide sort of everything, keep only their rows
		DSub *tmp = mab_alloc<DSub>(d, h.n_seq);
		unsigned long long saved = d.get_scal(SC_COUNT);
		dh_sub_global(d, h, min_dp, min_iden, end_clip, tmp, grp);
		MAB_CUDA(cudaMemcpyAsync(d.d_scal + SC_COUNT, &saved, 8, cudaMemcpyHostToDevice, d.stream));
		MAB_LAUNCH(d, k_sub_copy_listed, mab_grid(n_huge, 128), 128, 0, huge, n_huge, tmp, sub_out, d.d_scal + SC_COUNT);
		d.sync();
		d.free(tmp);
	}
	d.free(huge);
}

uint64_t dh_sub(MabDev &d, const DHits &h, int min_dp, float min_iden, int end_clip, DSub *sub_out)
{
	const uint32_t n_seq = h.n_seq;
	unsigned long long n_remained = 0;
	if (n_seq) MAB_CUDA(cudaMemsetAsync(sub_out, 0, (size_t)n_seq * sizeof(DSub), d.stream));
	if (h.n && n_seq) {
		if (h.n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 hits on one GPU\n"); exit(73); }
		uint64_t *grp = h.grp;              // the bounds the sort left, while no pass has moved the hits since
		if (!grp) {
			grp = mab_alloc<uint64_t>(d, n_seq);
			MAB_CUDA(cudaMemsetAsync(grp, 0, (size_t)n_seq * 8, d.stream));
			MAB_LAUNCH(d, k_group_bounds, mab_grid(h.n, 256), 256, 0, h.a, h.n, (uint32_t*)grp, nullptr);
		}
		uint32_t *big = mab_alloc<uint32_t>(d, n_seq);
		MAB_CUDA(cudaMemsetAsync(d.d_scal, 0, 8 * sizeof(unsigned long long), d.stream));
		unsigned grid = (n_seq + SUBW_WARPS - 1) / SUBW_WARPS;
		if (grid > MAB_SMS * 32u) grid = MAB_SMS * 32u;
		MAB_LAUNCH(d, k_sub_warp, grid, SUBW_WARPS * 32, 0, h.a, grp, n_seq, min_dp, min_iden, (uint32_t)end_clip, sub_out, big, d.d_scal);
		uint32_t n_big = (uint32_t)d.get_scal(SC_BIG);
		if (n_big) sub_big_reads(d, h, grp, big, n_big, min_dp, min_iden, end_clip, sub_out);
		n_remained = d.get_scal(SC_COUNT);
		if (grp != h.grp) d.free(grp);
		d.free(big);
	}
	sum_ranks(&n_remained, 1);          // a collective: every rank gets here, with or without hits
	if (ma_verbose_dev >= 3)
		fprintf(stderr, "[M::%s::%s] %ld query sequences remain after sub\n", "ma_hit_sub", sys_timestamp(), (long)n_remained);
	return n_remained;
}

static uint64_t dh_sub_global(MabDev &d, const DHits &h, int min_dp, float min_iden, int end_clip, DSub *sub_out, const uint64_t *grp)
{
	const uint32_t n_seq = h.n_seq;
	if (n_seq) MAB_CUDA(cudaMemsetAsync(sub_out, 0, (size_t)n_seq * sizeof(DSub), d.stream));
	if (h.n == 0 || n_seq == 0) return 0;
	if (h.n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 hits on one GPU\n"); exit(73); }
	size_t nk = 2 * h.n;
	uint64_t *ka = mab_alloc<uint64_t>(d, nk), *kb = mab_alloc<uint64_t>(d, nk);
	MAB_LAUNCH(d, k_sub_keys, mab_grid(h.n, 256), 256, 0, h.a, h.n, grp, min_iden, (uint32_t)end_clip, ka);
	cub::DoubleBuffer<uint64_t> dk(ka, kb);
	size_t tb = 0;
	int end_bit = 33 + (int)bits_for(n_seq - 1);
	cub::DeviceRadixSort::SortKeys(nullptr, tb, dk, (int64_t)nk, 0, end_bit, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceRadixSort::SortKeys(tmp, tb, dk, (int64_t)nk, 0, end_bit, d.stream);
	++d.n_lib;
	d.zero_scal(SC_COUNT);
	MAB_LAUNCH(d, k_sub_sweep, mab_grid((size_t)n_seq * 32, 256), 256, 0, dk.Current(), grp, n_seq, min_dp, (uint32_t)end_clip, sub_out, d.d_scal + SC_COUNT);
	uint64_t n_remained = d.get_scal(SC_COUNT);
	d.free(ka); d.free(kb);
	return n_remained;
}

// ma_hit_cut (hit.c:162-193): the clipping rule itself is mab_cut_hit in hit2arc.cuh (shared with the CPU-tier check of the
// conversion rules, tests/hostsim/hit_host.cpp)
__global__ void k_cut(DHit *a, size_t n, const DSub *__restrict__ reg, int min_span, uint8_t *flag)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		DHit p = ld_hit_rw(a + i);
		const bool keep = mab_cut_hit(p, reg[p.qns >> 32], reg[p.tn], min_span);
		if (keep) st_hit(a + i, p);
		flag[i] = keep;
	}
}

size_t dh_cut(MabDev &d, DHits &h, const DSub *reg, int min_span)
{
	if (h.n) {
		uint8_t *flag = mab_alloc<uint8_t>(d, h.n);
		MAB_LAUNCH(d, k_cut, mab_grid(h.n, 256), 256, 0, h.a, h.n, reg, min_span, flag);
		select_hits(d, h, flag);
		d.free(flag);
	}
	{ unsigned long long v[1] = { (unsigned long long)h.n }; sum_ranks(v, 1);
	  if (ma_verbose_dev >= 3) fprintf(stderr, "[M::%s::%s] %ld hits remain after cut\n", "ma_hit_cut", sys_timestamp(), (long)v[0]); }
	return h.n;
}

// ---------------------------------------------------------------------------------------------
// ma_hit_flt (hit.c:195-216)
// ---------------------------------------------------------------------------------------------
__global__ void k_flt(const DHit *a, size_t n, const DSub *__restrict__ sub, int max_hang, int min_ovlp, uint8_t *flag, unsigned long long *tot_dp)
{
	unsigned long long dp = 0;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		DHit h = ld_hit(a + i);
		uint32_t l;
		const bool keep = mab_flt_hit(h, sub[h.qns >> 32], sub[h.tn], max_hang, min_ovlp, &l);
		if (keep) dp += l;
		flag[i] = keep;
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long s = BR(ts).Sum(dp);
	if (threadIdx.x == 0 && s) atomicAdd(tot_dp, s);
}

__global__ void k_flt_len(const DHit *a, size_t n, const DSub *__restrict__ sub, unsigned long long *tot_len)
{
	unsigned long long len = 0;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		uint32_t q = (uint32_t)(a[i].qns >> 32);
		if (i == n - 1 || (uint32_t)(a[i + 1].qns >> 32) != q) len += sub[q].e - (sub[q].s_del & 0x7fffffffu);
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long s = BR(ts).Sum(len);
	if (threadIdx.x == 0 && s) atomicAdd(tot_len, s);
}

size_t dh_flt(MabDev &d, DHits &h, const DSub *sub, int max_hang, int min_ovlp, float *cov)
{
	unsigned long long tot_dp = 0, tot_len = 0;
	if (h.n) {
		uint8_t *flag = mab_alloc<uint8_t>(d, h.n);
		d.zero_scal(SC_AUX, 2);
		MAB_LAUNCH(d, k_flt, mab_grid(h.n, 256), 256, 0, h.a, h.n, sub, max_hang, min_ovlp, flag, d.d_scal + SC_AUX);
		select_hits(d, h, flag);
		d.free(flag);
		if (h.n) MAB_LAUNCH(d, k_flt_len, mab_grid(h.n, 256), 256, 0, h.a, h.n, sub, d.d_scal + SC_AUX2);
		tot_dp = d.get_scal(SC_AUX), tot_len = d.h_scal[SC_AUX2];
	}
	unsigned long long gv[3] = { tot_dp, tot_len, (unsigned long long)h.n };
	sum_ranks(gv, 3);
	*cov = (float)((double)gv[0] / gv[1]);
	if (ma_verbose_dev >= 3)
		fprintf(stderr, "[M::%s::%s] %ld hits remain after filtering; crude coverage after filtering: %.2f\n", "ma_hit_flt", sys_timestamp(), (long)gv[2], *cov);
	return h.n;
}

// ---------------------------------------------------------------------------------------------
// ma_sub_merge (hit.c:218-223): a.e = a.s + b.e; a.s += b.s  (31-bit s field; del of `a` is kept, del of `b` ignored)
// ---------------------------------------------------------------------------------------------
__global__ void k_sub_merge(uint32_t n, DSub *a, const DSub *b)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		DSub x = a[i], y = b[i];
		uint32_t s = x.s_del & 0x7fffffffu, del = x.s_del & MAB_DEL_BIT;
		x.e = s + y.e;
		x.s_del = ((s + (y.s_del & 0x7fffffffu)) & 0x7fffffffu) | del;
		a[i] = x;
	}
}

void dh_sub_merge(MabDev &d, uint32_t n_sub, DSub *a, const DSub *b)
{
	if (n_sub) MAB_LAUNCH(d, k_sub_merge, mab_grid(n_sub, 256), 256, 0, n_sub, a, b);
}

// ---------------------------------------------------------------------------------------------
// ma_hit_contained (hit.c:225-256)
// ---------------------------------------------------------------------------------------------
__global__ void k_cont_mark(const DHit *a, size_t n, DSub *sub, HitArcParams p, uint8_t *used)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		DHit h = ld_hit(a + i);
		const uint32_t q = (uint32_t)(h.qns >> 32), t = h.tn;
		const DSub sq = sub[q], st = sub[t];
		DArc tmp;
		// lengths use the 31-bit s field only, so concurrent del-bit updates by other threads cannot change them
		int r = mab_hit2arc(h, (int)(sq.e - (sq.s_del & 0x7fffffffu)), (int)(st.e - (st.s_del & 0x7fffffffu)), p.max_hang, p.int_frac, p.min_ovlp, &tmp);
		if (r == MAB_HT_QCONT) atomicOr(&sub[q].s_del, MAB_DEL_BIT);
		else if (r == MAB_HT_TCONT) atomicOr(&sub[t].s_del, MAB_DEL_BIT);
		used[q] = 1, used[t] = 1;                   // ma_hit_mark_unused: a read is "used" if any of the n hits names it
	}
}

__global__ void k_cont_keep(uint32_t n_seq, const DSub *sub, const uint8_t *used, const uint8_t *seq_del, uint32_t *keep)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_seq; i += gridDim.x * blockDim.x)
		keep[i] = used[i] && !(sub[i].s_del & MAB_DEL_BIT) && !(seq_del && seq_del[i]);
}

__global__ void k_cont_map(uint32_t n_seq, const uint32_t *keep, const uint32_t *excl, int32_t *map, const DSub *sub, DSub *sub_out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_seq; i += gridDim.x * blockDim.x) {
		if (keep[i]) { map[i] = (int32_t)excl[i]; sub_out[excl[i]] = sub[i]; }
		else map[i] = -1;
	}
}

__global__ void k_cont_apply(DHit *a, size_t n, const int32_t *__restrict__ map, uint8_t *flag)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		uint64_t qns = a[i].qns;
		int32_t qn = map[qns >> 32], tn = map[a[i].tn];
		bool keep = qn >= 0 && tn >= 0;
		if (keep) { a[i].qns = (uint64_t)(uint32_t)qn << 32 | (uint32_t)qns; a[i].tn = (uint32_t)tn; }
		flag[i] = keep;
	}
}

size_t dh_contained(MabDev &d, DHits &h, DSub *sub, const uint8_t *seq_del, const HitArcParams &p, int32_t *map_out)
{
	const uint32_t n_seq = h.n_seq;
	uint32_t n_new = 0;
	if (n_seq) {
		uint8_t *used = mab_alloc<uint8_t>(d, n_seq);
		uint32_t *keep = mab_alloc<uint32_t>(d, n_seq), *excl = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
		DSub *sub2 = mab_alloc<DSub>(d, n_seq);
		MAB_CUDA(cudaMemsetAsync(used, 0, n_seq, d.stream));
		if (h.n) MAB_LAUNCH(d, k_cont_mark, mab_grid(h.n, 256), 256, 0, h.a, h.n, sub, p, used);
		MAB_LAUNCH(d, k_cont_keep, mab_grid(n_seq, 256), 256, 0, n_seq, sub, used, seq_del, keep);
		size_t tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, keep, excl, (int)n_seq, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, keep, excl, (int)n_seq, d.stream);
		++d.n_lib;
		MAB_LAUNCH(d, k_cont_map, mab_grid(n_seq, 256), 256, 0, n_seq, keep, excl, map_out, sub, sub2);
		uint32_t last_keep, last_excl;
		MAB_CUDA(cudaMemcpyAsync(&last_keep, keep + n_seq - 1, 4, cudaMemcpyDeviceToHost, d.stream));
		MAB_CUDA(cudaMemcpyAsync(&last_excl, excl + n_seq - 1, 4, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		n_new = last_keep + last_excl;
		if (n_new) MAB_CUDA(cudaMemcpyAsync(sub, sub2, (size_t)n_new * sizeof(DSub), cudaMemcpyDeviceToDevice, d.stream));
		if (h.n) {
			uint8_t *flag = mab_alloc<uint8_t>(d, h.n);
			MAB_LAUNCH(d, k_cont_apply, mab_grid(h.n, 256), 256, 0, h.a, h.n, map_out, flag);
			select_hits(d, h, flag);
			d.free(flag);
		}
		d.free(used); d.free(keep); d.free(excl); d.free(sub2);
	}
	h.n_seq = n_new;
	drop_bounds(d, h);                  // reads renumbered
	unsigned long long n_hits = h.n;
	sum_ranks(&n_hits, 1);
	if (ma_verbose_dev >= 3)
		fprintf(stderr, "[M::%s::%s] %d sequences and %ld hits remain after containment removal\n", "ma_hit_contained", sys_timestamp(), n_new, (long)n_hits);
	return h.n;
}

// ---------------------------------------------------------------------------------------------
// dh_select: the default read selection as per-read passes over the sorted hit buckets.  Only the two cuts need another
// read's interval (the target's) and only the renumbering needs every read's containment flag; everything else is local to
// one query read.  So the hits stay in their buckets: each pass moves a read's surviving hits to the front of its bucket
// (in order: survivors only move down, behind everything the warp has loaded) and shrinks the bound in h.grp.  Dead slots keep
// their read's id.  A record is stored only when it moved or its cut changed it.  The renumbering leaves the survivors in
// their buckets (DHits::map): ma_sg_gen reads them there, and dh_hits_dense writes the dense, qid-ordered array the step
// functions would have left for the readers that need it.
// ---------------------------------------------------------------------------------------------
enum { SCS_CUT = SC_TMP0, SCS_DP, SCS_LEN, SCS_FLT, SCS_CUT2, SCS_NSEQ, SCS_NHITS }; // d_scal slots of dh_select's counters

__device__ __forceinline__ bool hit_clipped(const DHit &p, const DHit &o) { return p.qns != o.qns || p.qe != o.qe || p.ts != o.ts || p.te != o.te; }

// ma_hit_cut + ma_hit_flt with sub1 in one sweep, then ma_hit_sub with clip over the survivors (as k_sub_warp); one
// warp per read.  Reads with more than SUBW_HITS survivors go to big_list for the CTA tier.  A read left without hits keeps
// sub2 = {0,0}: ma_hit_sub never sees it.
__global__ void __launch_bounds__(SUBW_WARPS * 32)
k_sel_cut_flt_sub(DHit *a, uint64_t *grp, uint32_t n_seq, const DSub *__restrict__ sub1, int min_span, int max_hang, int min_ovlp,
                  int min_dp, float min_iden, uint32_t clip, DSub *sub2, uint32_t *big_list, unsigned long long *scal)
{
	__shared__ uint32_t s_key[SUBW_WARPS][2 * SUBW_HITS];
	__shared__ unsigned long long s_acc[3]; // per-read counters of the block (kept out of registers: the sort needs them)
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const unsigned lt = (1u << lane) - 1u;
	uint32_t *key = s_key[warp];
	unsigned long long dp = 0;
	unsigned n_cut = 0;
	if (threadIdx.x < 3) s_acc[threadIdx.x] = 0;
	__syncthreads();
	for (uint32_t r = blockIdx.x * SUBW_WARPS + warp; r < n_seq; r += gridDim.x * SUBW_WARPS) {
		const uint64_t g = grp[r];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		if (end == 0) continue;
		const DSub sq = sub1[r];
		uint32_t kept = 0, n = 0; // survivors and sub keys so far (uniform)
		for (uint32_t c = first; c < end; c += 32) {
			const uint32_t i = c + lane;
			DHit p;
			bool keep = false, dirty = false, key_ok = false;
			uint32_t ks = 0, ke = 0;
			if (i < end) {
				p = ld_hit_rw(a + i);
				const DHit o = p;
				const DSub st = sub1[p.tn];
				keep = mab_cut_hit(p, sq, st, min_span);
				if (keep) {
					++n_cut;
					uint32_t l;
					keep = mab_flt_hit(p, sq, st, max_hang, min_ovlp, &l);
					if (keep) {
						dp += l;
						dirty = hit_clipped(p, o);
						key_ok = sub_hit_keys(p, r, min_iden, clip, &ks, &ke);
					}
				}
			}
			const unsigned km = __ballot_sync(0xffffffffu, keep);
			const uint32_t dst = first + kept + __popc(km & lt);
			if (keep && (dst != i || dirty)) st_hit(a + dst, p);
			kept += __popc(km);
			const unsigned sm = __ballot_sync(0xffffffffu, key_ok);
			if (key_ok) { const uint32_t q = n + 2 * __popc(sm & lt); if (q < 2 * SUBW_HITS) key[q] = ks, key[q + 1] = ke; }
			n += 2 * __popc(sm);
		}
		if (lane == 0) grp[r] = kept ? (uint64_t)first << 32 | (first + kept) : 0;
		if (kept == 0) continue;
		if (lane == 0) atomicAdd(&s_acc[0], (unsigned long long)(sq.e - (sq.s_del & 0x7fffffffu))), atomicAdd(&s_acc[1], (unsigned long long)kept);
		if (kept > SUBW_HITS) { if (lane == 0) big_list[atomicAdd(scal + SC_BIG, 1ull)] = r; continue; }
		uint32_t np = 32; while (np < n) np <<= 1;
		__syncwarp();
		switch (np) {
			case 32: sub_sort_regs<1>(key, n, lane); break;
			case 64: sub_sort_regs<2>(key, n, lane); break;
			case 128: sub_sort_regs<4>(key, n, lane); break;
			case 256: sub_sort_regs<8>(key, n, lane); break;
			default: sub_sort_regs<16>(key, n, lane); break;
		}
		__syncwarp();
		if (sub_sweep_smem(key, n, min_dp, clip, sub2 + r, lane) && lane == 0) atomicAdd(&s_acc[2], 1ull);
		__syncwarp();
	}
	#pragma unroll
	for (int o = 16; o; o >>= 1) dp += __shfl_xor_sync(0xffffffffu, dp, o);
	n_cut = __reduce_add_sync(0xffffffffu, n_cut);
	if (lane == 0) {
		if (n_cut) atomicAdd(scal + SCS_CUT, (unsigned long long)n_cut);
		if (dp) atomicAdd(scal + SCS_DP, dp);
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		if (s_acc[0]) atomicAdd(scal + SCS_LEN, s_acc[0]);
		if (s_acc[1]) atomicAdd(scal + SCS_FLT, s_acc[1]);
		if (s_acc[2]) atomicAdd(scal + SC_COUNT, s_acc[2]);
	}
}

// second ma_hit_cut with sub2, then the flag pass of ma_hit_contained (as k_cont_mark) on the clipped hit: lengths from sub2 (the
// merged table's are the same), flags raised in the merged table sub; one warp per read.  tn_out[slot] = target of each surviving
// hit, for the count pass after the renumbering.
__global__ void __launch_bounds__(256)
k_sel_cut_cont(DHit *a, uint64_t *grp, uint32_t n_seq, const DSub *__restrict__ sub2, DSub *sub, int min_span, HitArcParams hp,
               uint8_t *used, uint32_t *tn_out, unsigned long long *n_cut)
{
	const int lane = threadIdx.x & 31;
	const unsigned lt = (1u << lane) - 1u;
	unsigned cut = 0;
	for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_seq; r += (gridDim.x * blockDim.x) >> 5) {
		const uint64_t g = grp[r];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		if (end == 0) continue;
		const DSub rq = sub2[r];
		uint32_t kept = 0;
		for (uint32_t c = first; c < end; c += 32) {
			const uint32_t i = c + lane;
			DHit p;
			bool keep = false, dirty = false;
			if (i < end) {
				p = ld_hit_rw(a + i);
				const DHit o = p;
				const DSub rt = sub2[p.tn];
				keep = mab_cut_hit(p, rq, rt, min_span);
				if (keep) {
					dirty = hit_clipped(p, o);
					DArc tmp;
					const int rr = mab_hit2arc(p, (int)(rq.e - rq.s_del), (int)(rt.e - rt.s_del), hp.max_hang, hp.int_frac, hp.min_ovlp, &tmp);
					if (rr == MAB_HT_QCONT) atomicOr(&sub[r].s_del, MAB_DEL_BIT);
					else if (rr == MAB_HT_TCONT) atomicOr(&sub[p.tn].s_del, MAB_DEL_BIT);
					used[p.tn] = 1;
				}
			}
			const unsigned km = __ballot_sync(0xffffffffu, keep);
			const uint32_t dst = first + kept + __popc(km & lt);
			if (keep) {
				if (dst != i || dirty) st_hit(a + dst, p);
				tn_out[dst] = p.tn;
			}
			kept += __popc(km);
		}
		if (lane == 0) {
			grp[r] = kept ? (uint64_t)first << 32 | (first + kept) : 0;
			if (kept) used[r] = 1, cut += kept;
		}
	}
	if (lane == 0 && cut) atomicAdd(n_cut, (unsigned long long)cut);
}

// hits of each kept read whose target is also kept, at the read's new id, and the read's bucket bounds in grp_out[new id] (a
// fresh array: other warps still read grp[r] of old ids r >= m)
__global__ void __launch_bounds__(256)
k_sel_final_count(const uint64_t *__restrict__ grp, const uint32_t *__restrict__ tn, const int32_t *__restrict__ map, uint32_t n_seq, uint32_t *cnt,
                  uint64_t *__restrict__ grp_out)
{
	const int lane = threadIdx.x & 31;
	for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_seq; r += (gridDim.x * blockDim.x) >> 5) {
		const int32_t m = map[r];
		if (m < 0) continue;
		const uint64_t g = grp[r];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		unsigned c = 0;
		if (end) for (uint32_t i = first + lane; i < end; i += 32) c += map[tn[i]] >= 0;
		c = __reduce_add_sync(0xffffffffu, c);
		if (lane == 0) cnt[m] = c, grp_out[m] = g;
	}
}

// A kept hit of read m (new id) read from its bucket, where it still carries the old ids: renumbered in registers.  false: its
// target was dropped, so the dense array does not hold it.
__device__ __forceinline__ bool sel_renumber(DHit &h, uint32_t m, const int32_t *__restrict__ map)
{
	const int32_t tn = map[h.tn];
	h.qns = (uint64_t)m << 32 | (uint32_t)h.qns, h.tn = (uint32_t)tn;
	return tn >= 0;
}

// renumber the kept hits of each kept read and write them densely at off[new id]; grp[new id] turns from the bucket bounds
// into the dense bounds
__global__ void __launch_bounds__(256)
k_sel_final_copy(const DHit *__restrict__ a, uint64_t *__restrict__ grp, const int32_t *__restrict__ map, uint32_t n_seq,
                 const uint32_t *__restrict__ off, DHit *__restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const unsigned lt = (1u << lane) - 1u;
	for (uint32_t m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < n_seq; m += (gridDim.x * blockDim.x) >> 5) {
		const uint64_t g = grp[m];
		const uint32_t end = (uint32_t)g, first = (uint32_t)(g >> 32);
		uint32_t o = off[m];
		if (end) for (uint32_t c = first; c < end; c += 32) {
			const uint32_t i = c + lane;
			DHit h;
			bool live = false;
			if (i < end) { h = ld_hit(a + i); live = sel_renumber(h, m, map); }
			const unsigned km = __ballot_sync(0xffffffffu, live);
			if (live) st_hit(out + o + __popc(km & lt), h);
			o += __popc(km);
		}
		__syncwarp(); // every lane has read grp[m]
		if (lane == 0) { const uint32_t s = off[m]; grp[m] = o > s ? (uint64_t)s << 32 | o : 0; }
	}
}

static unsigned warp_grid(uint32_t n_seq, unsigned warps_per_block)
{
	const unsigned g = (n_seq + warps_per_block - 1) / warps_per_block;
	return g < 1 ? 1 : g < MAB_SMS * 32u ? g : MAB_SMS * 32u;
}

static void exclusive_sum(MabDev &d, const uint32_t *in, uint32_t *out, size_t n)
{
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, (int64_t)n, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, in, out, (int64_t)n, d.stream);
	++d.n_lib;
}

void dh_hits_dense(MabDev &d, DHits &h)
{
	if (!h.map) return;
	if (h.n_seq) {
		MAB_LAUNCH(d, k_sel_final_copy, warp_grid(h.n_seq, 8), 256, 0, h.a, h.grp, h.map, h.n_seq, h.off, h.a2);
		DHit *t = h.a; h.a = h.a2; h.a2 = t;
	}
	drop_selected(d, h);
}

size_t dh_select(MabDev &d, DHits &h, DSub *sub, const SelectParams &o, int32_t *map_out, float *cov, const SelectHooks &hk)
{
	const uint32_t n_seq = h.n_seq;
	if (h.n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 hits on one GPU\n"); exit(73); }
	if (!h.grp) { // hits that did not come through the sort (mab_load_hits): the bounds of their runs
		h.grp = mab_alloc<uint64_t>(d, n_seq);
		MAB_CUDA(cudaMemsetAsync(h.grp, 0, (size_t)n_seq * 8, d.stream));
		if (h.n) MAB_LAUNCH(d, k_group_bounds, mab_grid(h.n, 256), 256, 0, h.a, h.n, (uint32_t*)h.grp, nullptr);
	}
	dh_sub(d, h, o.min_dp, o.min_iden, 0, sub);
	if (hk.sub_done) hk.sub_done(sub);
	d.trace("select:sub1");

	// ma_hit_cut + ma_hit_flt + ma_hit_sub (clip = min_span / 2)
	const int clip = o.min_span / 2;
	DSub *sub2 = mab_alloc<DSub>(d, n_seq);
	uint32_t *big = mab_alloc<uint32_t>(d, n_seq);
	MAB_CUDA(cudaMemsetAsync(sub2, 0, (size_t)n_seq * sizeof(DSub), d.stream));
	d.zero_scal(0, SCS_NHITS + 1);
	MAB_LAUNCH(d, k_sel_cut_flt_sub, warp_grid(n_seq, SUBW_WARPS), SUBW_WARPS * 32, 0, h.a, h.grp, n_seq, sub, o.min_span, o.flt_max_hang, o.flt_min_ovlp,
	           o.min_dp, o.min_iden, (uint32_t)clip, sub2, big, d.d_scal);
	const uint32_t n_big = (uint32_t)d.get_scal(SC_BIG);
	{
		unsigned long long gv[4] = { d.h_scal[SCS_DP], d.h_scal[SCS_LEN], d.h_scal[SCS_CUT], d.h_scal[SCS_FLT] };
		sum_ranks(gv, 4);
		*cov = (float)((double)gv[0] / gv[1]);
		if (ma_verbose_dev >= 3) {
			fprintf(stderr, "[M::%s::%s] %ld hits remain after cut\n", "ma_hit_cut", sys_timestamp(), (long)gv[2]);
			fprintf(stderr, "[M::%s::%s] %ld hits remain after filtering; crude coverage after filtering: %.2f\n", "ma_hit_flt", sys_timestamp(), (long)gv[3], *cov);
		}
	}
	if (hk.step3) hk.step3();
	if (n_big) sub_big_reads(d, h, h.grp, big, n_big, o.min_dp, o.min_iden, clip, sub2);
	d.free(big);
	{
		unsigned long long v[1] = { d.get_scal(SC_COUNT) };
		sum_ranks(v, 1);
		if (ma_verbose_dev >= 3) fprintf(stderr, "[M::%s::%s] %ld query sequences remain after sub\n", "ma_hit_sub", sys_timestamp(), (long)v[0]);
	}
	if (hk.sub_done) hk.sub_done(sub2);
	dh_sub_merge(d, n_seq, sub, sub2);
	d.trace("select:cut1+flt+sub2");

	// ma_hit_cut with sub2 + ma_hit_contained's flags; h.a2 is idle and holds the targets meanwhile
	uint8_t *used = mab_alloc<uint8_t>(d, n_seq);
	uint32_t *tn = reinterpret_cast<uint32_t*>(h.a2);
	MAB_CUDA(cudaMemsetAsync(used, 0, n_seq, d.stream));
	MAB_LAUNCH(d, k_sel_cut_cont, warp_grid(n_seq, 8), 256, 0, h.a, h.grp, n_seq, sub2, sub, o.min_span, o.cont, used, tn, d.d_scal + SCS_CUT2);
	if (hk.flags_done) hk.flags_done(sub, used, n_seq);

	// renumbering: keep flags -> new ids (sub2 is dead and takes the compacted table), then hit counts -> offsets; the kept hits
	// stay in their buckets
	uint32_t *keep = mab_alloc<uint32_t>(d, (size_t)n_seq + 1), *excl = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
	uint32_t *cnt = mab_alloc<uint32_t>(d, (size_t)n_seq + 1), *off = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
	int32_t *map = mab_alloc<int32_t>(d, n_seq);
	uint64_t *grp_new = mab_alloc<uint64_t>(d, n_seq);
	MAB_CUDA(cudaMemsetAsync(keep + n_seq, 0, 4, d.stream));
	MAB_CUDA(cudaMemsetAsync(cnt, 0, ((size_t)n_seq + 1) * 4, d.stream));
	MAB_LAUNCH(d, k_cont_keep, mab_grid(n_seq, 256), 256, 0, n_seq, sub, used, nullptr, keep);
	exclusive_sum(d, keep, excl, (size_t)n_seq + 1);   // excl[n_seq] = reads kept
	MAB_LAUNCH(d, k_cont_map, mab_grid(n_seq, 256), 256, 0, n_seq, keep, excl, map, sub, sub2);
	MAB_LAUNCH(d, k_sel_final_count, warp_grid(n_seq, 8), 256, 0, h.grp, tn, map, n_seq, cnt, grp_new); // cnt[0 ..< reads kept]
	exclusive_sum(d, cnt, off, (size_t)n_seq + 1);      // off[reads kept ..= n_seq] = hits kept
	MAB_CUDA(cudaMemcpyAsync(d.d_scal + SCS_NSEQ, excl + n_seq, 4, cudaMemcpyDeviceToDevice, d.stream)); // low halves of zeroed slots
	MAB_CUDA(cudaMemcpyAsync(d.d_scal + SCS_NHITS, off + n_seq, 4, cudaMemcpyDeviceToDevice, d.stream));
	if (n_seq) MAB_CUDA(cudaMemcpyAsync(map_out, map, (size_t)n_seq * 4, cudaMemcpyDeviceToDevice, d.stream));
	const uint32_t n_new = (uint32_t)d.get_scal(SCS_NSEQ);
	const size_t n_hits = (size_t)d.h_scal[SCS_NHITS];
	const unsigned long long n_cut2 = d.h_scal[SCS_CUT2];
	if (n_new) MAB_CUDA(cudaMemcpyAsync(sub, sub2, (size_t)n_new * sizeof(DSub), cudaMemcpyDeviceToDevice, d.stream));
	d.free(sub2); d.free(used); d.free(keep); d.free(excl); d.free(cnt);
	h.n = n_hits, h.n_seq = n_new;
	d.free(h.grp);
	h.grp = grp_new, h.map = map, h.off = off;
	d.trace("select:cut2+contained");

	unsigned long long gv[2] = { n_cut2, (unsigned long long)h.n };
	sum_ranks(gv, 2);
	if (ma_verbose_dev >= 3) {
		fprintf(stderr, "[M::%s::%s] %ld hits remain after cut\n", "ma_hit_cut", sys_timestamp(), (long)gv[0]);
		fprintf(stderr, "[M::%s::%s] %d sequences and %ld hits remain after containment removal\n", "ma_hit_contained", sys_timestamp(), n_new, (long)gv[1]);
	}
	return h.n;
}

// ---------------------------------------------------------------------------------------------
// ma_sg_gen (asm.c:9-39)
// ---------------------------------------------------------------------------------------------
__global__ void k_seq_set(uint32_t n_seq, const uint32_t *len, const uint8_t *del, uint32_t *seq, unsigned *max_len)
{
	unsigned mx = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_seq; i += gridDim.x * blockDim.x) {
		uint32_t l = len[i] & 0x7fffffffu;
		seq[i] = l | (del && del[i] ? MAB_DEL_BIT : 0);
		mx = l > mx ? l : mx;
	}
	mx = __reduce_max_sync(0xffffffffu, mx);
	if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_len, mx);
}

// one (key, value) column pair per hit: key = u << lb | len (or the sentinel 1 << (lb + vertex bits) when the hit yields no arc),
// value = ol:del << 32 | v.  Sorting the columns (stable) and dropping the sentinels equals asg.c's append + sort.  len32: the
// 32-bit read lengths ma_hit2arc takes (asm.c:23-24).  An arc of 2^lb or more raises *ovf; the caller then redoes the columns
// with lb = 32.
__global__ void k_sg_arcs(const DHit *a, size_t n, const uint32_t *len32, uint32_t *seq, HitArcParams p, uint32_t lb, uint64_t sentinel, uint64_t *key, uint64_t *val,
                          unsigned long long *n_emit, unsigned long long *ovf)
{
	unsigned cnt = 0;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
		DHit h = ld_hit(a + i);
		const uint32_t qn = (uint32_t)(h.qns >> 32);
		DArc t;
		t.ul = 0, t.v = 0, t.ol_del = 0;
		int r = mab_hit2arc(h, (int)len32[qn], (int)len32[h.tn], p.max_hang, p.int_frac, p.min_ovlp, &t);
		bool emit = false;
		if (r >= 0) {
			if (qn == h.tn) { // self match: only the palindromic artefact has an effect (asm.c:27-31)
				if ((uint32_t)h.qns == h.ts && h.qe == h.te && (h.ml_rev >> 31)) atomicOr(&seq[qn], MAB_DEL_BIT);
			} else emit = true;
		} else if (r == MAB_HT_QCONT) atomicOr(&seq[qn], MAB_DEL_BIT);
		if (emit && lb < 32 && (uint32_t)t.ul >> lb) *ovf = 1;
		key[i] = emit ? ((t.ul >> 32) << lb | (uint32_t)t.ul) : sentinel;
		val[i] = (uint64_t)t.ol_del << 32 | t.v;
		cnt += emit;
	}
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(n_emit, (unsigned long long)cnt);
}

// ---------------------------------------------------------------------------------------------
// ma_sg_gen without a device-wide sort (the default; MAB_SG_SEGSORT=0 or a case it declines -> the column sort above).
// Hits arrive grouped by query read (h.grp), and an arc's source vertex is its hit's query, so asg.c's "append, then sort
// by ul" only has to order each read's arcs by (direction, length), hit order on ties -- a per-read problem of ~100
// elements.  One pass over the hits: a CTA takes the next tile of SGW_WARPS consecutive reads, and each warp classifies
// its read's hits (with the deletion side effects of asm.c:27-33, which only ever set the read's own seq word) and sorts
// the keys ((dir << lb | len) << 9 | arc number) with the register network of ma_hit_sub.  The tile's arc count gets its
// offset from a decoupled look-back over the tiles before it (tiles start in order, so it never waits on one that is not
// running), and each warp writes its read's arcs and both index words: the sort puts direction 0 first, so the two slab
// lengths are the direction counts.  A read of 257..8192 hits is only counted by its warp, which reserves its arcs in the
// tile; a CTA with a shared-memory network sorts and writes it afterwards.  What the scheme cannot take (unsorted ids, a
// read beyond 8192 hits, reads longer than 4 Mb) is found before the launch and goes to the column sort, so results never
// depend on the switch.
// ---------------------------------------------------------------------------------------------
constexpr int SGW_WARPS = 8, SGW_HITS = 256, SGW_IDX_BITS = 9;
constexpr int SGC_HITS = 8192, SGC_THREADS = 512;

typedef cub::ScanTileState<uint32_t> ArcTileState;
typedef cub::TilePrefixCallbackOp<uint32_t, ::cuda::std::plus<uint32_t>, ArcTileState> ArcPrefixOp;

__global__ void k_arc_tiles_init(ArcTileState ts, int n_tile) { ts.InitializeStatus(n_tile); }

// the most hits of one read: from the bounds, or from the dense offsets of selected hits (off != null), whose bucket bounds also
// count the hits to dropped targets
__global__ void k_grp_max(const uint64_t *grp, const uint32_t *off, uint32_t n, unsigned long long *mx)
{
	unsigned m = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint64_t g = grp[i];
		const unsigned c = off ? off[i + 1] - off[i] : (uint32_t)g ? (uint32_t)g - (uint32_t)(g >> 32) : 0;
		m = c > m ? c : m;
	}
	m = __reduce_max_sync(0xffffffffu, m);
	if ((threadIdx.x & 31) == 0 && m) atomicMax(mx, (unsigned long long)m);
}

// SEL: the hits are selected, not compacted (DHits::map): grp holds bucket bounds, and a hit whose target was dropped is skipped
// before it is classified, so that its deletion side effects do not happen either.  Arcs are numbered among the kept hits, so the
// sort keys, and the arcs, are those of the dense array.  The warp / CTA choice goes by the bucket size; a read goes to the column
// sort only if it keeps more than 8192 hits.
template <bool SEL>
__global__ void __launch_bounds__(SGW_WARPS * 32)
k_sg_onepass(const DHit *__restrict__ a, const uint64_t *__restrict__ grp, const int32_t *__restrict__ map, const uint32_t *__restrict__ len32,
             uint32_t *seq, uint32_t n_seq, HitArcParams p, uint32_t lb, unsigned long long *tile_ctr, ArcTileState tstate, DArc *__restrict__ out,
             uint64_t *__restrict__ idx, uint2 *__restrict__ big_list, unsigned long long *scal)
{	// len32: the 32-bit read lengths ma_hit2arc takes (asm.c:23-24); seq only gets del bits.  An arc of 2^lb or more (a hit that
	// lies past its read's end) raises scal[SC_TMP0 + 1]; the caller then discards this pass and runs the column sort.
	__shared__ uint32_t s_key[SGW_WARPS][SGW_HITS], s_v[SGW_WARPS][SGW_HITS], s_ol[SGW_WARPS][SGW_HITS];
	__shared__ typename ArcPrefixOp::TempStorage s_pref;
	__shared__ uint32_t s_n[SGW_WARPS], s_tile, s_base;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const unsigned lt = (1u << lane) - 1u;
	uint32_t *key = s_key[warp], *pv = s_v[warp], *pol = s_ol[warp];
	const uint32_t len_mask = (1u << lb) - 1u; // lb <= 22 on this path
	if (threadIdx.x == 0) s_tile = (uint32_t)atomicAdd(tile_ctr, 1ull);
	__syncthreads();
	const uint32_t t = s_tile, r = t * SGW_WARPS + warp;
	uint32_t first = 0, cnt = 0, n = 0, n0 = 0; // n: arcs of this read, n0: those leaving vertex 2r (all uniform)
	int ql = 0;
	if (r < n_seq) {
		const uint64_t g = grp[r];
		if ((uint32_t)g) first = (uint32_t)(g >> 32), cnt = (uint32_t)g - first;
		ql = (int)len32[r];
	}
	const bool big = cnt > SGW_HITS;
	for (uint32_t c = 0; c < cnt; c += 32) {
		bool ok = false;
		DArc e;
		e.ul = 0, e.v = 0, e.ol_del = 0;
		if (c + lane < cnt) {
			DHit h = ld_hit(a + first + c + lane);
			if (!SEL || sel_renumber(h, r, map)) {
				const int rr = mab_hit2arc(h, ql, (int)len32[h.tn], p.max_hang, p.int_frac, p.min_ovlp, &e);
				if (rr >= 0) {
					if (h.tn == r) { // self match: only the palindromic artefact has an effect (asm.c:27-31)
						if ((uint32_t)h.qns == h.ts && h.qe == h.te && (h.ml_rev >> 31)) atomicOr(&seq[r], MAB_DEL_BIT);
					} else ok = true;
				} else if (rr == MAB_HT_QCONT) atomicOr(&seq[r], MAB_DEL_BIT);
			}
		}
		const uint32_t dir = (uint32_t)(e.ul >> 32) & 1u;
		if (ok && (uint32_t)e.ul > len_mask) scal[SC_TMP0 + 1] = 1; // (big reads too: the CTA pass sorts the same arcs)
		const unsigned m = __ballot_sync(0xffffffffu, ok), m0 = __ballot_sync(0xffffffffu, ok && dir == 0);
		if (ok && !big) {
			const uint32_t k = n + __popc(m & lt);
			key[k] = ((dir << lb | (uint32_t)e.ul) << SGW_IDX_BITS) | k;
			pv[k] = e.v, pol[k] = e.ol_del;
		}
		n += __popc(m), n0 += __popc(m0);
	}
	if (n && !big) {
		uint32_t np = 32; while (np < n) np <<= 1;
		__syncwarp();
		switch (np) {
			case 32: sub_sort_regs<1>(key, n, lane); break;
			case 64: sub_sort_regs<2>(key, n, lane); break;
			case 128: sub_sort_regs<4>(key, n, lane); break;
			default: sub_sort_regs<8>(key, n, lane); break;
		}
		__syncwarp();
	}
	if (lane == 0) {
		s_n[warp] = n;
		// the read's del bit is final here: the input set it, or this warp did (no other warp writes seq[r])
		if (r < n_seq && (atomicOr(&seq[r], 0u) & MAB_DEL_BIT)) atomicAdd(scal + SC_NSEL, 1ull);
	}
	__syncthreads();
	if (warp == 0) {
		const uint32_t agg = __reduce_add_sync(0xffffffffu, lane < SGW_WARPS ? s_n[lane] : 0u);
		if (t == 0) {
			if (lane == 0) tstate.SetInclusive(0, agg), s_base = 0;
		} else {
			ArcPrefixOp op(tstate, s_pref, ::cuda::std::plus<uint32_t>(), (int)t);
			const uint32_t ex = op(agg);
			if (lane == 0) s_base = ex;
		}
		if (lane == 0 && agg) atomicAdd(scal + SC_COUNT, (unsigned long long)agg);
	}
	__syncthreads();
	if (r >= n_seq) return;
	uint32_t base = s_base;
	for (int w = 0; w < warp; ++w) base += s_n[w];
	if (lane == 0) {
		idx[2 * (size_t)r] = n0 ? (uint64_t)base << 32 | n0 : 0;
		idx[2 * (size_t)r + 1] = n > n0 ? (uint64_t)(base + n0) << 32 | (n - n0) : 0;
		if (big && n) big_list[atomicAdd(scal + SC_BIG, 1ull)] = make_uint2(r, base);
	}
	if (big) return;
	for (uint32_t j = lane; j < n; j += 32) {
		const uint32_t k = key[j], src = k & ((1u << SGW_IDX_BITS) - 1u), kl = k >> SGW_IDX_BITS;
		*reinterpret_cast<uint4*>(out + base + j) = make_uint4(kl & len_mask, r << 1 | kl >> lb, pv[src], pol[src]);
	}
}

// the reads of 257..8192 hits k_sg_onepass counted and placed: big_list[b] = (read, offset of its first arc); SEL as there
template <bool SEL>
__global__ void __launch_bounds__(SGC_THREADS)
k_sg_sort_cta(const DHit *__restrict__ a, const uint64_t *__restrict__ grp, const int32_t *__restrict__ map, const uint32_t *__restrict__ len32,
              const uint2 *__restrict__ big_list, uint32_t n_big, HitArcParams p, DArc *__restrict__ out)
{
	typedef cub::BlockScan<uint32_t, SGC_THREADS> BS;
	extern __shared__ __align__(16) unsigned char sg_smem[];
	uint64_t *key = reinterpret_cast<uint64_t*>(sg_smem);         // (dir << 31 | len) << 32 | arc number
	uint32_t *pv = reinterpret_cast<uint32_t*>(key + SGC_HITS), *pol = pv + SGC_HITS;
	__shared__ typename BS::TempStorage s_scan;
	const uint32_t tid = threadIdx.x, nt = blockDim.x;
	for (uint32_t b = blockIdx.x; b < n_big; b += gridDim.x) {
		const uint2 rb = big_list[b];
		const uint32_t r = rb.x, base = rb.y;
		const uint64_t g = grp[r];
		const uint32_t first = (uint32_t)(g >> 32), cnt = (uint32_t)g - first;
		const int ql = (int)len32[r];
		uint32_t n = 0; // arcs of the chunks before (uniform)
		for (uint32_t c0 = 0; c0 < cnt; c0 += nt) {
			const uint32_t c = c0 + tid;
			bool ok = false;
			DArc e;
			e.ul = 0, e.v = 0, e.ol_del = 0;
			if (c < cnt) {
				DHit h = ld_hit(a + first + c);
				if (!SEL || sel_renumber(h, r, map)) {
					const int rr = mab_hit2arc(h, ql, (int)len32[h.tn], p.max_hang, p.int_frac, p.min_ovlp, &e);
					ok = rr >= 0 && h.tn != r;
				}
			}
			uint32_t k, tot;
			BS(s_scan).ExclusiveSum((uint32_t)ok, k, tot);
			if (ok) {
				k += n;
				key[k] = (uint64_t)((((uint32_t)(e.ul >> 32) & 1u) << 31) | (uint32_t)e.ul) << 32 | k;
				pv[k] = e.v, pol[k] = e.ol_del;
			}
			n += tot;
			__syncthreads();
		}
		uint32_t np = 2; while (np < n) np <<= 1;
		for (uint32_t i = n + tid; i < np; i += nt) key[i] = ~0ull;
		__syncthreads();
		for (uint32_t k = 2, lk = 1; k <= np; k <<= 1, ++lk)
			for (uint32_t lj = lk; lj-- > 0;) {
				const uint32_t j = 1u << lj;
				for (uint32_t t = tid; t < np / 2; t += nt) {
					const uint32_t lo = ((t >> lj) << (lj + 1)) | (t & (j - 1)), hi = lo + j;
					const uint64_t x = key[lo], y = key[hi];
					const bool asc = (lo & k) == 0;
					if ((x > y) == asc) key[lo] = y, key[hi] = x;
				}
				__syncthreads();
			}
		for (uint32_t j = tid; j < n; j += nt) {
			const uint64_t k = key[j];
			const uint32_t src = (uint32_t)k, kl = (uint32_t)(k >> 32);
			*reinterpret_cast<uint4*>(out + base + j) = make_uint4(kl & 0x7fffffffu, r << 1 | kl >> 31, pv[src], pol[src]);
		}
		__syncthreads();
	}
}

// true: g.arc holds the sorted arcs, g.idx their index and *n_del the deleted reads.  false: the caller runs the column sort, which
// rewrites g.arc and g.idx (if an arc outgrew lb, the del bits set in g.seq here are ones the column sort sets too).
static bool sg_emit_segmented(MabDev &d, const DHits &h, const uint32_t *len32, const HitArcParams &p, uint32_t lb, DGraph &g, uint32_t *n_del)
{
	const size_t n = h.n;
	const uint32_t n_seq = h.n_seq;
	if (lb + 1 + SGW_IDX_BITS > 32 || n >= (1ull << 31) || n_seq == 0) return false;
	d.zero_scal(SC_COUNT, 5); // SC_COUNT .. SC_AUX2
	d.zero_scal(SC_NSEL);
	d.zero_scal(SC_TMP0, 2);
	const uint64_t *grp = h.grp;
	uint64_t *own = nullptr;
	if (!grp) { // hits that did not come through the sort or the selection: the bounds of their runs, and whether the ids ascend
		own = mab_alloc<uint64_t>(d, n_seq);
		MAB_CUDA(cudaMemsetAsync(own, 0, (size_t)n_seq * 8, d.stream));
		MAB_LAUNCH(d, k_group_bounds, mab_grid(n, 256), 256, 0, h.a, n, (uint32_t*)own, d.d_scal + SC_AUX2);
		grp = own;
	}
	MAB_LAUNCH(d, k_grp_max, mab_grid(n_seq, 256), 256, 0, grp, h.off, n_seq, d.d_scal + SC_AUX);
	bool ok = d.get_scal(SC_AUX) <= (unsigned long long)SGC_HITS && d.h_scal[SC_AUX2] == 0;
	if (ok) {
		dg_reserve(d, g, n); // an arc never outnumbers its hits
		const int n_tile = (int)((n_seq + SGW_WARPS - 1) / SGW_WARPS);
		size_t ts_bytes = 0;
		MAB_CUDA(ArcTileState::AllocationSize(n_tile, ts_bytes));
		void *ts_mem = d.alloc(ts_bytes);
		ArcTileState ts;
		MAB_CUDA(ts.Init(n_tile, ts_mem, ts_bytes));
		MAB_LAUNCH(d, k_arc_tiles_init, mab_grid((size_t)n_tile, 256, 1u << 30), 256, 0, ts, n_tile);
		uint2 *big = mab_alloc<uint2>(d, n_seq);
		auto onepass = h.map ? k_sg_onepass<true> : k_sg_onepass<false>;
		MAB_LAUNCH(d, onepass, n_tile, SGW_WARPS * 32, 0, h.a, grp, h.map, len32, g.seq, n_seq, p, lb, d.d_scal + SC_TMP0, ts, g.arc, g.idx, big, d.d_scal);
		g.n_arc = (uint32_t)d.get_scal(SC_COUNT);
		*n_del = (uint32_t)d.h_scal[SC_NSEL];
		const uint32_t n_big = (uint32_t)d.h_scal[SC_BIG];
		ok = d.h_scal[SC_TMP0 + 1] == 0; // else an arc outgrew lb: the column sort redoes it all (the del bits set here are its own too)
		if (ok && n_big) {
			const size_t smem = (size_t)SGC_HITS * 16;
			const unsigned grid = n_big < MAB_SMS ? n_big : MAB_SMS;
			auto kern = h.map ? k_sg_sort_cta<true> : k_sg_sort_cta<false>;
			MAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
			MAB_LAUNCH(d, kern, grid, SGC_THREADS, smem, h.a, grp, h.map, len32, big, n_big, p, g.arc);
		}
		d.free(ts_mem); d.free(big);
		if (ok) g.len_bits = lb, g.is_srt = true, g.has_idx = true;
	}
	d.free(own);
	return ok;
}

void dh_sg_gen(MabDev &d, DHits &h, const uint32_t *len, const uint8_t *del, const HitArcParams &p, DGraph &g)
{
	const int64_t n_del = dh_sg_emit(d, h, len, del, p, g);
	// hit2arc never sets an arc's del bit: without a deleted read asg_arc_rm keeps every arc, and the sweep that finds out is skipped
	if ((n_del < 0 ? dg_n_del_seq(d, g) : (uint32_t)n_del) != 0) dg_cleanup(d, g);
	else if (!g.has_idx) dg_arc_index(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] read %d arcs\n", "ma_sg_gen", g.n_arc);
}

int64_t dh_sg_emit(MabDev &d, DHits &h, const uint32_t *len, const uint8_t *del, const HitArcParams &p, DGraph &g)
{
	const uint32_t n_seq = h.n_seq;
	dg_set_nseq(d, g, n_seq);
	g.n_arc = 0, g.is_srt = false, g.is_symm = false, g.has_idx = false;
	d.zero_scal(SC_AUX);
	d.zero_scal(SC_COUNT);
	unsigned *d_max = (unsigned*)(d.d_scal + SC_AUX);
	if (n_seq) MAB_LAUNCH(d, k_seq_set, mab_grid(n_seq, 256), 256, 0, n_seq, len, del, g.seq, d_max);
	const unsigned mx = (unsigned)(d.get_scal(SC_AUX) & 0xffffffffu); // the arc of a hit within its read is never longer than the read (miniasm.h:97-98); the kernels flag the others
	uint32_t lb = bits_for(mx);
	if (h.n) {
		if (h.n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 arcs on one GPU\n"); exit(73); }
		static const bool seg_sort = !(getenv("MAB_SG_SEGSORT") && atoi(getenv("MAB_SG_SEGSORT")) == 0); // default on; 0 = device-wide column sort
		uint32_t n_del = 0;
		if (seg_sort && sg_emit_segmented(d, h, len, p, lb, g, &n_del)) return n_del;
		dh_hits_dense(d, h);
		uint64_t *ka = mab_alloc<uint64_t>(d, h.n), *kb = mab_alloc<uint64_t>(d, h.n), *va = mab_alloc<uint64_t>(d, h.n), *vb = mab_alloc<uint64_t>(d, h.n);
		uint32_t n_arc;
		for (;;) { // lb bounds the arcs of hits that lie within their reads; one past its read's end takes the full 32 bits
			d.zero_scal(SC_COUNT);
			d.zero_scal(SC_AUX);
			const uint64_t sentinel = 1ull << (lb + bits_for((uint64_t)n_seq * 2 - 1));
			MAB_LAUNCH(d, k_sg_arcs, mab_grid(h.n, 256), 256, 0, h.a, h.n, len, g.seq, p, lb, sentinel, ka, va, d.d_scal + SC_COUNT, d.d_scal + SC_AUX);
			n_arc = (uint32_t)d.get_scal(SC_COUNT);
			if (!d.h_scal[SC_AUX]) break;
			lb = 32;
		}
		dg_build_sorted(d, g, ka, va, kb, vb, (uint32_t)h.n, n_arc, lb, true);
		d.free(ka); d.free(kb); d.free(va); d.free(vb);
	} else { dg_reserve(d, g, 1); g.is_srt = true; }
	return -1;
}
