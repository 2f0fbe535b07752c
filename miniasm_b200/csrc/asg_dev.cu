// asg_dev.cu -- string-graph container passes on the GPU (sm_90a).
//
// Reference behaviour being reproduced (file:line into lh3/miniasm):
//   asg_arc_rm          asg.c:57-70     stable compaction of live arcs
//   asg_arc_sort        asg.c:22-25     sort arcs by 64-bit ul (source vertex, then length)
//   asg_arc_index       asg.c:27-42     idx[v] = first<<32 | count
//   asg_cleanup         asg.c:72-80
//   asg_arc_del_multi   asg.c:104-121   asg_arc_del_asymm asg.c:124-138   asg_symm asg.c:140-145
//   asg_arc_del_trans   asg.c:148-193   Myers transitive reduction with fuzz
//   asg_arc_del_short   asg.c:83-101
//
// Everything here is integer / indexing work bounded by HBM bandwidth: arcs move as one 128-bit
// load each, slabs are staged in shared memory, vertices map to warps (CTAs for very long slabs).
#include "asg_dev.cuh"
#include <cub/cub.cuh>

int mab_verbose = 3;
thread_local int mab_mute = 0;
int mab_del_trans_count_inner = 0;
thread_local DelTransStats g_del_trans_stats;

// ---------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ DArc ld_arc(const DArc *p)
{
	uint4 t = *reinterpret_cast<const uint4*>(p);
	DArc a;
	a.ul = (uint64_t)t.y << 32 | t.x; a.v = t.z; a.ol_del = t.w;
	return a;
}
__device__ __forceinline__ DArc ld_arc_nc(const DArc *p)
{
	uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
	DArc a;
	a.ul = (uint64_t)t.y << 32 | t.x; a.v = t.z; a.ol_del = t.w;
	return a;
}

// one LDG.128 through the read-only path, kept as a single instruction even when only some words are used
// (two 32-bit loads of a 16-byte record cost twice the L1 wavefronts)
__device__ __forceinline__ uint4 ld_arc4(const DArc *p)
{
	uint4 t;
	asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(p));
	return t;
}

// Where the slab of a NEIGHBOUR vertex lives.  Single GPU: peer == nullptr, slab = arc + (idx[w] >> 32).
// Sharded run with peer access: nidx[w] is (offset in the owner's arc array) << 32 | count, owner = orig[w >> 1] % world
// (orig == nullptr: identity) and peer[owner] is that rank's arc array mapped through CUDA IPC -- the transitive
// reduction then reads remote slabs over NVLink as it needs them instead of first all-gathering every arc.
struct SlabView {
	const DArc *const *peer;
	const uint64_t *nidx;
	const uint32_t *orig;
	uint32_t world;
};
__device__ __forceinline__ const DArc *slab_base(const SlabView &sv, const DArc *arc, uint32_t w)
{
	if (sv.peer == nullptr) return arc;
	const uint32_t r = (sv.orig ? __ldg(sv.orig + (w >> 1)) : (w >> 1)) % sv.world;
	return sv.peer[r];
}

static inline uint32_t bits_for(uint64_t x) { uint32_t b = 0; while (x) ++b, x >>= 1; return b ? b : 1; }

void dg_reserve(MabDev &d, DGraph &g, size_t m_arc)
{
	if (m_arc <= g.m_arc) return;
	DArc *na = mab_alloc<DArc>(d, m_arc), *nb = mab_alloc<DArc>(d, m_arc);
	if (g.n_arc) MAB_CUDA(cudaMemcpyAsync(na, g.arc, (size_t)g.n_arc * sizeof(DArc), cudaMemcpyDeviceToDevice, d.stream));
	d.free(g.arc); d.free(g.arc2);
	g.arc = na, g.arc2 = nb, g.m_arc = m_arc;
}

void dg_set_nseq(MabDev &d, DGraph &g, uint32_t n_seq)
{
	d.free(g.seq); d.free(g.idx);
	g.n_seq = n_seq;
	g.seq = mab_alloc<uint32_t>(d, n_seq);
	g.idx = mab_alloc<uint64_t>(d, (size_t)n_seq * 2);
	g.has_idx = false;
}

void dg_free(MabDev &d, DGraph &g)
{
	d.free(g.arc); d.free(g.arc2); d.free(g.seq); d.free(g.idx);
	g = DGraph();
}

// ---------------------------------------------------------------------------------------------
// asg_arc_rm: keep arc iff !del && !seq[u>>1].del && !seq[v>>1].del   (asg.c:60-64)
// ---------------------------------------------------------------------------------------------
struct ArcKeep {
	const DArc *arc; const uint32_t *seq; const uint8_t *flag;
	__device__ __forceinline__ bool operator()(uint32_t i) const
	{
		DArc a = ld_arc_nc(arc + i);
		if (flag && flag[i]) return false;
		if (a.ol_del & MAB_DEL_BIT) return false;
		uint32_t u = (uint32_t)(a.ul >> 32);
		return !((seq[u >> 1] | seq[a.v >> 1]) & MAB_DEL_BIT);
	}
};

__global__ void k_arc_count_dead(ArcKeep keep, uint32_t n, unsigned long long *n_dead)
{
	unsigned dead = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dead += !keep(i);
	dead = __reduce_add_sync(0xffffffffu, dead);
	if ((threadIdx.x & 31) == 0 && dead) atomicAdd(n_dead, (unsigned long long)dead);
}

__global__ void k_seq_count_del(const uint32_t *seq, uint32_t n, unsigned long long *n_del)
{
	unsigned c = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += seq[i] >> 31;
	c = __reduce_add_sync(0xffffffffu, c);
	if ((threadIdx.x & 31) == 0 && c) atomicAdd(n_del, (unsigned long long)c);
}

uint32_t dg_n_del_seq(MabDev &d, const DGraph &g)
{
	if (g.n_seq == 0) return 0;
	d.zero_scal(SC_NSEL);
	MAB_LAUNCH(d, k_seq_count_del, mab_grid(g.n_seq, 256), 256, 0, g.seq, g.n_seq, d.d_scal + SC_NSEL);
	return (uint32_t)d.get_scal(SC_NSEL);
}

void dg_arc_rm(MabDev &d, DGraph &g, const uint8_t *flag)
{
	if (g.n_arc == 0) return;
	cub::CountingInputIterator<uint32_t> cnt(0);
	ArcKeep keep{g.arc, g.seq, flag};
	if (!flag && g.n_arc > (1u << 20)) { // a read-only sweep is half the traffic of a compaction: skip the copy when nothing dies
		d.zero_scal(SC_NSEL);
		MAB_LAUNCH(d, k_arc_count_dead, mab_grid(g.n_arc, 256), 256, 0, keep, g.n_arc, d.d_scal + SC_NSEL);
		if (d.get_scal(SC_NSEL) == 0) return;
	}
	cub::TransformInputIterator<bool, ArcKeep, cub::CountingInputIterator<uint32_t>> flags(cnt, keep);
	size_t tb = 0;
	unsigned long long *d_n = d.d_scal + SC_NSEL;
	cub::DeviceSelect::Flagged(nullptr, tb, g.arc, flags, g.arc2, d_n, (int)g.n_arc, d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceSelect::Flagged(tmp, tb, g.arc, flags, g.arc2, d_n, (int)g.n_arc, d.stream);
	++d.n_lib;
	uint32_t n = (uint32_t)d.get_scal(SC_NSEL);
	if (n < g.n_arc) g.has_idx = false; // arc index is out of sync (asg.c:65-68)
	DArc *t = g.arc; g.arc = g.arc2; g.arc2 = t;
	g.n_arc = n;
}

// ---------------------------------------------------------------------------------------------
// asg_arc_sort: radix sort on a compacted key (u << len_bits | len) with the 8 remaining bytes of
// the arc as payload.  CUB's sort is stable (ties keep input order); the reference's in-place MSD
// radix sort is not, see DESIGN.md "tie order".
// ---------------------------------------------------------------------------------------------
__global__ void k_arc_split(const DArc *arc, uint32_t n, uint32_t len_bits, uint64_t *key, uint64_t *val)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		DArc a = ld_arc_nc(arc + i);
		key[i] = (a.ul >> 32) << len_bits | (uint32_t)a.ul;
		val[i] = (uint64_t)a.ol_del << 32 | a.v;
	}
}

__global__ void k_arc_merge(const uint64_t *key, const uint64_t *val, uint32_t n, uint32_t len_bits, DArc *arc)
{
	const uint64_t lm = len_bits >= 64 ? ~0ull : ((1ull << len_bits) - 1);
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		uint64_t k = key[i], v = val[i];
		uint4 o;
		o.x = (uint32_t)(k & lm); o.y = (uint32_t)(k >> len_bits); o.z = (uint32_t)v; o.w = (uint32_t)(v >> 32);
		*reinterpret_cast<uint4*>(arc + i) = o;
	}
}

void dg_arc_sort(MabDev &d, DGraph &g)
{
	uint32_t n = g.n_arc;
	if (n > 1) {
		uint32_t lb = g.len_bits > 32 ? 32 : g.len_bits;
		uint32_t end_bit = lb + bits_for((uint64_t)g.n_seq * 2 - 1);
		uint64_t *ka = mab_alloc<uint64_t>(d, n), *kb = mab_alloc<uint64_t>(d, n);
		uint64_t *va = mab_alloc<uint64_t>(d, n), *vb = mab_alloc<uint64_t>(d, n);
		MAB_LAUNCH(d, k_arc_split, mab_grid(n, 256), 256, 0, g.arc, n, lb, ka, va);
		cub::DoubleBuffer<uint64_t> dk(ka, kb), dv(va, vb);
		size_t tb = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)n, 0, (int)end_bit, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)n, 0, (int)end_bit, d.stream);
		++d.n_lib;
		MAB_LAUNCH(d, k_arc_merge, mab_grid(n, 256), 256, 0, dk.Current(), dv.Current(), n, lb, g.arc);
		d.free(ka); d.free(kb); d.free(va); d.free(vb);
	}
	g.is_srt = true;
}

// Builds the sorted AoS arc array from unsorted (key, value) columns; keys equal to `sentinel` (placed past every
// real key) are padding and end up behind the n_real arcs.  Used by ma_sg_gen, which emits the columns directly.
void dg_build_sorted(MabDev &d, DGraph &g, uint64_t *key, uint64_t *val, uint64_t *key2, uint64_t *val2, uint32_t n_in, uint32_t n_real, uint32_t lb, bool has_sentinel)
{
	dg_reserve(d, g, n_real ? n_real : 1);
	g.len_bits = lb;
	if (n_in > 1) {
		uint32_t end_bit = lb + bits_for((uint64_t)g.n_seq * 2 - 1) + (has_sentinel ? 1 : 0);
		cub::DoubleBuffer<uint64_t> dk(key, key2), dv(val, val2);
		size_t tb = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)n_in, 0, (int)end_bit, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)n_in, 0, (int)end_bit, d.stream);
		++d.n_lib;
		if (n_real) MAB_LAUNCH(d, k_arc_merge, mab_grid(n_real, 256), 256, 0, dk.Current(), dv.Current(), n_real, lb, g.arc);
	} else if (n_real) MAB_LAUNCH(d, k_arc_merge, 1, 32, 0, key, val, n_real, lb, g.arc);
	g.n_arc = n_real, g.is_srt = true, g.has_idx = false;
}

// ---------------------------------------------------------------------------------------------
// asg_arc_index: run boundaries of ul>>32 -> idx[v] = first<<32 | count
// ---------------------------------------------------------------------------------------------
__global__ void k_index_bounds(const DArc *arc, uint32_t n, uint32_t *idx32)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		uint32_t u = (uint32_t)(arc[i].ul >> 32);
		if (i == 0 || (uint32_t)(arc[i - 1].ul >> 32) != u) idx32[2 * (size_t)u + 1] = i;      // first
		if (i == n - 1 || (uint32_t)(arc[i + 1].ul >> 32) != u) idx32[2 * (size_t)u] = i + 1;  // end (exclusive)
	}
}
__global__ void k_index_fix(uint64_t *idx, uint32_t n_vtx)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) {
		uint64_t x = idx[v];
		uint32_t first = (uint32_t)(x >> 32), end = (uint32_t)x;
		idx[v] = end ? ((uint64_t)first << 32 | (end - first)) : 0;
	}
}

void dg_arc_index(MabDev &d, DGraph &g)
{
	uint32_t n_vtx = g.n_seq * 2;
	if (n_vtx == 0) { g.has_idx = true; return; }
	MAB_CUDA(cudaMemsetAsync(g.idx, 0, (size_t)n_vtx * 8, d.stream));
	if (g.n_arc) {
		MAB_LAUNCH(d, k_index_bounds, mab_grid(g.n_arc, 256), 256, 0, g.arc, g.n_arc, (uint32_t*)g.idx);
		MAB_LAUNCH(d, k_index_fix, mab_grid(n_vtx, 256), 256, 0, g.idx, n_vtx);
	}
	g.has_idx = true;
}

void dg_cleanup(MabDev &d, DGraph &g, const uint8_t *flag)
{
	dg_arc_rm(d, g, flag);
	if (!g.is_srt) dg_arc_sort(d, g);
	if (!g.has_idx) dg_arc_index(d, g);
}

// ---------------------------------------------------------------------------------------------
// asg_arc_del_multi: within a slab keep only the lowest-index arc to each target (asg.c:112-115:
// the counter walk from the back deletes every arc that has an earlier arc to the same target).
// asg_arc_del_asymm: delete u->v when v^1 -> u^1 is absent (asg.c:127-133).
// Both run on slabs; the heavy case (the unreduced graph) is rare, so one thread per arc suffices.
// ---------------------------------------------------------------------------------------------
__global__ void k_del_multi(DArc *arc, const uint64_t *idx, uint32_t n_arc, unsigned long long *n_out)
{
	unsigned long long cnt = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_arc; i += gridDim.x * blockDim.x) {
		DArc a = ld_arc(arc + i);
		uint64_t x = idx[a.ul >> 32];
		uint32_t first = (uint32_t)(x >> 32), nv = (uint32_t)x;
		if (nv < 2) continue;
		bool dup = false;
		for (uint32_t j = first; j < i; ++j)
			if (arc[j].v == a.v) { dup = true; break; }
		if (dup) { arc[i].ol_del = a.ol_del | MAB_DEL_BIT; ++cnt; }
	}
	cnt = __reduce_add_sync(0xffffffffu, (unsigned)cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(n_out, cnt);
}

__global__ void k_del_asymm(DArc *arc, const uint64_t *idx, uint32_t n_arc, unsigned long long *n_out)
{
	unsigned cnt = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_arc; i += gridDim.x * blockDim.x) {
		DArc a = ld_arc(arc + i);
		uint32_t v = a.v ^ 1, u = (uint32_t)(a.ul >> 32) ^ 1;
		uint64_t x = idx[v];
		uint32_t first = (uint32_t)(x >> 32), nv = (uint32_t)x, j;
		for (j = 0; j < nv; ++j)
			if (arc[first + j].v == u) break;
		if (j == nv) { arc[i].ol_del = a.ol_del | MAB_DEL_BIT; ++cnt; }
	}
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(n_out, (unsigned long long)cnt);
}

uint32_t dg_del_multi(MabDev &d, DGraph &g)
{
	uint32_t n_multi = 0;
	if (g.n_arc) {
		d.zero_scal(SC_COUNT);
		MAB_LAUNCH(d, k_del_multi, mab_grid(g.n_arc, 256), 256, 0, g.arc, g.idx, g.n_arc, d.d_scal + SC_COUNT);
		n_multi = (uint32_t)d.get_scal(SC_COUNT);
	}
	if (n_multi) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] removed %d multi-arcs\n", "asg_arc_del_multi", n_multi);
	return n_multi;
}

uint32_t dg_del_asymm(MabDev &d, DGraph &g)
{
	uint32_t n_asymm = 0;
	if (g.n_arc) {
		d.zero_scal(SC_COUNT);
		MAB_LAUNCH(d, k_del_asymm, mab_grid(g.n_arc, 256), 256, 0, g.arc, g.idx, g.n_arc, d.d_scal + SC_COUNT);
		n_asymm = (uint32_t)d.get_scal(SC_COUNT);
	}
	if (n_asymm) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] removed %d asymmetric arcs\n", "asg_arc_del_asymm", n_asymm);
	return n_asymm;
}

void dg_symm(MabDev &d, DGraph &g)
{
	dg_del_multi(d, g);
	dg_del_asymm(d, g);
	g.is_symm = true;
}

// ---------------------------------------------------------------------------------------------
// asg_arc_del_trans (asg.c:148-193).
//
// For vertex v with out-slab av[0..nv) (length ascending):  every target gets mark 1;  L = longest
// arc + fuzz;  for i ascending, if mark[target_i] is still 1, scan the slab of w = target_i while
// len(w->x) + len(v->w) <= L and promote mark[x] to 2 when x is one of v's targets;  finally every
// arc whose target carries mark 2 is reduced.  A vertex only writes flags of its own slab and never
// reads another slab's flags, so all vertices are independent (SURVEY.md 3.2); inside a vertex the
// i loop is sequential (the "still 1" test) and the j loop is lane-parallel.
//
// Mapping: one warp per vertex for slabs up to DT_MAXD arcs (targets + lengths + the idx words of
// all targets staged in shared memory, an open-addressing table target -> first slab position for
// the mark lookups); one CTA per vertex for longer slabs; a global mark array for slabs beyond the
// CTA table.  Output is one byte per arc (flag[i] = reduced), consumed by the compaction pass.
// ---------------------------------------------------------------------------------------------
constexpr int DT_WARPS = 8;      // warps per CTA, warp kernel
constexpr int DT_MAXD  = 128;    // longest slab the warp kernel takes
constexpr int DT_HASH  = 256;    // table slots per warp (the live part is the next power of two >= 2*nv)
constexpr int DT_EAGER = 4;      // slab positions whose neighbour index word is fetched ahead of use
constexpr uint32_t DT_EMPTY = 0xffffffffu;

__device__ __forceinline__ uint32_t dt_hash(uint32_t x, uint32_t mask) { return (x * 2654435761u) >> 7 & mask; }

// ---------------------------------------------------------------------------------------------
// k_del_trans_warp -- one warp per vertex.  Shared memory per warp: hkey (target vertex per table slot) | tl (arc length
// per slab entry) | hmark (mark per slot: 1 = target of v, 2 = reduced) | slot (table slot of slab entry i) | fmin
// (lowest slab position per slot, only when a slab holds multi-arcs).  The mark lives in the table, so arcs to the same
// target share it exactly like mark[] indexed by vertex does in the reference.
// The kernel is issue-bound (an earlier version spent ~476 warp instructions per vertex, nearly all of them per-vertex
// bookkeeping), so this version keeps the instruction stream short: peer/no-peer is a
// template parameter, the table is cleared with one or two 128-bit stores, every slab loop stays rolled (two entries per
// lane cover 64 arcs), the next vertex's index/seq words are prefetched, and (SORTED, i.e. whenever the graph says
// is_srt) a slab sorted by length makes the arcs that satisfy the length bound a prefix by themselves.
// ---------------------------------------------------------------------------------------------
template <bool STATS, bool P2P, bool SORTED>
__global__ void __launch_bounds__(DT_WARPS * 32, 6)
k_del_trans_warp(const DArc *__restrict__ arc, const uint64_t *__restrict__ idx, const uint32_t *__restrict__ seq,
                 uint32_t n_vtx, uint32_t fuzz, uint8_t *__restrict__ flag,
                 uint32_t *__restrict__ big_list, unsigned long long *scal, uint32_t own_lo, uint32_t own_hi, SlabView sv)
{	// [own_lo, own_hi): arc positions this rank is responsible for (sharded runs); a vertex is processed iff its slab starts there
	const uint64_t *__restrict__ nidx = P2P ? sv.nidx : idx; // index words of the neighbours (global offsets in sharded runs)
	__shared__ __align__(16) uint32_t s_hkey[DT_WARPS][DT_HASH];
	__shared__ uint32_t s_tl[DT_WARPS][DT_MAXD];
	__shared__ uint32_t s_fmin[DT_WARPS][DT_HASH];
	__shared__ uint8_t  s_hmark[DT_WARPS][DT_HASH];
	__shared__ uint8_t  s_slot[DT_WARPS][DT_MAXD];

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	uint32_t *hkey = s_hkey[warp], *tl = s_tl[warp], *fmin = s_fmin[warp];
	uint8_t *hmark = s_hmark[warp], *slot = s_slot[warp];
	unsigned n_red = 0;
	unsigned long long n_inner = 0;

	// Software pipeline over the vertices of this warp: while vertex v is worked on, the index / seq words of the next one are
	// already in flight, and its first 64 slab entries are requested as soon as those words have landed: without it the
	// warps stall on the first use of the own slab and on idx/seq.
	const uint32_t stride = gridDim.x * DT_WARPS;
	uint32_t v = blockIdx.x * DT_WARPS + warp;
	uint64_t iv = 0, iv_n = 0;
	uint32_t sq = 0, sq_n = 0;
	uint4 p0 = make_uint4(0, 0, 0, 0), p1 = p0, p0n = p0, p1n = p0;   // slab entries lane / lane + 32 of the current / next vertex
	if (v < n_vtx) {
		iv = __ldg(idx + v), sq = __ldg(seq + (v >> 1));
		if (lane < (uint32_t)iv) p0 = ld_arc4(arc + (iv >> 32) + lane);
		if (lane + 32 < (uint32_t)iv) p1 = ld_arc4(arc + (iv >> 32) + lane + 32);
	}
	#pragma unroll 1
	for (; v < n_vtx; v += stride, iv = iv_n, sq = sq_n, p0 = p0n, p1 = p1n) {
		const bool more = v + stride < n_vtx;
		if (more) iv_n = __ldg(idx + v + stride), sq_n = __ldg(seq + ((v + stride) >> 1));
		#define DT_PREFETCH_NEXT() do { if (more) { \
			if (lane < (uint32_t)iv_n) p0n = ld_arc4(arc + (iv_n >> 32) + lane); \
			if (lane + 32 < (uint32_t)iv_n) p1n = ld_arc4(arc + (iv_n >> 32) + lane + 32); } } while (0)
		const uint32_t nv = (uint32_t)iv, off = (uint32_t)(iv >> 32);
		if (nv == 0 || off < own_lo || off >= own_hi) { DT_PREFETCH_NEXT(); continue; }
		if (sq & MAB_DEL_BIT) { // deleted read: every arc goes (asg.c:158-161)
			DT_PREFETCH_NEXT();
			for (uint32_t i = lane; i < nv; i += 32) flag[off + i] = 1;
			if (lane == 0) n_red += nv;
			continue;
		}
		if (nv > DT_MAXD) { // hand over to the CTA kernel
			DT_PREFETCH_NEXT();
			if (lane == 0) big_list[atomicAdd(scal + SC_BIG, 1ull)] = v;
			continue;
		}
		// table = next power of two >= 4*nv (load <= 1/4: the v4 profile shows 1.7-1.9 probes per lookup at load ~0.4), 32..256 slots
		const uint32_t mask = nv <= 8 ? 31u : (nv > 32 ? (uint32_t)DT_HASH - 1u : (0xffffffffu >> __clz(4 * nv - 1)));
		// the table of a warp has DT_HASH = 256 slots; clearing 128 of them (one 128-bit store per lane) covers every mask <= 127
		*reinterpret_cast<uint4*>(hkey + 4 * lane) = make_uint4(DT_EMPTY, DT_EMPTY, DT_EMPTY, DT_EMPTY);
		if (mask > 127) *reinterpret_cast<uint4*>(hkey + 128 + 4 * lane) = make_uint4(DT_EMPTY, DT_EMPTY, DT_EMPTY, DT_EMPTY);
		__syncwarp();
		// stage the slab and build the target table in one sweep; every lane carries two slab entries per
		// iteration (i and i+32), so slabs of up to 64 arcs -- nearly all of them -- take a single iteration
		bool dup = false;
		uint64_t my_iw = 0; // lanes 0..DT_EAGER-1: index word of the target of slab entry `lane`, fetched ahead of use
		#pragma unroll 1
		for (uint32_t base = 0; base < nv; base += 64) {
			const uint32_t i0 = base + lane, i1 = i0 + 32;
			const bool v0 = i0 < nv, v1 = i1 < nv;
			uint4 a0 = p0, a1 = p1;                      // base 0: loaded one iteration ahead
			if (base) {
				if (v0) a0 = ld_arc4(arc + off + i0);   // x = len, z = target
				if (v1) a1 = ld_arc4(arc + off + i1);
			}
			if (v0) {
				tl[i0] = a0.x;
				if (i0 < DT_EAGER) my_iw = __ldg(nidx + a0.z);
				uint32_t h = dt_hash(a0.z, mask);
				for (;;) {
					const uint32_t prev = atomicCAS(&hkey[h], DT_EMPTY, a0.z);
					if (prev == DT_EMPTY) { hmark[h] = 1; break; }
					if (prev == a0.z) { dup = true; break; }
					h = (h + 1) & mask;
				}
				slot[i0] = (uint8_t)h;
			}
			if (v1) {
				tl[i1] = a1.x;
				uint32_t h = dt_hash(a1.z, mask);
				for (;;) {
					const uint32_t prev = atomicCAS(&hkey[h], DT_EMPTY, a1.z);
					if (prev == DT_EMPTY) { hmark[h] = 1; break; }
					if (prev == a1.z) { dup = true; break; }
					h = (h + 1) & mask;
				}
				slot[i1] = (uint8_t)h;
			}
		}
		const bool has_dup = __any_sync(0xffffffffu, dup); // multi-arcs: several slab entries share one mark
		__syncwarp();
		DT_PREFETCH_NEXT();                                // idx/seq of the next vertex have landed by now: request its slab
		const uint32_t L = tl[nv - 1] + fuzz;
		// i ascends over the slab entries whose target still carries mark 1 (asg.c:164-168); found by ballot
		for (uint32_t i = 0;;) {
			uint32_t nxt = nv;
			#pragma unroll 1
			for (uint32_t base = i & ~63u; base < nv; base += 64) {
				const uint32_t k0 = base + lane, k1 = k0 + 32;
				const bool l0 = k0 >= i && k0 < nv && hmark[slot[k0]] == 1;
				const bool l1 = k1 >= i && k1 < nv && hmark[slot[k1]] == 1;
				const unsigned m0 = __ballot_sync(0xffffffffu, l0), m1 = __ballot_sync(0xffffffffu, l1);
				if (m0) { nxt = base + __ffs(m0) - 1; break; }
				if (m1) { nxt = base + 32 + __ffs(m1) - 1; break; }
			}
			// (no __syncwarp here: every lane's reads of hmark feed its ballot predicate and no lane passes the ballot before all have
			// arrived, so the marks are read before any lane rewrites them below.  racecheck reports the pattern as a warp-level WAR
			// *warning*; an explicit barrier silences it at the cost of a slower kernel)
			if (nxt >= nv) break;
			i = nxt;
			const uint32_t w = hkey[slot[i]], li = tl[i];
			uint64_t iw; // i is warp-uniform: the prefetched word sits in lane i's register
			if (i < DT_EAGER) iw = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(my_iw >> 32), i) << 32 | __shfl_sync(0xffffffffu, (uint32_t)my_iw, i);
			else iw = __ldg(nidx + w);
			const uint32_t nw = (uint32_t)iw;
			const DArc *pw = (P2P ? slab_base(sv, arc, w) : arc) + (iw >> 32) + lane;
			#pragma unroll 1
			for (uint32_t j0 = 0; j0 < nw; j0 += 64, pw += 64) {
				const bool in0 = j0 + lane < nw, in1 = j0 + 32 + lane < nw;
				uint4 a0 = make_uint4(0, 0, 0, 0), a1 = make_uint4(0, 0, 0, 0);
				if (in0) a0 = ld_arc4(pw);
				if (in1) a1 = ld_arc4(pw + 32);
				const bool ok0 = in0 && a0.x + li <= L, ok1 = in1 && a1.x + li <= L;
				const unsigned m0 = __ballot_sync(0xffffffffu, ok0), m1 = __ballot_sync(0xffffffffu, ok1);
				// the scan of the reference stops at the first j that violates the bound: entries before it, in slab order
				// (SORTED: the slab is sorted by length, so the entries that pass already form that prefix)
				const unsigned pre0 = SORTED ? m0 : (m0 == 0xffffffffu ? m0 : ((1u << (__ffs(~m0) - 1)) - 1));
				const unsigned pre1 = SORTED ? m1 : (m0 != 0xffffffffu ? 0u : (m1 == 0xffffffffu ? m1 : ((1u << (__ffs(~m1) - 1)) - 1)));
				if (pre0 >> lane & 1) {
					uint32_t h = dt_hash(a0.z, mask);
					for (;;) {
						const uint32_t kx = hkey[h];
						if (kx == a0.z) { hmark[h] = 2; break; }
						if (kx == DT_EMPTY) break;
						h = (h + 1) & mask;
					}
				}
				if (pre1 >> lane & 1) {
					uint32_t h = dt_hash(a1.z, mask);
					for (;;) {
						const uint32_t kx = hkey[h];
						if (kx == a1.z) { hmark[h] = 2; break; }
						if (kx == DT_EMPTY) break;
						h = (h + 1) & mask;
					}
				}
				if (STATS && lane == 0) n_inner += __popc(pre0) + __popc(pre1);
				if (m0 != 0xffffffffu || m1 != 0xffffffffu) break;
			}
			__syncwarp();
			++i;
		}
		// The reference clears mark[target] right after looking at the first arc to that target
		// (asg.c:181-184), so of several arcs to one reduced target only the lowest-index one is deleted.
		if (has_dup) {
			for (uint32_t i = lane; i <= mask; i += 32) fmin[i] = DT_EMPTY;
			__syncwarp();
			for (uint32_t i = lane; i < nv; i += 32) atomicMin(&fmin[slot[i]], i);
			__syncwarp();
		}
		#pragma unroll 1
		for (uint32_t base = 0; base < nv; base += 64) { // two slab entries per lane, like the staging sweep
			const uint32_t i0 = base + lane, i1 = i0 + 32;
			if (i0 < nv) {
				const uint32_t s0 = slot[i0];
				const bool r = hmark[s0] == 2 && (!has_dup || fmin[s0] == i0);
				flag[off + i0] = r;
				n_red += r;
			}
			if (i1 < nv) {
				const uint32_t s1 = slot[i1];
				const bool r = hmark[s1] == 2 && (!has_dup || fmin[s1] == i1);
				flag[off + i1] = r;
				n_red += r;
			}
		}
		__syncwarp();
	}
	n_red = __reduce_add_sync(0xffffffffu, n_red);
	if (lane == 0) {
		if (n_red) atomicAdd(scal + SC_COUNT, (unsigned long long)n_red);
		if (STATS && n_inner) atomicAdd(scal + SC_AUX, n_inner);
	}
}

// CTA per vertex, slabs of DT_MAXD < nv <= DT_BIG_MAXD.  Dynamic shared memory:
//   tv[DT_BIG_MAXD] | hash[2*DT_BIG_MAXD] | fmin[DT_BIG_MAXD] | rep (u16)[DT_BIG_MAXD] | st (u8)[DT_BIG_MAXD]
constexpr int DT_BIG_MAXD = 8192;
constexpr int DT_BIG_HASH = 2 * DT_BIG_MAXD;
constexpr size_t DT_BIG_SMEM = (size_t)DT_BIG_MAXD * 4 + (size_t)DT_BIG_HASH * 4 + (size_t)DT_BIG_MAXD * 4 + (size_t)DT_BIG_MAXD * 2 + DT_BIG_MAXD;

__global__ void __launch_bounds__(256)
k_del_trans_cta(const DArc *__restrict__ arc, const uint64_t *__restrict__ idx, uint32_t fuzz, uint8_t *__restrict__ flag,
                const uint32_t *__restrict__ big_list, uint32_t n_big, uint32_t *__restrict__ huge_list, unsigned long long *scal, SlabView sv)
{
	extern __shared__ __align__(16) unsigned char smem[];
	uint32_t *tv = (uint32_t*)smem;
	uint32_t *hs = tv + DT_BIG_MAXD;
	uint32_t *fmin = hs + DT_BIG_HASH;
	uint16_t *rep = (uint16_t*)(fmin + DT_BIG_MAXD);
	uint8_t *st = (uint8_t*)(rep + DT_BIG_MAXD);
	__shared__ uint32_t s_go, s_red;
	__shared__ unsigned long long s_inner;
	const int tid = threadIdx.x, nt = blockDim.x;

	for (uint32_t b = blockIdx.x; b < n_big; b += gridDim.x) {
		const uint32_t v = big_list[b];
		const uint64_t iv = idx[v];
		const uint32_t nv = (uint32_t)iv, off = (uint32_t)(iv >> 32);
		if (nv > DT_BIG_MAXD) {
			if (tid == 0) huge_list[atomicAdd(scal + SC_AUX2, 1ull)] = v;
			continue;
		}
		if (tid == 0) s_red = 0, s_inner = 0;
		for (uint32_t i = tid; i < DT_BIG_HASH; i += nt) hs[i] = DT_EMPTY;
		for (uint32_t i = tid; i < nv; i += nt) tv[i] = arc[off + i].v, st[i] = 1, fmin[i] = DT_EMPTY;
		__syncthreads();
		for (uint32_t i = tid; i < nv; i += nt) {
			uint32_t x = tv[i], h = dt_hash(x, DT_BIG_HASH - 1);
			for (;;) {
				uint32_t prev = atomicCAS(&hs[h], DT_EMPTY, i);
				if (prev == DT_EMPTY) { rep[i] = (uint16_t)i; break; }
				if (tv[prev] == x) { rep[i] = (uint16_t)prev; break; }
				h = (h + 1) & (DT_BIG_HASH - 1);
			}
		}
		__syncthreads();
		for (uint32_t i = tid; i < nv; i += nt) atomicMin(&fmin[rep[i]], i); // lowest slab position per target
		__syncthreads();
		const uint32_t L = (uint32_t)arc[off + nv - 1].ul + fuzz;
		for (uint32_t i = 0; i < nv; ++i) {
			if (st[rep[i]] != 1) continue; // uniform: shared state, barrier at the end of the previous round
			const uint64_t iw = (sv.peer ? sv.nidx : idx)[tv[i]];
			const uint32_t nw = (uint32_t)iw, li = (uint32_t)arc[off + i].ul;
			const DArc *aw = slab_base(sv, arc, tv[i]) + (iw >> 32);
			// the scan stops at the first j violating the bound; lengths ascend, so find it per chunk
			for (uint32_t j0 = 0; j0 < nw; j0 += nt) {
				if (tid == 0) s_go = 0xffffffffu;
				__syncthreads();
				uint32_t j = j0 + tid, x = 0;
				bool ok = false;
				if (j < nw) {
					DArc a = ld_arc_nc(aw + j);
					ok = ((uint32_t)a.ul + li <= L);
					x = a.v;
					if (!ok) atomicMin(&s_go, j);
				}
				__syncthreads();
				const uint32_t stop = s_go; // first failing j in this chunk (or none)
				if (j < nw && j < stop) {
					uint32_t h = dt_hash(x, DT_BIG_HASH - 1);
					for (;;) {
						uint32_t p = hs[h];
						if (p == DT_EMPTY) break;
						if (tv[p] == x) { st[p] = 2; break; }
						h = (h + 1) & (DT_BIG_HASH - 1);
					}
				}
				if (tid == 0) { uint32_t e = j0 + nt < nw ? j0 + nt : nw; s_inner += (stop < e ? stop : e) - j0; }
				__syncthreads();
				if (stop != 0xffffffffu) break;
			}
			__syncthreads();
		}
		unsigned r_cnt = 0;
		for (uint32_t i = tid; i < nv; i += nt) {
			bool r = st[rep[i]] == 2 && fmin[rep[i]] == i; // only the first arc to a reduced target goes (asg.c:181-184)
			flag[off + i] = r;
			r_cnt += r;
		}
		if (r_cnt) atomicAdd(&s_red, r_cnt);
		__syncthreads();
		if (tid == 0) {
			if (s_red) atomicAdd(scal + SC_COUNT, (unsigned long long)s_red);
			if (s_inner) atomicAdd(scal + SC_AUX, s_inner);
		}
		__syncthreads();
	}
}

// Slabs beyond the CTA table: one CTA walks them one after another with a global mark array, i.e. the
// reference's own formulation (mark[] indexed by target vertex), the j loop spread over the CTA.
__global__ void __launch_bounds__(1024)
k_del_trans_huge(const DArc *__restrict__ arc, const uint64_t *__restrict__ idx, uint32_t fuzz, uint8_t *__restrict__ flag,
                 const uint32_t *__restrict__ huge_list, uint32_t n_huge, uint8_t *mark, uint32_t *first_pos, unsigned long long *scal, SlabView sv)
{
	__shared__ uint32_t s_go, s_red;
	__shared__ unsigned long long s_inner;
	const int tid = threadIdx.x, nt = blockDim.x;
	if (tid == 0) s_red = 0, s_inner = 0;
	__syncthreads();
	for (uint32_t b = 0; b < n_huge; ++b) {
		const uint32_t v = huge_list[b];
		const uint64_t iv = idx[v];
		const uint32_t nv = (uint32_t)iv, off = (uint32_t)(iv >> 32);
		for (uint32_t i = tid; i < nv; i += nt) mark[arc[off + i].v] = 1, atomicMin(&first_pos[arc[off + i].v], i);
		__syncthreads();
		const uint32_t L = (uint32_t)arc[off + nv - 1].ul + fuzz;
		for (uint32_t i = 0; i < nv; ++i) {
			const uint32_t w = arc[off + i].v;
			if (mark[w] != 1) continue;
			const uint64_t iw = (sv.peer ? sv.nidx : idx)[w];
			const uint32_t nw = (uint32_t)iw, li = (uint32_t)arc[off + i].ul;
			const DArc *aw = slab_base(sv, arc, w) + (iw >> 32);
			for (uint32_t j0 = 0; j0 < nw; j0 += nt) {
				if (tid == 0) s_go = 0xffffffffu;
				__syncthreads();
				uint32_t j = j0 + tid, x = 0;
				if (j < nw) {
					DArc a = ld_arc_nc(aw + j);
					x = a.v;
					if (!((uint32_t)a.ul + li <= L)) atomicMin(&s_go, j);
				}
				__syncthreads();
				const uint32_t stop = s_go;
				if (j < nw && j < stop && mark[x]) mark[x] = 2;
				if (tid == 0) { uint32_t e = j0 + nt < nw ? j0 + nt : nw; s_inner += (stop < e ? stop : e) - j0; }
				__syncthreads();
				if (stop != 0xffffffffu) break;
			}
			__syncthreads();
		}
		unsigned r_cnt = 0;
		for (uint32_t i = tid; i < nv; i += nt) {
			bool r = mark[arc[off + i].v] == 2 && first_pos[arc[off + i].v] == i;
			flag[off + i] = r;
			r_cnt += r;
		}
		if (r_cnt) atomicAdd(&s_red, r_cnt);
		__syncthreads();
		for (uint32_t i = tid; i < nv; i += nt) mark[arc[off + i].v] = 0, first_pos[arc[off + i].v] = 0xffffffffu;
		__syncthreads();
	}
	if (tid == 0) {
		if (s_red) atomicAdd(scal + SC_COUNT, (unsigned long long)s_red);
		if (s_inner) atomicAdd(scal + SC_AUX, s_inner);
	}
}

uint32_t dg_del_trans(MabDev &d, DGraph &g, uint32_t fuzz)
{
	uint8_t *flag = nullptr;
	uint32_t n_reduced = dg_del_trans_flags(d, g, fuzz, 0, 0xffffffffu, &flag, nullptr, nullptr, nullptr, 1);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] transitively reduced %d arcs\n", "asg_arc_del_trans", n_reduced);
	if (n_reduced) {
		dg_cleanup(d, g, flag);
		dg_symm(d, g);
	}
	d.free(flag);
	return n_reduced;
}

// the marking part of asg_arc_del_trans for the vertices whose slabs start in [own_lo, own_hi): one flag byte per arc
// of those slabs (other positions of *flag_out are not written); returns the number of arcs flagged
uint32_t dg_del_trans_flags(MabDev &d, DGraph &g, uint32_t fuzz, uint32_t own_lo, uint32_t own_hi, uint8_t **flag_out,
                            const DArc *const *peer, const uint64_t *nidx, const uint32_t *orig, uint32_t world)
{
	SlabView sv{peer, nidx, orig, world};
	const uint32_t n_vtx = g.n_seq * 2;
	uint32_t n_reduced = 0;
	memset(&g_del_trans_stats, 0, sizeof(g_del_trans_stats));
	g_del_trans_stats.n_arc_in = g.n_arc, g_del_trans_stats.n_vtx = n_vtx;
	uint8_t *flag = nullptr;
	if (g.n_arc) {
		flag = mab_alloc<uint8_t>(d, g.n_arc);
		uint32_t *big = mab_alloc<uint32_t>(d, n_vtx);
		// no memset of flag[]: every arc lies in the slab of exactly one vertex, and every vertex with arcs writes its slab's flags
		MAB_CUDA(cudaMemsetAsync(d.d_scal, 0, 10 * sizeof(unsigned long long), d.stream));
		cudaEvent_t e0, e1;
		MAB_CUDA(cudaEventCreate(&e0)); MAB_CUDA(cudaEventCreate(&e1));
		MAB_CUDA(cudaEventRecord(e0, d.stream));
		unsigned grid = (n_vtx + DT_WARPS - 1) / DT_WARPS;
		if (grid > MAB_SMS * 64u) grid = MAB_SMS * 64u;
		// the inner-iteration counter (for the roofline arithmetic) costs issue slots: only counted when asked for
		{
			const bool st = mab_del_trans_count_inner != 0, p2p = peer != nullptr, srt = g.is_srt;
			#define DT(S, P, O) MAB_LAUNCH(d, (k_del_trans_warp<S, P, O>), grid, DT_WARPS * 32, 0, g.arc, g.idx, g.seq, n_vtx, fuzz, flag, big, d.d_scal, own_lo, own_hi, sv)
			if (st) { if (p2p) { if (srt) DT(true, true, true); else DT(true, true, false); } else { if (srt) DT(true, false, true); else DT(true, false, false); } }
			else { if (p2p) { if (srt) DT(false, true, true); else DT(false, true, false); } else { if (srt) DT(false, false, true); else DT(false, false, false); } }
			#undef DT
		}
		MAB_CUDA(cudaEventRecord(e1, d.stream));
		uint32_t n_big = (uint32_t)d.get_scal(SC_BIG);
		float ms = 0;
		MAB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
		g_del_trans_stats.kernel_ms = ms;
		MAB_CUDA(cudaEventDestroy(e0)); MAB_CUDA(cudaEventDestroy(e1));
		if (n_big) {
			MAB_CUDA(cudaFuncSetAttribute(k_del_trans_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DT_BIG_SMEM)); // per device: set on every use
			uint32_t *huge = mab_alloc<uint32_t>(d, n_big);
			MAB_LAUNCH(d, k_del_trans_cta, n_big < MAB_SMS * 2 ? n_big : MAB_SMS * 2, 256, DT_BIG_SMEM, g.arc, g.idx, fuzz, flag, big, n_big, huge, d.d_scal, sv);
			uint32_t n_huge = (uint32_t)d.get_scal(SC_AUX2);
			if (n_huge) {
				uint8_t *mark = mab_alloc<uint8_t>(d, n_vtx);
				uint32_t *first_pos = mab_alloc<uint32_t>(d, n_vtx);
				MAB_CUDA(cudaMemsetAsync(mark, 0, n_vtx, d.stream));
				MAB_CUDA(cudaMemsetAsync(first_pos, 0xff, (size_t)n_vtx * 4, d.stream));
				MAB_LAUNCH(d, k_del_trans_huge, 1, 1024, 0, g.arc, g.idx, fuzz, flag, huge, n_huge, mark, first_pos, d.d_scal, sv);
				d.free(mark); d.free(first_pos);
			}
			d.free(huge);
		}
		n_reduced = (uint32_t)d.get_scal(SC_COUNT);
		g_del_trans_stats.inner_iters = d.h_scal[SC_AUX];
		g_del_trans_stats.n_big = n_big;
		d.free(big);
	}
	g_del_trans_stats.n_reduced = n_reduced;
	*flag_out = flag;
	return n_reduced;
}

// ---------------------------------------------------------------------------------------------
// asg_arc_del_short (asg.c:83-101): per vertex with >= 2 arcs, thres = (uint32)(ol(first)*ratio + .499)
// (float product, double sum); the trailing run of arcs with ol < thres is deleted.
// ---------------------------------------------------------------------------------------------
__global__ void k_del_short(DArc *arc, const uint64_t *idx, uint32_t n_vtx, float ratio, unsigned long long *n_out)
{
	unsigned cnt = 0;
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) {
		uint64_t x = idx[v];
		uint32_t nv = (uint32_t)x, off = (uint32_t)(x >> 32);
		if (nv < 2) continue;
		int ol0 = (int)(arc[off].ol_del & ~MAB_DEL_BIT);
		float prod = __fmul_rn((float)ol0, ratio);
		uint32_t thres = (uint32_t)__dadd_rn((double)prod, .499);
		uint32_t i;
		for (i = nv - 1; i >= 1 && (arc[off + i].ol_del & ~MAB_DEL_BIT) < thres; --i);
		for (i = i + 1; i < nv; ++i) arc[off + i].ol_del |= MAB_DEL_BIT, ++cnt;
	}
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(n_out, (unsigned long long)cnt);
}

uint32_t dg_del_short(MabDev &d, DGraph &g, float ratio)
{
	uint32_t n_vtx = g.n_seq * 2, n_short = 0;
	if (n_vtx && g.n_arc) {
		d.zero_scal(SC_COUNT);
		MAB_LAUNCH(d, k_del_short, mab_grid(n_vtx, 256), 256, 0, g.arc, g.idx, n_vtx, ratio, d.d_scal + SC_COUNT);
		n_short = (uint32_t)d.get_scal(SC_COUNT);
	}
	if (n_short) {
		dg_cleanup(d, g);
		dg_symm(d, g);
	}
	if (MAB_V(1)) fprintf(stderr, "[M::%s] removed %d short overlaps\n", "asg_arc_del_short", n_short);
	return n_short;
}
