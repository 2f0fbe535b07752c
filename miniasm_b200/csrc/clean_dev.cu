// clean_dev.cu -- stage (iii) on the GPU: the order-dependent graph-cleaning passes (asg.c:238-306, 312-433), bit-exact
// with the reference's ascending-vertex sequential loops, and unitig construction (asm.c:121-210).
//
// The cleaning passes are the Jacobi iteration of clean_fix.cuh's timestamp fixed point: per sweep ONE kernel in which
// every vertex decides under T_old and stamps T_new with atomicMin, ONE kernel that compares the two and re-arms the
// old buffer, and one 8-byte read-back.  The sweep count is the length of the longest dependency chain of the pass
// (2-3 for bubbles, up to a few dozen for tips on the parity sets), not the number of actions.
#include "clean_dev.cuh"
#include "clean_fix.cuh"
#include <cub/cub.cuh>
#include <algorithm>

thread_local CleanStats g_clean_stats;
static inline void clean_note(uint32_t rounds, uint32_t committed)
{
	CleanStats &c = g_clean_stats;
	c.rounds = rounds, c.committed = committed;
	++c.passes, c.sum_rounds += rounds, c.sum_committed += committed;
	if (rounds > c.max_rounds) c.max_rounds = rounds;
}

struct GV { // device view of the graph (unitig construction)
	DArc *arc;
	const uint64_t *idx;
	uint32_t *seq;
	uint32_t n_vtx;
};

// ---------------------------------------------------------------------------------------------
// sweep machinery shared by the four passes
// ---------------------------------------------------------------------------------------------
struct FxBuf {
	uint32_t *ts[2], *ta[2];
	uint32_t n_seq, n_arc;
	int cur;
};

__global__ void k_fx_init(const DArc *arc, const uint32_t *seq, uint32_t n_arc, uint32_t n_seq, uint32_t *ts0, uint32_t *ts1, uint32_t *ta0, uint32_t *ta1)
{
	const uint32_t n = n_arc + n_seq;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (i < n_arc) ta0[i] = ta1[i] = arc[i].ol_del & MAB_DEL_BIT ? 0u : FX_LIVE;
		else { const uint32_t s = i - n_arc; ts0[s] = ts1[s] = seq[s] & MAB_DEL_BIT ? 0u : FX_LIVE; }
	}
}

template <class View, class Rule>
__global__ void k_fx_sweep(View g, Rule rule, unsigned long long *n_act)
{
	unsigned cnt = 0;
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x)
		cnt += rule.act(g, v);
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(n_act, (unsigned long long)cnt);
}

// changed |= T_old != T_new; T_old <- init (it is the T_new of the next sweep)
__global__ void k_fx_diff_rearm(const DArc *arc, const uint32_t *seq, uint32_t n_arc, uint32_t n_seq, uint32_t *ts_old, const uint32_t *ts_new,
                                uint32_t *ta_old, const uint32_t *ta_new, unsigned long long *changed)
{
	const uint32_t n = n_arc + n_seq;
	bool diff = false;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (i < n_arc) { diff |= ta_old[i] != ta_new[i]; ta_old[i] = arc[i].ol_del & MAB_DEL_BIT ? 0u : FX_LIVE; }
		else { const uint32_t s = i - n_arc; diff |= ts_old[s] != ts_new[s]; ts_old[s] = seq[s] & MAB_DEL_BIT ? 0u : FX_LIVE; }
	}
	if (__any_sync(0xffffffffu, diff) && (threadIdx.x & 31) == 0) atomicOr(changed, 1ull);
}

__global__ void k_fx_finish(DArc *arc, uint32_t *seq, uint32_t n_arc, uint32_t n_seq, const uint32_t *ts, const uint32_t *ta)
{
	const uint32_t n = n_arc + n_seq;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (i < n_arc) { if (ta[i] != FX_LIVE) arc[i].ol_del |= MAB_DEL_BIT; }
		else { const uint32_t s = i - n_arc; if (ts[s] != FX_LIVE) seq[s] |= MAB_DEL_BIT; }
	}
}

static void fx_alloc(MabDev &d, const DGraph &g, FxBuf &b)
{
	b.n_seq = g.n_seq, b.n_arc = g.n_arc, b.cur = 0;
	for (int k = 0; k < 2; ++k) b.ts[k] = mab_alloc<uint32_t>(d, g.n_seq), b.ta[k] = mab_alloc<uint32_t>(d, g.n_arc);
	MAB_LAUNCH(d, k_fx_init, mab_grid((size_t)g.n_arc + g.n_seq, 256), 256, 0, g.arc, g.seq, g.n_arc, g.n_seq, b.ts[0], b.ts[1], b.ta[0], b.ta[1]);
}
static FxView fx_view(const DGraph &g, const FxBuf &b)
{
	return FxView{g.arc, g.idx, b.ts[b.cur], b.ta[b.cur], b.ts[b.cur ^ 1], b.ta[b.cur ^ 1], g.n_seq * 2};
}
// end of a sweep: true if it changed nothing (then buffer `cur` holds the fixed point)
static bool fx_next(MabDev &d, const DGraph &g, FxBuf &b)
{
	d.zero_scal(SC_AUX2);
	MAB_LAUNCH(d, k_fx_diff_rearm, mab_grid((size_t)g.n_arc + g.n_seq, 256), 256, 0, g.arc, g.seq, g.n_arc, g.n_seq,
	           b.ts[b.cur], b.ts[b.cur ^ 1], b.ta[b.cur], b.ta[b.cur ^ 1], d.d_scal + SC_AUX2);
	b.cur ^= 1;
	return d.get_scal(SC_AUX2) == 0;
}
static void fx_finish(MabDev &d, DGraph &g, FxBuf &b)
{
	MAB_LAUNCH(d, k_fx_finish, mab_grid((size_t)g.n_arc + g.n_seq, 256), 256, 0, g.arc, g.seq, g.n_arc, g.n_seq, b.ts[b.cur], b.ta[b.cur]);
	for (int k = 0; k < 2; ++k) d.free(b.ts[k]), d.free(b.ta[k]);
}

template <class Rule>
static uint32_t run_fixpoint(MabDev &d, DGraph &g, Rule rule)
{
	if (g.n_seq == 0) { clean_note(0, 0); return 0; }                        // (a graph WITHOUT arcs still has work: every live read is a tip, asg.c:243-249)
	// probe: the first sweep straight on the deletion bits, stamping nothing.  Nobody acts -> the pass is over.
	d.zero_scal(SC_COUNT);
	MAB_LAUNCH(d, (k_fx_sweep<FxProbe, Rule>), mab_grid((size_t)g.n_seq * 2, 128), 128, 0, FxProbe{g.arc, g.idx, g.seq, g.n_seq * 2}, rule, d.d_scal + SC_COUNT);
	if (d.get_scal(SC_COUNT) == 0) { clean_note(1, 0); return 0; }
	FxBuf b;
	fx_alloc(d, g, b);
	uint32_t sweeps = 0, cnt;
	for (;;) {
		d.zero_scal(SC_COUNT);
		MAB_LAUNCH(d, (k_fx_sweep<FxView, Rule>), mab_grid((size_t)g.n_seq * 2, 128), 128, 0, fx_view(g, b), rule, d.d_scal + SC_COUNT);
		++sweeps;
		const bool fixed = fx_next(d, g, b);
		cnt = (uint32_t)d.h_scal[SC_COUNT];
		if (fixed) break;       // the sweep ran on the fixed point itself: its count is the reference's
	}
	fx_finish(d, g, b);
	clean_note(sweeps + 1, cnt);
	return cnt;
}

uint32_t dg_cut_tip(MabDev &d, DGraph &g, int max_ext)
{
	uint32_t cnt = run_fixpoint(d, g, FxTip{max_ext});
	if (cnt > 0) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] cut %d tips\n", "asg_cut_tip", cnt);
	return cnt;
}

uint32_t dg_cut_internal(MabDev &d, DGraph &g, int max_ext)
{
	uint32_t cnt = run_fixpoint(d, g, FxInternal{max_ext});
	if (cnt > 0) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] cut %d internal sequences\n", "asg_cut_internal", cnt);
	return cnt;
}

uint32_t dg_cut_biloop(MabDev &d, DGraph &g, int max_ext)
{
	uint32_t cnt = run_fixpoint(d, g, FxBiloop{max_ext});
	if (cnt > 0) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] cut %d small bi-loops\n", "asg_cut_biloop", cnt);
	return cnt;
}

// ---------------------------------------------------------------------------------------------
// Bubble popping (asg.c:312-433): one thread walks one source; its {p,d,c,r} map lives in a scratch slot in HBM.
// Only vertices with >= 2 arcs in the index can ever be sources (the pass only deletes): they are listed once.
// ---------------------------------------------------------------------------------------------
struct FxSlots {
	uint32_t *hkey, *hp, *hd, *hc, *hr;  // [n_slot][hcap]
	uint32_t *b, *bslot, *S;             // [n_slot][bcap]
	uint32_t *e;                         // [n_slot][ecap]
	uint32_t bcap, ecap, hcap, n_slot;
	__device__ FxSlot slot(uint32_t k) const
	{
		const size_t h = (size_t)k * hcap, q = (size_t)k * bcap, r = (size_t)k * ecap;
		return FxSlot{hkey + h, hp + h, hd + h, hc + h, hr + h, b + q, bslot + q, S + q, e + r, bcap, ecap, hcap - 1};
	}
};

__global__ void k_fx_bub_sources(const uint64_t *idx, const uint32_t *seq, uint32_t n_vtx, uint32_t *src, unsigned long long *n_src)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x)
		if ((uint32_t)idx[v] >= 2 && !(seq[v >> 1] & MAB_DEL_BIT)) src[atomicAdd(n_src, 1ull)] = v;
}

// counts[0] pops, [1] trimmed tips, [2] scratch overflows, [3] revived-a-dead-bit (pass not deletion-only)
__global__ void k_fx_bub_sweep(FxView g, uint32_t max_dist, FxSlots sl, const uint32_t *src, uint32_t n_src, unsigned long long *counts)
{
	const uint32_t k0 = blockIdx.x * blockDim.x + threadIdx.x;
	if (k0 >= sl.n_slot) return;
	const FxSlot s = sl.slot(k0);
	for (uint32_t k = k0; k < n_src; k += sl.n_slot) {
		uint32_t nt = 0;
		bool mono = true;
		const int r = fx_bub_act(g, src[k], max_dist, s, &nt, &mono);
		if (r == 1) {
			atomicAdd(&counts[0], 1ull);
			if (nt) atomicAdd(&counts[1], (unsigned long long)nt);
			if (!mono) atomicAdd(&counts[3], 1ull);
		} else if (r < 0) atomicAdd(&counts[2], 1ull);
	}
}

static void fx_slots_alloc(MabDev &d, FxSlots &sl, uint32_t n_slot, uint32_t bcap, uint32_t ecap)
{
	sl.n_slot = n_slot, sl.bcap = bcap, sl.ecap = ecap;
	sl.hcap = 1; while (sl.hcap < 2 * bcap) sl.hcap <<= 1;
	const size_t nh = (size_t)n_slot * sl.hcap, nb = (size_t)n_slot * sl.bcap, ne = (size_t)n_slot * sl.ecap;
	sl.hkey = mab_alloc<uint32_t>(d, nh); sl.hp = mab_alloc<uint32_t>(d, nh); sl.hd = mab_alloc<uint32_t>(d, nh);
	sl.hc = mab_alloc<uint32_t>(d, nh); sl.hr = mab_alloc<uint32_t>(d, nh);
	sl.b = mab_alloc<uint32_t>(d, nb); sl.bslot = mab_alloc<uint32_t>(d, nb); sl.S = mab_alloc<uint32_t>(d, nb);
	sl.e = mab_alloc<uint32_t>(d, ne);
	MAB_CUDA(cudaMemsetAsync(sl.hkey, 0xff, nh * 4, d.stream));
}

static void fx_slots_free(MabDev &d, FxSlots &sl)
{
	d.free(sl.hkey); d.free(sl.hp); d.free(sl.hd); d.free(sl.hc); d.free(sl.hr);
	d.free(sl.b); d.free(sl.bslot); d.free(sl.S); d.free(sl.e);
}

uint64_t dg_pop_bubble(MabDev &d, DGraph &g, int max_dist)
{
	const uint32_t n_vtx = g.n_seq * 2;
	uint64_t n_pop = 0, n_tip = 0;
	uint32_t sweeps = 0;
	if (!g.is_symm) dg_symm(d, g);
	if (n_vtx && g.n_arc) {
		uint32_t *src = mab_alloc<uint32_t>(d, n_vtx);
		d.zero_scal(SC_AUX);
		MAB_LAUNCH(d, k_fx_bub_sources, mab_grid(n_vtx, 256), 256, 0, g.idx, g.seq, n_vtx, src, d.d_scal + SC_AUX);
		const uint32_t n_src = (uint32_t)d.get_scal(SC_AUX);
		if (n_src) {
			FxBuf b;
			fx_alloc(d, g, b);
			FxSlots sl;
			uint32_t bcap = 64, ecap = 256, n_slot = n_src < 16384 ? (n_src + 63) / 64 * 64 : 16384;
			fx_slots_alloc(d, sl, n_slot, bcap, ecap);
			for (;;) {
				d.zero_scal(SC_TMP0, 4);
				MAB_LAUNCH(d, k_fx_bub_sweep, (sl.n_slot + 63) / 64, 64, 0, fx_view(g, b), (uint32_t)max_dist, sl, src, n_src, d.d_scal + SC_TMP0);
				if (d.get_scal(SC_TMP0 + 2)) { // a traversal outgrew its scratch slot: enlarge, re-arm T_new and redo the sweep
					// A walk visits each vertex other than its source at most once and scans each arc at most once, so with
					// bcap >= n_vtx and ecap >= n_arc no walk can overflow; the arc list grows with the arcs a walk scans,
					// which a dense graph makes far more than 4 per vertex, so each capacity grows up to its own bound.
					if (bcap >= n_vtx && ecap >= g.n_arc) { fprintf(stderr, "[E::miniasm_b200] bubble scratch overflow\n"); exit(75); }
					fx_slots_free(d, sl);
					bcap = (uint32_t)std::min<uint64_t>((uint64_t)bcap * 4, std::max(bcap, n_vtx));
					ecap = (uint32_t)std::min<uint64_t>((uint64_t)ecap * 4, std::max(ecap, g.n_arc));
					if (n_slot > 64) n_slot /= 4;
					fx_slots_alloc(d, sl, n_slot, bcap, ecap);
					MAB_LAUNCH(d, k_fx_init, mab_grid((size_t)g.n_arc + g.n_seq, 256), 256, 0, g.arc, g.seq, g.n_arc, g.n_seq,
					           b.ts[b.cur ^ 1], b.ts[b.cur ^ 1], b.ta[b.cur ^ 1], b.ta[b.cur ^ 1]);
					continue;
				}
				++sweeps;
				const bool fixed = fx_next(d, g, b);
				n_pop = d.h_scal[SC_TMP0], n_tip = d.h_scal[SC_TMP0 + 1];
				if (fixed) {
					if (d.h_scal[SC_TMP0 + 3]) { // asg_bub_backtrack would revive a bit deleted earlier: impossible on the symmetric,
						// multi-arc-free graph asg_pop_bubble works on; refuse rather than return a different graph
						fprintf(stderr, "[E::miniasm_b200] asg_pop_bubble: the graph is not symmetric (best path over a deleted arc)\n");
						exit(76);
					}
					break;
				}
			}
			fx_slots_free(d, sl);
			fx_finish(d, g, b);
		}
		d.free(src);
	}
	clean_note(sweeps, (uint32_t)n_pop);
	if (n_pop) dg_cleanup(d, g);
	if (MAB_V(1)) fprintf(stderr, "[M::%s] popped %d bubbles and trimmed %d tips\n", "asg_pop_bubble", (uint32_t)n_pop, (uint32_t)n_tip);
	return (n_pop & 0xffffffffull) | n_tip << 32;
}

// ---------------------------------------------------------------------------------------------
// ma_ug_gen (asm.c:121-210): unitigs = maximal chains of arcs w->x with out(w) == 1 and out(x^1) == 1.
//
// Sequential reference: scan v ascending; the first unvisited v with arcs seeds a unitig, walks forward to
// the chain end, then backward to the chain start, and marks both strands of everything on it.  Consequences
// used here: (1) every oriented vertex lies on exactly one chain of the successor function F (and the
// complement strand on the mirrored chain); (2) a chain pair {C, rc(C)} yields ONE unitig, oriented like the
// chain that holds the smallest seedable vertex (not deleted, has arcs) of C u rc(C), and unitigs are numbered
// by ascending seed; (3) a chain that closes on itself is circular and listed from its seed.
//
// GPU shape: F/B successor arrays -> pointer doubling along both directions (min seedable id, hop count and
// arc-length prefix sums to the chain head) -> seeds flagged, exclusive scans give unitig numbers and item
// offsets -> every vertex of an emitted chain writes its own item.  O(n log n) work, log n launches.
// The doubling needs F and B to be mutually inverse, which holds on a symmetric graph (every pass after
// transitive reduction leaves one); otherwise (e.g. `-S5 -p ug` on the raw graph) one thread replays the
// reference's walk literally.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t NONE = 0xffffffffu;

struct UgArrays {
	uint32_t *F, *B;          // successor / predecessor on the chain (NONE at the ends)
	uint32_t *jf, *jb;        // doubling pointers
	uint32_t *mf, *mb;        // min seedable vertex over the covered span, forward / backward
	uint32_t *rk;             // hops to the head (paths) or to the seed (cycles)
	uint64_t *ps;             // sum of arc lengths from the head/seed up to (excluding) this vertex
	uint32_t *cnt;            // hops to the tail, forward
	uint32_t *seedmin;        // min seedable vertex of the vertex's own chain
};

__device__ __forceinline__ uint32_t ug_fwd(const GV &g, uint32_t w)
{
	const uint64_t iw = g.idx[w];
	if ((uint32_t)iw != 1) return NONE;
	const uint32_t x = g.arc[iw >> 32].v;
	return (uint32_t)g.idx[x ^ 1] == 1 ? x : NONE;
}
__device__ __forceinline__ uint32_t ug_bwd(const GV &g, uint32_t x)
{
	const uint64_t ix = g.idx[x ^ 1];
	if ((uint32_t)ix != 1) return NONE;
	const uint32_t w = g.arc[ix >> 32].v ^ 1;
	return (uint32_t)g.idx[w] == 1 ? w : NONE;
}

__global__ void k_ug_links(GV g, uint32_t *F, uint32_t *B)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x)
		F[v] = ug_fwd(g, v), B[v] = ug_bwd(g, v);
}

__global__ void k_ug_consistent(uint32_t n_vtx, const uint32_t *F, const uint32_t *B, unsigned long long *bad)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) {
		bool ok = true;
		if (F[v] != NONE && B[F[v]] != v) ok = false;
		if (B[v] != NONE && F[B[v]] != v) ok = false;
		if (F[v] != NONE && F[v] == (v ^ 1)) ok = false; // a read chained to its own complement: let the literal walk handle it
		if (!ok) atomicAdd(bad, 1ull);
	}
}

__global__ void k_ug_init(GV g, UgArrays a)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x) {
		const bool seedable = !(g.seq[v >> 1] & MAB_DEL_BIT) && (uint32_t)g.idx[v] != 0;
		const uint32_t m = seedable ? v : NONE;
		a.jf[v] = a.F[v], a.jb[v] = a.B[v];
		a.mf[v] = m, a.mb[v] = m;
	}
}

// one doubling step for the minima (double-buffered by the caller through jf/jb + mf/mb copies)
__global__ void k_ug_min_step(uint32_t n_vtx, const uint32_t *jf, const uint32_t *jb, const uint32_t *mf, const uint32_t *mb,
                              uint32_t *jf2, uint32_t *jb2, uint32_t *mf2, uint32_t *mb2)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) {
		uint32_t f = jf[v], b = jb[v], x = mf[v], y = mb[v];
		if (f != NONE) { uint32_t t = mf[f]; x = t < x ? t : x; f = jf[f]; }
		if (b != NONE) { uint32_t t = mb[b]; y = t < y ? t : y; b = jb[b]; }
		jf2[v] = f, jb2[v] = b, mf2[v] = x, mb2[v] = y;
	}
}

// after the min doubling: seedmin = min(forward, backward); cycles are cut open just before their seed
__global__ void k_ug_cut(GV g, UgArrays a, const uint32_t *jb_final)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x) {
		const uint32_t m = a.mf[v] < a.mb[v] ? a.mf[v] : a.mb[v];
		a.seedmin[v] = m;
		// a vertex still holding a live backward pointer after ceil(log2 n)+1 doublings sits on a cycle
		const bool cyc = jb_final[v] != NONE;
		uint32_t b = a.B[v];
		if (cyc && v == m) b = NONE;               // the seed becomes the head of its (opened) cycle
		a.jb[v] = b;
		a.rk[v] = b == NONE ? 0 : 1;
		uint64_t l = 0;
		if (b != NONE) l = (uint32_t)g.arc[g.idx[b] >> 32].ul; // length of the arc b -> v (b has exactly one arc)
		a.ps[v] = l;
		uint32_t f = a.F[v];
		if (cyc && f == m) f = NONE;               // ... and its predecessor the tail
		a.jf[v] = f;
		a.cnt[v] = f == NONE ? 0 : 1;
	}
}

__global__ void k_ug_rank_step(uint32_t n_vtx, const uint32_t *jb, const uint32_t *rk, const uint64_t *ps, const uint32_t *jf, const uint32_t *cnt,
                               uint32_t *jb2, uint32_t *rk2, uint64_t *ps2, uint32_t *jf2, uint32_t *cnt2)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) {
		uint32_t b = jb[v], r = rk[v], f = jf[v], c = cnt[v];
		uint64_t p = ps[v];
		if (b != NONE) r += rk[b], p += ps[b], b = jb[b];
		if (f != NONE) c += cnt[f], f = jf[f];
		jb2[v] = b, rk2[v] = r, ps2[v] = p, jf2[v] = f, cnt2[v] = c;
	}
}

// head of an emitted chain: rank 0 and its chain wins over the mirrored chain (or is its own mirror)
__global__ void k_ug_heads(GV g, UgArrays a, const uint32_t *is_cyc, uint32_t *flag_seed, uint32_t *n_items_at_seed)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x) {
		// v is "the seed" iff it is the smallest seedable vertex of its chain pair and lies on the chain
		const uint32_t m = a.seedmin[v], mr = a.seedmin[v ^ 1];
		const bool seed = m != NONE && v == m && m < mr; // m == mr impossible: the two chains are disjoint vertex sets
		flag_seed[v] = seed;
		n_items_at_seed[v] = seed ? a.rk[v] + a.cnt[v] + 1 : 0; // chain length = hops to head + hops to tail + 1
	}
}

__global__ void k_ug_emit(GV g, UgArrays a, const uint32_t *is_cyc, const uint32_t *utg_of_seed, const uint32_t *first_of_seed,
                          uint64_t *items, DUtgMeta *meta)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < g.n_vtx; v += gridDim.x * blockDim.x) {
		const uint32_t m = a.seedmin[v];
		if (m == NONE || !(m < a.seedmin[v ^ 1])) continue; // chain not emitted in this orientation
		const uint32_t u = utg_of_seed[m];
		const bool cyc = is_cyc[v] != 0;
		const bool tail = a.cnt[v] == 0;
		uint32_t l;
		if (!tail || cyc) l = (uint32_t)g.arc[g.idx[v] >> 32].ul; // arc to the successor (for a cycle: also tail -> seed)
		else l = g.seq[v >> 1] & 0x7fffffffu;                       // the last read contributes its full length
		items[first_of_seed[m] + a.rk[v]] = (uint64_t)v << 32 | l;
		if (tail) { // the tail knows the total: prefix up to itself + its own item
			DUtgMeta mt;
			mt.len = (uint32_t)((a.ps[v] + l) & 0x7fffffffu);
			mt.circ = cyc;
			mt.n = a.rk[v] + 1;
			mt.first = first_of_seed[m];
			mt.end = cyc ? NONE : (v ^ 1);
			mt.start = NONE; // filled by the head below for linear unitigs
			meta[u].len = mt.len, meta[u].circ = mt.circ, meta[u].n = mt.n, meta[u].first = mt.first, meta[u].end = mt.end;
			if (cyc) meta[u].start = NONE;
		}
		if (a.rk[v] == 0 && !cyc) meta[u].start = v;
	}
}

// unitig-graph arcs (asm.c:181-202): an arc u->v of the read graph joins two unitigs when u^1 and v are unitig ends
__global__ void k_ug_mark(const DUtgMeta *meta, uint32_t n_utg, int32_t *mark)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_utg; i += gridDim.x * blockDim.x) {
		if (meta[i].circ) continue;
		// The sequential loop (asm.c:182-186) lets the last write win when walks on a non-symmetric graph share an end
		// vertex, or when start == end; "last" = larger unitig index, end after start = the larger value: atomicMax.
		atomicMax(&mark[meta[i].start], (int32_t)(i << 1 | 0));
		atomicMax(&mark[meta[i].end], (int32_t)(i << 1 | 1));
	}
}

__global__ void k_ug_arcs(const DArc *arc, uint32_t n_arc, const int32_t *mark, const DUtgMeta *meta, DArc *out, uint8_t *flag)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_arc; i += gridDim.x * blockDim.x) {
		const DArc p = arc[i];
		bool emit = false;
		if (!(p.ol_del & MAB_DEL_BIT)) {
			const int32_t mu = mark[(uint32_t)(p.ul >> 32) ^ 1], mv = mark[p.v];
			if (mu >= 0 && mv >= 0) {
				const uint32_t u = (uint32_t)mu ^ 1, ol = p.ol_del & 0x7fffffffu;
				int l = (int)(meta[u >> 1].len - ol);
				if (l < 0) l = 1;
				DArc q;
				q.ul = (uint64_t)u << 32 | (uint32_t)l, q.v = (uint32_t)mv, q.ol_del = ol;
				out[i] = q;
				emit = true;
			}
		}
		flag[i] = emit;
	}
}

__global__ void k_ug_seq(const DUtgMeta *meta, uint32_t n_utg, uint32_t *seq)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_utg; i += gridDim.x * blockDim.x) seq[i] = meta[i].len & 0x7fffffffu;
}

__global__ void k_ug_cycflag(uint32_t n_vtx, const uint32_t *jb_final, uint32_t *is_cyc)
{
	for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_vtx; v += gridDim.x * blockDim.x) is_cyc[v] = jb_final[v] != NONE;
}

// Literal replay of asm.c:121-178 by one thread: used when F and B are not mutually inverse.
__global__ void k_ug_literal(GV g, int32_t *mark, uint64_t *items, uint64_t cap, uint64_t *tmp, DUtgMeta *meta, unsigned long long *out_counts)
{
	if (blockIdx.x || threadIdx.x) return;
	uint32_t n_utg = 0;
	uint64_t n_items = 0;
	out_counts[2] = 0;
	for (uint32_t v = 0; v < g.n_vtx; ++v) {
		if (n_items + 2ull * g.n_vtx + 2 > cap) { out_counts[2] = 1; break; } // overlapping walks outgrew the buffer
		if ((g.seq[v >> 1] & MAB_DEL_BIT) || (uint32_t)g.idx[v] == 0 || mark[v]) continue;
		mark[v] = 1;
		uint32_t start = v, end = v ^ 1, len = 0, w = v, x, l;
		uint64_t nf = 0, nb = 0; // forward items go to items[n_items..], backward items to tmp[] (reversed later)
		while (1) {
			if ((uint32_t)g.idx[w] != 1) break;
			x = g.arc[g.idx[w] >> 32].v;
			if ((uint32_t)g.idx[x ^ 1] != 1) break;
			mark[x] = mark[w ^ 1] = 1;
			l = (uint32_t)g.arc[g.idx[w] >> 32].ul;
			items[n_items + nf++] = (uint64_t)w << 32 | l;
			end = x ^ 1, len += l;
			w = x;
			if (x == v) break;
		}
		bool circ = false;
		if (start != (end ^ 1) || nf == 0) {
			l = g.seq[end >> 1] & 0x7fffffffu;
			items[n_items + nf++] = (uint64_t)(end ^ 1) << 32 | l;
			len += l;
			x = v;
			while (1) {
				if ((uint32_t)g.idx[x ^ 1] != 1) break;
				w = g.arc[g.idx[x ^ 1] >> 32].v ^ 1;
				if ((uint32_t)g.idx[w] != 1) break;
				mark[x] = mark[w ^ 1] = 1;
				l = (uint32_t)g.arc[g.idx[w] >> 32].ul;
				tmp[nb++] = (uint64_t)w << 32 | l;
				start = w, len += l;
				x = w;
			}
		} else circ = true, start = end = NONE;
		if (start != NONE) mark[start] = mark[end] = 1;
		if (nb) { // prepend the backward items in walk-reversed order
			for (uint64_t k = nf; k-- > 0;) items[n_items + nb + k] = items[n_items + k];
			for (uint64_t k = 0; k < nb; ++k) items[n_items + k] = tmp[nb - 1 - k];
		}
		DUtgMeta mt;
		mt.len = len & 0x7fffffffu, mt.circ = circ, mt.start = start, mt.end = end, mt.n = (uint32_t)(nf + nb), mt.first = (uint32_t)n_items;
		meta[n_utg++] = mt;
		n_items += nf + nb;
	}
	out_counts[0] = n_utg, out_counts[1] = n_items;
}

void dg_ug_free(MabDev &d, DUnitigs &ug)
{
	d.free(ug.meta); d.free(ug.items);
	dg_free(d, ug.g);
	ug = DUnitigs();
}

void dg_ug_gen(MabDev &d, const DGraph &g, DUnitigs &ug)
{
	const uint32_t n_vtx = g.n_seq * 2;
	ug = DUnitigs();
	GV gv{g.arc, g.idx, g.seq, n_vtx};
	if (n_vtx) {
		const unsigned grid = mab_grid(n_vtx, 256);
		UgArrays a;
		a.F = mab_alloc<uint32_t>(d, n_vtx); a.B = mab_alloc<uint32_t>(d, n_vtx);
		MAB_LAUNCH(d, k_ug_links, grid, 256, 0, gv, a.F, a.B);
		d.zero_scal(SC_COUNT);
		MAB_LAUNCH(d, k_ug_consistent, grid, 256, 0, n_vtx, a.F, a.B, d.d_scal + SC_COUNT);
		const bool consistent = d.get_scal(SC_COUNT) == 0;
		if (consistent) {
			uint32_t *buf[12];
			for (int i = 0; i < 12; ++i) buf[i] = mab_alloc<uint32_t>(d, n_vtx);
			uint64_t *ps_buf0 = mab_alloc<uint64_t>(d, n_vtx), *ps_buf1 = mab_alloc<uint64_t>(d, n_vtx);
			uint64_t *ps = ps_buf0, *ps2 = ps_buf1;
			a.jf = buf[0], a.jb = buf[1], a.mf = buf[2], a.mb = buf[3];
			uint32_t *jf2 = buf[4], *jb2 = buf[5], *mf2 = buf[6], *mb2 = buf[7];
			a.rk = buf[8], a.cnt = buf[9], a.seedmin = buf[10];
			uint32_t *is_cyc = buf[11];
			a.ps = ps;
			MAB_LAUNCH(d, k_ug_init, grid, 256, 0, gv, a);
			int steps = 1; while ((1ull << steps) < (uint64_t)n_vtx + 1) ++steps;
			++steps;
			for (int s = 0; s < steps; ++s) {
				MAB_LAUNCH(d, k_ug_min_step, grid, 256, 0, n_vtx, a.jf, a.jb, a.mf, a.mb, jf2, jb2, mf2, mb2);
				uint32_t *t;
				t = a.jf, a.jf = jf2, jf2 = t; t = a.jb, a.jb = jb2, jb2 = t;
				t = a.mf, a.mf = mf2, mf2 = t; t = a.mb, a.mb = mb2, mb2 = t;
			}
			// a.jb now: NONE for path vertices, still live for cycle vertices
			MAB_LAUNCH(d, k_ug_cycflag, grid, 256, 0, n_vtx, a.jb, is_cyc);
			uint32_t *jb_final = jb2; // reuse: copy the final jb aside because k_ug_cut overwrites a.jb
			MAB_CUDA(cudaMemcpyAsync(jb_final, a.jb, (size_t)n_vtx * 4, cudaMemcpyDeviceToDevice, d.stream));
			MAB_LAUNCH(d, k_ug_cut, grid, 256, 0, gv, a, jb_final);
			uint32_t *rk2 = mf2, *cnt2 = mb2; // the min buffers are free now (values kept in seedmin)
			for (int s = 0; s < steps; ++s) {
				MAB_LAUNCH(d, k_ug_rank_step, grid, 256, 0, n_vtx, a.jb, a.rk, a.ps, a.jf, a.cnt, jb2, rk2, ps2, jf2, cnt2);
				uint32_t *t; uint64_t *t8;
				t = a.jb, a.jb = jb2, jb2 = t; t = a.rk, a.rk = rk2, rk2 = t; t8 = a.ps, a.ps = ps2, ps2 = t8;
				t = a.jf, a.jf = jf2, jf2 = t; t = a.cnt, a.cnt = cnt2, cnt2 = t;
			}
			// seeds -> unitig numbers and item offsets
			uint32_t *flag_seed = jb2, *n_at_seed = jf2, *utg_of = rk2, *first_of = cnt2;
			MAB_LAUNCH(d, k_ug_heads, grid, 256, 0, gv, a, is_cyc, flag_seed, n_at_seed);
			size_t tb = 0, tb2 = 0;
			cub::DeviceScan::ExclusiveSum(nullptr, tb, flag_seed, utg_of, (int)n_vtx, d.stream);
			cub::DeviceScan::ExclusiveSum(nullptr, tb2, n_at_seed, first_of, (int)n_vtx, d.stream);
			void *tmp = d.tmp(tb > tb2 ? tb : tb2);
			cub::DeviceScan::ExclusiveSum(tmp, tb, flag_seed, utg_of, (int)n_vtx, d.stream);
			cub::DeviceScan::ExclusiveSum(tmp, tb2, n_at_seed, first_of, (int)n_vtx, d.stream);
			d.n_lib += 2;
			uint32_t last[4];
			MAB_CUDA(cudaMemcpyAsync(&last[0], flag_seed + n_vtx - 1, 4, cudaMemcpyDeviceToHost, d.stream));
			MAB_CUDA(cudaMemcpyAsync(&last[1], utg_of + n_vtx - 1, 4, cudaMemcpyDeviceToHost, d.stream));
			MAB_CUDA(cudaMemcpyAsync(&last[2], n_at_seed + n_vtx - 1, 4, cudaMemcpyDeviceToHost, d.stream));
			MAB_CUDA(cudaMemcpyAsync(&last[3], first_of + n_vtx - 1, 4, cudaMemcpyDeviceToHost, d.stream));
			d.sync();
			ug.n_utg = last[0] + last[1];
			ug.n_items = (uint64_t)last[2] + last[3];
			ug.meta = mab_alloc<DUtgMeta>(d, ug.n_utg);
			ug.items = mab_alloc<uint64_t>(d, ug.n_items);
			if (ug.n_utg) MAB_LAUNCH(d, k_ug_emit, grid, 256, 0, gv, a, is_cyc, utg_of, first_of, ug.items, ug.meta);
			for (int i = 0; i < 12; ++i) d.free(buf[i]);
			d.free(ps_buf0); d.free(ps_buf1);
		} else {
			int32_t *mark = mab_alloc<int32_t>(d, n_vtx);
			MAB_CUDA(cudaMemsetAsync(mark, 0, (size_t)n_vtx * 4, d.stream));
			ug.meta = mab_alloc<DUtgMeta>(d, n_vtx);
			const uint64_t cap = (uint64_t)n_vtx * 6 + 8;
			ug.items = mab_alloc<uint64_t>(d, cap);
			uint64_t *tmp = mab_alloc<uint64_t>(d, (size_t)n_vtx + 1);
			MAB_LAUNCH(d, k_ug_literal, 1, 32, 0, gv, mark, ug.items, cap, tmp, ug.meta, d.d_scal + SC_TMP0);
			ug.n_utg = (uint32_t)d.get_scal(SC_TMP0);
			ug.n_items = d.h_scal[SC_TMP0 + 1];
			if (d.h_scal[SC_TMP0 + 2]) { fprintf(stderr, "[E::miniasm_b200] ma_ug_gen: unitig walks on a non-symmetric graph outgrew the item buffer\n"); exit(76); }
			d.free(mark); d.free(tmp);
		}
		d.free(a.F); d.free(a.B);
	}
	// unitig graph
	DGraph &q = ug.g;
	dg_set_nseq(d, q, ug.n_utg);
	dg_reserve(d, q, g.n_arc ? g.n_arc : 1);
	q.n_arc = 0, q.is_srt = false, q.is_symm = false, q.len_bits = 32;
	if (ug.n_utg) {
		MAB_LAUNCH(d, k_ug_seq, mab_grid(ug.n_utg, 256), 256, 0, ug.meta, ug.n_utg, q.seq);
		if (g.n_arc) {
			int32_t *mark = mab_alloc<int32_t>(d, n_vtx);
			uint8_t *flag = mab_alloc<uint8_t>(d, g.n_arc);
			MAB_CUDA(cudaMemsetAsync(mark, 0xff, (size_t)n_vtx * 4, d.stream));
			MAB_LAUNCH(d, k_ug_mark, mab_grid(ug.n_utg, 256), 256, 0, ug.meta, ug.n_utg, mark);
			MAB_LAUNCH(d, k_ug_arcs, mab_grid(g.n_arc, 256), 256, 0, g.arc, g.n_arc, mark, ug.meta, q.arc2, flag);
			size_t tb = 0;
			unsigned long long *d_n = d.d_scal + SC_NSEL;
			cub::DeviceSelect::Flagged(nullptr, tb, q.arc2, flag, q.arc, d_n, (int)g.n_arc, d.stream);
			void *tmp = d.tmp(tb);
			cub::DeviceSelect::Flagged(tmp, tb, q.arc2, flag, q.arc, d_n, (int)g.n_arc, d.stream);
			++d.n_lib;
			q.n_arc = (uint32_t)d.get_scal(SC_NSEL);
			d.free(mark); d.free(flag);
		}
	}
	dg_cleanup(d, q);
}
