// ingest_dev.cu -- GPU ingest of PAF text (the reference spends 55-60 % of its wall time here, SURVEY.md 3.1).
//
// Reference semantics reproduced (paf.c:34-67, kseq.h:101-149, hit.c:82-104, sdict.c:27-45):
//   * lines end at '\n'; one trailing '\r' is dropped when the line is longer than one byte;
//   * fields split on TAB; columns 2-4,7-11 via strtol(.,10) truncated to uint32 (ml to 31 bits);
//     rev = first byte of column 5 is '-'; fewer than 10 fields -> line skipped; exactly 10 fields -> bl is
//     whatever the last line with an 11th field left behind;
//   * a line is stored iff qe-qs >= min_span && te-ts >= min_span (unsigned) && ml >= min_match;
//   * read ids = order of first appearance among stored lines, query name before target name; the length
//     kept for a read is the one seen at that first appearance;
//   * every stored line yields a hit and, when bi_dir and query != target, the mirrored hit right after it;
//   * hits sorted by (query id, query start).
//
// GPU shape: (1) line starts (per 8 KB tile, numbered by a decoupled look-back over the tiles) and (2) one thread per line parses
// it, applies the store filter, enters both names into an exact open-addressing dictionary (slot word = hash fragment + byte offset
// of a witness occurrence: an occurrence with the same fragment compares its bytes with the witness's; value = smallest occurrence
// number, atomicMin) and counts the line's hits per slot -- all in ONE pass over the text that leaves a 32-byte record per line,
// (3) distinct names ranked by first occurrence = ids, the slot counts become per-read counts, (4) every hit emitted straight into
// its read's bucket, (5) each bucket sorted (dh_sort_buckets, hit_dev.cu).  ingest_paf_stream runs (1)-(2) chunk by chunk while
// the next chunks of the text are still crossing PCIe.
#include "ingest_dev.cuh"
#include "shard_comm.cuh"
#include <cub/cub.cuh>

struct PLine {                 // one parsed PAF line, in registers only
	uint32_t ql, qs, qe, tl, ts, te, ml_rev, bl;
	uint32_t tdelta;           // target name offset from the line start
	uint32_t qnl, tnl;         // name lengths
	uint32_t nf;               // number of fields (capped at 11)
};

// What a line leaves in HBM: 32 bytes.  The names went into the dictionary while the line was still in shared memory.
struct __align__(16) PRec {
	uint32_t qs, qe, ts, te;
	uint32_t ml_rev;           // ml:31 | rev << 31
	uint32_t bl_f;             // bl:31 | (the line has an 11th field) << 31
	uint32_t slot_q, slot_t;   // dictionary slots of the two names; slot_q == NOSLOT: the line is not stored
};
static_assert(sizeof(PRec) == 32, "PRec layout");
constexpr uint32_t NOSLOT = 0xffffffffu;

// ---- line starts -----------------------------------------------------------------------------------------
// (dev_line_starts, for the reads file of -f in ugseq_dev.cu; the PAF parse finds its own lines, k_parse_tiles below.)
// A line starts at byte 0 and after every '\n' that is not the last byte.  Tiles of NL_TILE bytes, one CTA each,
// 128-bit loads laid out so that a warp reads 512 contiguous bytes per instruction.
constexpr int NL_THREADS = 256;
constexpr int NL_PER_THREAD = 4;                      // uint4 words per thread
constexpr uint64_t NL_TILE = (uint64_t)NL_THREADS * NL_PER_THREAD * 16;

__device__ __forceinline__ uint32_t nl_mask4(uint32_t w) { return __vcmpeq4(w, 0x0a0a0a0au); } // 0xff in every byte equal to '\n'

// newline bytes of the 16-byte word at `off` that are followed by another byte of the text; bit k = byte k
__device__ __forceinline__ uint32_t nl_bits16(const char *text, size_t len, uint64_t off)
{
	if (off >= len) return 0;
	uint32_t bits = 0;
	if (off + 16 <= len) {
		const uint4 w = __ldg(reinterpret_cast<const uint4*>(text + off));
		const uint32_t m[4] = { nl_mask4(w.x), nl_mask4(w.y), nl_mask4(w.z), nl_mask4(w.w) };
		#pragma unroll
		for (int k = 0; k < 4; ++k) bits |= ((m[k] & 1) | (m[k] >> 7 & 2) | (m[k] >> 14 & 4) | (m[k] >> 21 & 8)) << (4 * k);
	} else for (uint64_t k = 0; off + k < len; ++k) bits |= (uint32_t)(text[off + k] == '\n') << k;
	if (off + 16 >= len && len - 1 - off < 16) bits &= ~(1u << (len - 1 - off)); // a newline ending the file starts no line
	return bits;
}

__global__ void __launch_bounds__(NL_THREADS) k_nl_count(const char *__restrict__ text, size_t len, uint64_t n_tile, uint64_t *cnt)
{
	typedef cub::BlockReduce<uint32_t, NL_THREADS> BR;
	__shared__ typename BR::TempStorage ts;
	for (uint64_t t = blockIdx.x; t < n_tile; t += gridDim.x) {
		uint32_t c = 0;
		#pragma unroll
		for (int k = 0; k < NL_PER_THREAD; ++k) c += __popc(nl_bits16(text, len, t * NL_TILE + ((uint64_t)k * NL_THREADS + threadIdx.x) * 16));
		c = BR(ts).Sum(c);
		if (threadIdx.x == 0) cnt[t] = c;
		__syncthreads();
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) cnt[n_tile] = 0;
}

__global__ void __launch_bounds__(NL_THREADS) k_nl_write(const char *__restrict__ text, size_t len, uint64_t n_tile, const uint64_t *__restrict__ base, uint64_t *out)
{
	typedef cub::BlockScan<uint32_t, NL_THREADS> BS;
	__shared__ typename BS::TempStorage ts;
	for (uint64_t t = blockIdx.x; t < n_tile; t += gridDim.x) {
		uint64_t at = base[t];
		#pragma unroll
		for (int k = 0; k < NL_PER_THREAD; ++k) {
			const uint64_t off = t * NL_TILE + ((uint64_t)k * NL_THREADS + threadIdx.x) * 16;
			uint32_t bits = nl_bits16(text, len, off), rank, total;
			BS(ts).ExclusiveSum((uint32_t)__popc(bits), rank, total);
			uint64_t *o = out + at + rank;
			while (bits) { const int b = __ffs(bits) - 1; *o++ = off + b + 1; bits &= bits - 1; }
			at += total;
			__syncthreads();
		}
	}
}

// strtol(field, 0, 10) narrowed to uint32, on the byte range [p, e).  Up to 18 significant digits cannot
// overflow a long, so the common path is one multiply-add per digit; only longer digit strings take the clamping
// path (LONG_MAX / LONG_MIN, then truncation to 32 bits, as the reference's assignment does).
__host__ __device__ __forceinline__ uint32_t field_to_u32(const char *p, const char *e)
{
	while (p < e && (*p == ' ' || (*p >= '\t' && *p <= '\r'))) ++p;
	bool neg = false;
	if (p < e && (*p == '-' || *p == '+')) neg = *p == '-', ++p;
	while (p < e && *p == '0') ++p;                    // leading zeros carry no value
	unsigned long long v = 0;
	int nd = 0;
	for (; p < e; ++p, ++nd) {
		const unsigned dgt = (unsigned)(*p - '0');
		if (dgt > 9) break;
		if (nd < 18) { v = v * 10 + dgt; continue; }
		const unsigned long long lim = neg ? 9223372036854775808ull : 9223372036854775807ull; // rare: 19+ digits
		if (v > (lim - dgt) / 10) { v = lim; while (p < e && (unsigned)(*p - '0') <= 9) ++p; break; }
		v = v * 10 + dgt;
	}
	const long long sv = neg ? (long long)(0ull - v) : (long long)v;
	return (uint32_t)sv;
}

// bit k set iff byte k of the little-endian word is a TAB
__host__ __device__ __forceinline__ uint32_t tab_bits4(uint32_t w)
{
#ifdef __CUDA_ARCH__
	const uint32_t m = __vcmpeq4(w, 0x09090909u);
	return (m & 1) | (m >> 7 & 2) | (m >> 14 & 4) | (m >> 21 & 8);
#else
	uint32_t b = 0;
	for (int k = 0; k < 4; ++k) if (((w >> (8 * k)) & 0xffu) == 9u) b |= 1u << k;
	return b;
#endif
}

// decimal field [s, t) of the line at p: the plain case (1..9 digits, nothing else) is one multiply-add per byte in
// 32 bits; anything else (sign, blanks, junk, long digit strings) goes through the exact strtol restatement
__host__ __device__ __forceinline__ uint32_t num_field(const char *p, uint32_t s, uint32_t t)
{
	uint32_t v = 0;
	bool plain = t > s && t - s <= 9;
	for (uint32_t i = s; plain && i < t; ++i) {
		const unsigned dgt = (unsigned)((unsigned char)p[i] - '0');
		plain = dgt <= 9;
		v = v * 10 + dgt;
	}
	return plain ? v : field_to_u32(p + s, p + t);
}

// Parse one line [p, e) (no terminator, '\r' already dropped), one thread per line.
// Pass 1 finds the first 11 TABs a 32-bit word at a time (SWAR compare, positions parked in shared memory);
// pass 2 converts each column from its known byte range.  Byte-at-a-time loops cost ~170 warp instructions per line
// because the 32 lines of a warp sit in different columns at every step; with the boundaries known up front the
// per-column loops are short and uniform.
// Semantics: columns split on TAB only; numbers follow strtol(.,10) truncated to 32 bits (ml to 31); rev = first
// byte of column 5 is '-'.  tab: this lane's column of an [11][32] shared scratch.
__host__ __device__ __forceinline__ void parse_line(const char *p, const char *e, PLine &r, uint32_t *tab)
{
	const uint32_t len = (uint32_t)(e - p);
	uint32_t nt = 0;
	{
		const uintptr_t a = (uintptr_t)p & ~(uintptr_t)3;
		const int lead = (int)((uintptr_t)p - a);                // bytes of the first word that precede the line
		for (int off = -lead; off < (int)len && nt < 11; off += 4) {
			uint32_t bits = tab_bits4(*reinterpret_cast<const uint32_t*>(p + off));
			while (bits) {
#ifdef __CUDA_ARCH__
				const int pos = off + __ffs(bits) - 1;
#else
				const int pos = off + __builtin_ctz(bits);
#endif
				bits &= bits - 1;
				if (pos >= 0 && pos < (int)len && nt < 11) tab[nt++ * 32] = (uint32_t)pos;
			}
		}
	}
	const uint32_t nf = nt + 1 < 11 ? nt + 1 : 11;           // columns seen, capped (only the first 11 matter)
	#define COL_S(k) ((k) ? tab[((k) - 1) * 32] + 1 : 0u)
	#define COL_T(k) ((uint32_t)(k) < nt ? tab[(k) * 32] : len)
	memset(&r, 0, sizeof(r));
	r.nf = nf;
	r.qnl = COL_T(0);
	if (nf > 1) r.ql = num_field(p, COL_S(1), COL_T(1));
	if (nf > 2) r.qs = num_field(p, COL_S(2), COL_T(2));
	if (nf > 3) r.qe = num_field(p, COL_S(3), COL_T(3));
	if (nf > 4) { const uint32_t s4 = COL_S(4); r.ml_rev = (COL_T(4) > s4 && p[s4] == '-') ? 0x80000000u : 0; }
	if (nf > 5) {
		const uint32_t s5 = COL_S(5), t5 = COL_T(5);
		r.tnl = t5 - s5, r.tdelta = s5;
	}
	if (nf > 6) r.tl = num_field(p, COL_S(6), COL_T(6));
	if (nf > 7) r.ts = num_field(p, COL_S(7), COL_T(7));
	if (nf > 8) r.te = num_field(p, COL_S(8), COL_T(8));
	if (nf > 9) r.ml_rev |= num_field(p, COL_S(9), COL_T(9)) & 0x7fffffffu;
	if (nf > 10) r.bl = num_field(p, COL_S(10), COL_T(10));
	#undef COL_S
	#undef COL_T
}

// --------------------------------------------------------------------------------------------- dictionary
// Open addressing, one 64-bit word per slot: [hash fragment : 27][byte offset of a WITNESS occurrence of the name + 1 : 37].
// An occurrence that finds a slot with its fragment compares its bytes with the witness's bytes in the text (both names
// end at a TAB): equal -> same name, same slot; different -> a true collision of the fragment, it simply probes on.
// The table is therefore exact without a verification pass or a re-seeded retry.  first[slot] = smallest occurrence
// number (2*line + {0 query, 1 target}) among the stored lines: the read's rank by it is its id (hit.c:87-90).
struct NameTab {
	unsigned long long *key;
	unsigned long long *first;
	uint32_t *id;                // read id of the slot (after ranking)
	uint64_t mask;
	uint32_t *hits = nullptr;    // optional: hits whose query read is the slot's name (the bucket sizes of the hit sort)
};
constexpr int NT_OFF_BITS = 37;
constexpr unsigned long long NT_OFF_MASK = (1ull << NT_OFF_BITS) - 1;

// name = nm[0 .. nl) (shared or global memory), followed by a TAB; goff = its byte offset in `text`
__device__ __forceinline__ uint32_t tab_insert(const NameTab &t, const char *__restrict__ text, const char *nm, uint32_t nl, uint64_t goff, uint64_t occ,
                                               unsigned long long *overflow)
{
	const uint64_t h = name_hash(nm, 0, nl, 0);
	const unsigned long long mine = (h >> 37) << NT_OFF_BITS | (goff + 1);
	uint64_t s = h & t.mask;
	for (int probe = 0; probe < 1 << 14; ++probe, s = (s + 1) & t.mask) {
		unsigned long long k = t.key[s];
		if (k == 0) {
			k = atomicCAS(&t.key[s], 0ull, mine);
			if (k == 0) k = mine;
		}
		if ((k ^ mine) >> NT_OFF_BITS) continue;                      // another fragment
		bool same = k == mine;
		if (!same) {
			const char *w = text + ((k & NT_OFF_MASK) - 1);
			same = true;
			for (uint32_t i = 0; same && i < nl; ++i) same = w[i] == nm[i];
			same = same && w[nl] == '\t';
		}
		if (!same) continue;
		if (t.first[s] > occ) atomicMin(&t.first[s], (unsigned long long)occ); // values only decrease: the plain read filters most atomics
		return (uint32_t)s;
	}
	atomicAdd(overflow, 1ull);
	return 0;
}

// ---- the parse: one pass over the text finds the lines, numbers them, parses them and enters their names ------------
// The text is cut into tiles of PT_TILE bytes.  Line 0 belongs to tile 0 and every other line to the tile that holds the
// '\n' ending the line before it.  A CTA takes the next tile from a counter, so tiles start in index order and the
// look-back below only ever waits on tiles that are already running.  The CTA
//   * stages its tile and PT_OVER bytes after it in shared memory with 128-bit loads (byte-wise walking of global
//     memory makes every warp-level load touch ~16 cache lines),
//   * counts the line starts of the tile there and publishes the count; a single-pass decoupled look-back over the
//     tiles (cub::TilePrefixCallbackOp) returns the global number of its first line,
//   * lists the starts and hands one line to each thread, which parses it, applies the store filter of hit.c:85 and
//     enters both names into the dictionary while the line is still in shared memory, then writes start[line] and the
//     32-byte record, and (optionally) adds the line's hits to the bucket sizes of its slots.
// The tile's last line is the only one that can end past the staged bytes: it is parsed straight from global memory.
// Lines numbered line_cap or more are counted but not parsed (the host parses again with room for all of them).
constexpr int PT_THREADS = 128;
constexpr uint32_t PT_TILE = 8192;
constexpr uint32_t PT_OVER = 1024;
constexpr uint32_t PT_LIST = 1024;                       // line starts listed at once: a tile with more lines is parsed in rounds
static_assert(PT_TILE == PT_THREADS * 64, "each thread scans 64 bytes of its tile for line starts");
static_assert(PT_OVER % 16 == 0 && PT_OVER <= PT_TILE, "the overhang ends inside the tile after the parsed ones");

typedef cub::ScanTileState<unsigned long long> LineTileState;
typedef cub::TilePrefixCallbackOp<unsigned long long, ::cuda::std::plus<unsigned long long>, LineTileState> LinePrefixOp;

// counts[]: [0] lines with >= 10 fields, [1] lines stored, [2] dictionary overflow, [3] lines of the text (set by its last tile),
// [4] lines that run past the bytes that have arrived
enum { PC_PARSED = 0, PC_STORED, PC_OVERFLOW, PC_LINES, PC_CUT, PC_N };

__device__ __forceinline__ uint32_t nl_bits_u4(const uint4 w)  // bit k = byte k of the 16 bytes is '\n'
{
	const uint32_t m[4] = { nl_mask4(w.x), nl_mask4(w.y), nl_mask4(w.z), nl_mask4(w.w) };
	uint32_t bits = 0;
	#pragma unroll
	for (int k = 0; k < 4; ++k) bits |= ((m[k] & 1) | (m[k] >> 7 & 2) | (m[k] >> 14 & 4) | (m[k] >> 21 & 8)) << (4 * k);
	return bits;
}

__global__ void k_tiles_init(LineTileState ts, int n_tile) { ts.InitializeStatus(n_tile); }

// Tiles [t_lo, t_lo + gridDim.x) of the text, one per CTA.  avail: bytes of the text present (== len unless the text is still
// arriving, and then at least PT_TILE past the last tile of the launch).
__global__ void __launch_bounds__(PT_THREADS)
k_parse_tiles(const char *__restrict__ text, size_t len, size_t avail, uint64_t t_lo, unsigned *tile_ctr, LineTileState tstate,
              int min_span, int min_match, int bi_dir, NameTab tab, PRec *out, uint64_t *start, uint64_t line_cap, unsigned long long *counts)
{
	typedef cub::BlockScan<uint32_t, PT_THREADS> BS;
	__shared__ __align__(16) char s_text[PT_TILE + PT_OVER + 16];  // (+16: parse_line reads whole aligned words)
	__shared__ uint16_t s_start[PT_LIST + 1];                      // line starts, offsets from the tile's first byte
	__shared__ uint32_t s_vals[PT_THREADS / 32][11][32];
	__shared__ typename BS::TempStorage s_scan;
	__shared__ typename LinePrefixOp::TempStorage s_pref;
	__shared__ unsigned long long s_first, s_tile, s_eol;
	__shared__ uint32_t s_nl;
	const uint32_t lane = threadIdx.x & 31;
	if (threadIdx.x == 0) s_tile = t_lo + atomicAdd(tile_ctr, 1u), s_nl = ~0u;
	__syncthreads();
	const uint64_t t = s_tile, b0 = t * PT_TILE, b1 = b0 + PT_TILE < len ? b0 + PT_TILE : len;
	const uint64_t w_end = b1 + PT_OVER < avail ? b1 + PT_OVER : avail;       // staged bytes: [b0, w_end)
	{
		const uint32_t n16 = (uint32_t)((w_end - b0 + 15) >> 4);  // the tail word may reach past `len` but stays inside the (padded) allocation
		for (uint32_t k = threadIdx.x; k < n16; k += PT_THREADS)
			reinterpret_cast<uint4*>(s_text)[k] = __ldg(reinterpret_cast<const uint4*>(text + b0) + k);
	}
	__syncthreads();
	// newlines of this thread's 64 bytes that start a line: those before `lim` (a newline ending the text starts none)
	const uint32_t my0 = threadIdx.x * 64, lim = (uint32_t)((b1 == len ? len - 1 : b1) - b0);
	uint64_t bits = 0;
	#pragma unroll
	for (int k = 0; k < 4; ++k) bits |= (uint64_t)nl_bits_u4(reinterpret_cast<const uint4*>(s_text + my0)[k]) << (16 * k);
	bits &= lim <= my0 ? 0ull : lim - my0 >= 64 ? ~0ull : (1ull << (lim - my0)) - 1;
	const bool line0 = t == 0 && threadIdx.x == 0;            // line 0 starts at byte 0
	uint32_t rank, n;
	BS(s_scan).ExclusiveSum((uint32_t)__popcll(bits) + line0, rank, n);
	// the tile's last line ends at the first '\n' from `lim` on (or at the end of the text)
	for (uint32_t o = lim + threadIdx.x; o < (uint32_t)(w_end - b0); o += PT_THREADS)
		if (s_text[o] == '\n' && b0 + o < len) { atomicMin(&s_nl, o); break; }
	if (threadIdx.x < 32) {
		if (t == 0) {
			if (threadIdx.x == 0) tstate.SetInclusive(0, n), s_first = 0;
		} else {
			LinePrefixOp op(tstate, s_pref, ::cuda::std::plus<unsigned long long>(), (int)t);
			const unsigned long long ex = op(n);
			if (threadIdx.x == 0) s_first = ex;
		}
	}
	__syncthreads();
	const uint64_t first = s_first;
	if (threadIdx.x == 0 && b1 == len) counts[PC_LINES] = first + n;
	if (n == 0) return;
	uint64_t last_eol = s_nl != ~0u ? b0 + s_nl : w_end >= len ? len : ~0ull; // ~0: not staged, ends past the overhang
	if (last_eol == ~0ull) { // (the same for the whole CTA) warp 0 looks for the end of that long line in global memory
		if (threadIdx.x < 32) {
			uint64_t e = ~0ull;
			for (uint64_t p = w_end; p < avail; p += 32 * 16) {
				const uint64_t q = p + 16 * lane;
				uint32_t m = 0;
				for (uint32_t k = 0; k < 16 && q + k < avail; ++k) m |= (uint32_t)(text[q + k] == '\n') << k;
				const unsigned hit = __ballot_sync(0xffffffffu, m != 0);
				if (hit) { e = __shfl_sync(0xffffffffu, q + __ffs(m) - 1, __ffs(hit) - 1); break; }
			}
			if (e == ~0ull && avail == len) e = len;
			if (threadIdx.x == 0) {
				s_eol = e;
				if (e == ~0ull) atomicAdd(counts + PC_CUT, 1ull); // it runs past the bytes that have arrived
			}
		}
		__syncthreads();
		last_eol = s_eol;
	}
	unsigned n_parsed = 0, n_pass = 0;
	for (uint32_t r0 = 0; r0 < n; r0 += PT_LIST) {
		{	// list the starts of the lines r0 .. r0 + PT_LIST of the tile (the last one only ends the one before it)
			uint32_t r = rank;
			uint64_t b = bits;
			if (line0) { if (r == r0) s_start[0] = 0; ++r; }
			for (; b && r <= r0 + PT_LIST; ++r, b &= b - 1)
				if (r >= r0) s_start[r - r0] = (uint16_t)(my0 + __ffsll((long long)b));
		}
		__syncthreads();
		const uint32_t cnt = n - r0 < PT_LIST ? n - r0 : PT_LIST;
		for (uint32_t j0 = 0; j0 < cnt; j0 += PT_THREADS) {
			const uint32_t j = j0 + threadIdx.x;
			const uint64_t i = first + r0 + j;
			uint32_t sq = NOSLOT, st = 0;
			if (j < cnt && i < line_cap) {
				const uint64_t s = b0 + s_start[j];
				uint64_t eol = r0 + j + 1 < n ? b0 + s_start[j + 1] - 1 : last_eol;
				if (eol != ~0ull) {
					const char *base = eol <= w_end ? s_text - b0 : text; // base + file offset = address of that byte
					if (eol - s > 1 && base[eol - 1] == '\r') --eol;
					PLine r;
					parse_line(base + s, base + eol, r, &s_vals[threadIdx.x >> 5][0][lane]);
					if (r.nf >= 10) {
						++n_parsed;
						if (!(r.qe - r.qs < (uint32_t)min_span || r.te - r.ts < (uint32_t)min_span || (int)(r.ml_rev & 0x7fffffffu) < min_match)) {
							++n_pass;
							sq = tab_insert(tab, text, base + s, r.qnl, s, 2 * i, counts + PC_OVERFLOW);
							st = tab_insert(tab, text, base + s + r.tdelta, r.tnl, s + r.tdelta, 2 * i + 1, counts + PC_OVERFLOW);
						}
					}
					start[i] = s;
					*reinterpret_cast<uint4*>(out + i) = make_uint4(r.qs, r.qe, r.ts, r.te);
					*(reinterpret_cast<uint4*>(out + i) + 1) = make_uint4(r.ml_rev, (r.bl & 0x7fffffffu) | (r.nf >= 11 ? 0x80000000u : 0u), sq, st);
				}
			}
			if (tab.hits) { // consecutive lines often share their query read: one add per distinct slot of the warp
				const unsigned grp = __match_any_sync(0xffffffffu, sq);
				if (sq != NOSLOT && lane == (uint32_t)__ffs(grp) - 1) atomicAdd(&tab.hits[sq], (uint32_t)__popc(grp));
				if (sq != NOSLOT && bi_dir && st != sq) atomicAdd(&tab.hits[st], 1u);
			}
		}
		__syncthreads(); // the list is rewritten by the next round
	}
	n_parsed = __reduce_add_sync(0xffffffffu, n_parsed), n_pass = __reduce_add_sync(0xffffffffu, n_pass);
	if (lane == 0) {
		if (n_parsed) atomicAdd(counts + PC_PARSED, (unsigned long long)n_parsed);
		if (n_pass) atomicAdd(counts + PC_STORED, (unsigned long long)n_pass);
	}
}

// bl of a 10-field line: the value of the closest earlier line that had an 11th field (paf.c:47, hit.c:73);
// carry_bl = what the lines before this rank's byte range left behind (sharded runs), else 0
__device__ __forceinline__ uint32_t line_bl(const PRec *ln, uint64_t i, uint32_t carry_bl)
{
	if (ln[i].bl_f >> 31) return ln[i].bl_f & 0x7fffffffu;
	for (uint64_t j = i; j-- > 0;)
		if (ln[j].bl_f >> 31) return ln[j].bl_f & 0x7fffffffu;
	return carry_bl & 0x7fffffffu;
}

struct SlotUsed { // a name is in the dictionary iff some stored line carries it (after -R: iff such a line is left)
	const unsigned long long *first;
	__device__ __forceinline__ bool operator()(uint64_t s) const { return first[s] != ~0ull; }
};

// name and sequence length of an occurrence (2*line + role), read back from the text: the name starts the line (query) or
// follows the 5th TAB (target) and its length column comes right after it
__device__ __forceinline__ void occ_name(const char *text, const uint64_t *start, uint64_t occ, uint64_t *noff, uint32_t *nlen, uint32_t *slen)
{
	const char *p = text + start[occ >> 1];
	uint64_t q = 0;
	if (occ & 1) { int tabs = 0; while (tabs < 5) tabs += p[q++] == '\t'; }
	uint64_t e = q;
	while (p[e] != '\t') ++e;
	*noff = start[occ >> 1] + q, *nlen = (uint32_t)(e - q);
	uint64_t f = e + 1;
	while (p[f] != '\t') ++f;
	*slen = field_to_u32(p + e + 1, p + f);
}

// ---- -R: ma_hit_no_cont (hit.c:38-68) as two passes over the parsed lines -----------------------------------------
// A read is dropped when some stored line shows it clearly inside a read at least twice as long; every line that
// names a dropped read is skipped BEFORE ids are given out (hit.c:86), so first appearances are taken again afterwards.
__global__ void k_nocont_mark(const PRec *ln, uint64_t n_lines, const char *text, const uint64_t *start, int max_hang, float int_frac, uint8_t *excl)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const PRec r = ln[i];
		if (r.slot_q == NOSLOT) continue;
		uint64_t no; uint32_t nl, ql, tl;                              // the two length columns are not kept in the record: read them back
		occ_name(text, start, 2 * i, &no, &nl, &ql);
		occ_name(text, start, 2 * i + 1, &no, &nl, &tl);
		const bool rev = r.ml_rev >> 31;
		const int l5 = (int)(rev ? tl - r.te : r.ts), l3 = (int)(rev ? r.ts : tl - r.te);
		if (ql >> 1 > tl) { // query at least twice as long: is the target inside it?
			if (l5 > max_hang >> 2 || l3 > max_hang >> 2 || (float)(r.te - r.ts) < __fmul_rn((float)tl, int_frac)) continue; // internal match
			if ((int)r.qs - l5 > max_hang << 1 && (int)(ql - r.qe) - l3 > max_hang << 1) excl[r.slot_t] = 1;
		} else if (ql < tl >> 1) {
			if (r.qs > (uint32_t)(max_hang >> 2) || ql - r.qe > (uint32_t)(max_hang >> 2) || (float)(r.qe - r.qs) < __fmul_rn((float)ql, int_frac)) continue;
			if (l5 - (int)r.qs > max_hang << 1 && l3 - (int)(ql - r.qe) > max_hang << 1) excl[r.slot_q] = 1;
		}
	}
}

// (t.first reset to ~0 and t.hits to 0 before: both are taken again over the lines that are left)
__global__ void k_nocont_drop(PRec *ln, uint64_t n_lines, const uint8_t *excl, int bi_dir, NameTab t)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t sq = ln[i].slot_q, st = ln[i].slot_t;
		if (sq == NOSLOT) continue;
		if (excl[sq] || excl[st]) { ln[i].slot_q = NOSLOT; continue; }
		if (t.first[sq] > 2 * i) atomicMin(&t.first[sq], (unsigned long long)(2 * i));
		if (t.first[st] > 2 * i + 1) atomicMin(&t.first[st], (unsigned long long)(2 * i + 1));
		atomicAdd(&t.hits[sq], 1u);
		if (bi_dir && st != sq) atomicAdd(&t.hits[st], 1u);
	}
}

__global__ void k_count_u8(const uint8_t *a, uint64_t n, unsigned long long *out)
{
	unsigned c = 0;
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) c += a[i] != 0;
	c = __reduce_add_sync(0xffffffffu, c);
	if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

__global__ void k_dict_pairs(const uint64_t *slots, uint32_t n, NameTab t, unsigned long long *first_out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) first_out[i] = t.first[slots[i]];
}

// read_cnt[id] = hits of the read (slot -> id is a permutation: the per-slot counts of the parse become per-read counts here)
__global__ void k_dict_rank(const unsigned long long *first_sorted, const uint64_t *slot_sorted, uint32_t n, NameTab t,
                            const char *text, const uint64_t *start, uint64_t *noff, uint32_t *nlen, uint32_t *slen, unsigned long long *tot_len,
                            uint32_t *read_cnt)
{
	unsigned long long sum = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		t.id[slot_sorted[i]] = i;
		read_cnt[i] = t.hits[slot_sorted[i]];
		occ_name(text, start, first_sorted[i], &noff[i], &nlen[i], &slen[i]); // the length kept for a read is the one of its first appearance (sdict.c:36)
		sum += slen[i];
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long s = BR(ts).Sum(sum);
	if (threadIdx.x == 0 && s) atomicAdd(tot_len, s);
}

// --------------------------------------------------------------------------------------------- hits
// every stored line's hit, and its mirror, straight into the bucket of its query read, with the ordinal 2 * line (+ 1 for the
// mirror) in the query-id half of qns: the order of the ordinals is the file order of the hits, as dh_sort_buckets needs
__global__ void k_hit_emit(const PRec *ln, uint64_t n_lines, int bi_dir, NameTab t, const uint32_t *__restrict__ first, uint32_t *cur, DHit *out)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const PRec r = ln[i];
		if (r.slot_q == NOSLOT) continue;
		const uint32_t qid = t.id[r.slot_q], tid = t.id[r.slot_t], bl = line_bl(ln, i, 0), ord = (uint32_t)(2 * i);
		uint4 *o = reinterpret_cast<uint4*>(out + first[qid] + atomicAdd(&cur[qid], 1u));
		o[0] = make_uint4(r.qs, ord, r.qe, tid);
		o[1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
		if (bi_dir && qid != tid) { // the same overlap seen from the target (hit.c:92-98)
			o = reinterpret_cast<uint4*>(out + first[tid] + atomicAdd(&cur[tid], 1u));
			o[0] = make_uint4(r.ts, ord + 1, r.te, qid);
			o[1] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
		}
	}
}

// start[i] = byte offset of line i (a line starts at byte 0 and after every '\n' that is not the last byte); len > 0
uint64_t *dev_line_starts(MabDev &d, const char *d_text, size_t len, uint64_t *n_lines_out)
{
	const uint64_t n_tile = (len + NL_TILE - 1) / NL_TILE;
	uint64_t *cnt = mab_alloc<uint64_t>(d, n_tile + 1);
	uint64_t *base = mab_alloc<uint64_t>(d, n_tile + 1);
	MAB_LAUNCH(d, k_nl_count, mab_grid(n_tile, 1, MAB_SMS * 32u), NL_THREADS, 0, d_text, len, n_tile, cnt);
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, base, (int64_t)(n_tile + 1), d.stream);
	void *tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, base, (int64_t)(n_tile + 1), d.stream);
	++d.n_lib;
	uint64_t n_nl;
	MAB_CUDA(cudaMemcpyAsync(&n_nl, base + n_tile, 8, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	const uint64_t n_lines = n_nl + 1; // newlines that are followed by at least one byte, plus the first line
	uint64_t *start = mab_alloc<uint64_t>(d, n_lines + 1);
	MAB_CUDA(cudaMemsetAsync(start, 0, 8, d.stream));
	MAB_LAUNCH(d, k_nl_write, mab_grid(n_tile, 1, MAB_SMS * 32u), NL_THREADS, 0, d_text, len, n_tile, base, start + 1);
	d.free(cnt); d.free(base);
	*n_lines_out = n_lines;
	return start;
}

void names_free(MabDev &d, DNames &n)
{
	d.free(n.off); d.free(n.nlen); d.free(n.slen);
	n = DNames();
}

static inline uint32_t bits_for(uint64_t x) { uint32_t b = 0; while (x) ++b, x >>= 1; return b ? b : 1; }

static NameTab tab_alloc(MabDev &d, uint64_t cap, bool with_hits)
{
	NameTab tab;
	tab.key = (unsigned long long*)mab_alloc<uint64_t>(d, cap);
	tab.first = (unsigned long long*)mab_alloc<uint64_t>(d, cap);
	tab.id = mab_alloc<uint32_t>(d, cap);
	tab.mask = cap - 1;
	MAB_CUDA(cudaMemsetAsync(tab.key, 0, cap * 8, d.stream));
	MAB_CUDA(cudaMemsetAsync(tab.first, 0xff, cap * 8, d.stream));
	if (with_hits) {
		tab.hits = mab_alloc<uint32_t>(d, cap);
		MAB_CUDA(cudaMemsetAsync(tab.hits, 0, cap * 4, d.stream));
	}
	return tab;
}

static void tab_free(MabDev &d, NameTab &t)
{
	d.free(t.key); d.free(t.first); d.free(t.id);
	if (t.hits) d.free(t.hits);
	t = NameTab{nullptr, nullptr, nullptr, 0};
}

// What the parse leaves: start[line], the record of every line and the dictionary of the stored lines' names.
struct Parsed {
	uint64_t *start = nullptr;
	PRec *ln = nullptr;
	NameTab tab{nullptr, nullptr, nullptr, 0};
	uint64_t cap = 0, n_lines = 0, n_parsed = 0;
	uint32_t regrow = 0;         // dictionary overflows that made the parse run again with a larger table
};

// Room for the lines before they are counted (a PAF line of 12 columns has at least 24 bytes) and the dictionary size
// for it: ~50 lines name a read twice each, so the load stays <= 1/6 at that ratio; an overflow quadruples it.
static inline uint64_t line_estimate(size_t len) { return len / 24 + 1024; }
static inline uint64_t tab_cap_for(uint64_t line_cap) { uint64_t cap = 1ull << 20; while (cap < line_cap / 8) cap <<= 1; return cap; }

// look-back state of k_parse_tiles over n_tile tiles; tiles_reset marks every tile "not done"
static LineTileState tiles_alloc(MabDev &d, uint64_t n_tile, void **mem)
{
	if (n_tile >= (1ull << 31) - 64) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 tiles of PAF on one GPU\n"); exit(73); }
	size_t bytes = 0;
	MAB_CUDA(LineTileState::AllocationSize((int)n_tile, bytes));
	*mem = d.alloc(bytes);
	LineTileState ts;
	MAB_CUDA(ts.Init((int)n_tile, *mem, bytes));
	return ts;
}

static void tiles_reset(MabDev &d, LineTileState ts, uint64_t n_tile)
{
	MAB_LAUNCH(d, k_tiles_init, mab_grid(n_tile, 256, 1u << 30), 256, 0, ts, (int)n_tile);
}

// The whole text is resident: one launch over all tiles, with no host synchronisation before it.  start and ln are sized from
// the estimate; a text with more lines, or with more names than the dictionary holds, is parsed again with room for all of them.
static void parse_resident(MabDev &d, const char *d_text, size_t len, int min_span, int min_match, int bi_dir, bool count_hits, Parsed &p)
{
	const uint64_t n_tile = (len + PT_TILE - 1) / PT_TILE;
	uint64_t line_cap = line_estimate(len), cap = tab_cap_for(line_cap);
	unsigned *ctr = mab_alloc<unsigned>(d, 1);
	void *ts_mem = nullptr;
	const LineTileState ts = tiles_alloc(d, n_tile, &ts_mem);
	for (;;) {
		p.start = mab_alloc<uint64_t>(d, line_cap);
		p.ln = mab_alloc<PRec>(d, line_cap);
		p.tab = tab_alloc(d, cap, count_hits);
		d.zero_scal(SC_COUNT, PC_N);
		if (n_tile) {
			tiles_reset(d, ts, n_tile);
			MAB_CUDA(cudaMemsetAsync(ctr, 0, 4, d.stream));
			MAB_LAUNCH(d, k_parse_tiles, (unsigned)n_tile, PT_THREADS, 0, d_text, len, len, 0, ctr, ts, min_span, min_match, bi_dir, p.tab, p.ln, p.start,
			           line_cap, d.d_scal + SC_COUNT);
		}
		p.n_parsed = d.get_scal(SC_COUNT + PC_PARSED);
		p.n_lines = d.h_scal[SC_COUNT + PC_LINES];
		const bool more_lines = p.n_lines > line_cap, overflow = d.h_scal[SC_COUNT + PC_OVERFLOW] != 0;
		if (!more_lines && !overflow) break;
		d.free(p.start); d.free(p.ln); tab_free(d, p.tab);
		if (more_lines) line_cap = p.n_lines;
		if (overflow) cap <<= 2, ++p.regrow;
		if (cap > (1ull << 33)) { fprintf(stderr, "[E::miniasm_b200] read-name table overflow\n"); exit(77); }
	}
	d.free(ctr); d.free(ts_mem);
	p.cap = cap;
}

static void ingest_finish(MabDev &d, const char *d_text, size_t len, uint64_t *start, PRec *ln, uint64_t n_lines, NameTab tab, uint64_t cap, int bi_dir,
                          const NoContParams *nocont, DHits &h, DNames &names, IngestStats &st);

void ingest_paf(MabDev &d, const char *d_text, size_t len, int min_span, int min_match, int bi_dir, DHits &h, DNames &names, IngestStats &st,
                const NoContParams *nocont)
{
	memset(&st, 0, sizeof(st));
	names = DNames();
	h.n = 0, h.n_seq = 0;
	if (len == 0) { dh_reserve(d, h, 1); return; }
	if (len >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of PAF on one GPU\n"); exit(73); }

	d.trace("ingest:begin");
	// (1)+(2) line starts, parse, store filter, dictionary insert and hit counts per name in one pass
	Parsed p;
	parse_resident(d, d_text, len, min_span, min_match, bi_dir, true, p);
	st.n_parsed = p.n_parsed, st.n_lines = p.n_lines, st.name_regrow = p.regrow;
	d.trace("ingest:parse");
	ingest_finish(d, d_text, len, p.start, p.ln, p.n_lines, p.tab, p.cap, bi_dir, nocont, h, names, st);
}

// Front end of an ingest with the text still on the host: it crosses PCIe in 64 MB chunks on a copy stream while the tiles that
// have arrived are parsed (line starts, store filter, dictionary) on the context's stream, one launch of k_parse_tiles per chunk.
// The look-back state lives across the launches; the last tile that has arrived waits for the next chunk, so every parsed tile
// has its overhang.  host_text may be pageable or pinned (pinned overlaps fully); d_text has room for len + 64.  Capacities are
// estimates: false = the text broke them (more lines than estimated, more names than slots, or a line that runs past a chunk),
// nothing is kept and the caller parses the now-resident text the plain way.  No collectives inside (the sharded ingest calls it
// rank by rank).
static bool stream_parse(MabDev &d, char *d_text, const char *host_text, size_t len, int min_span, int min_match, int bi_dir, bool count_hits, Parsed &p)
{
	const uint64_t CH_TILES = (64ull << 20) / PT_TILE, n_tile = (len + PT_TILE - 1) / PT_TILE;       // 64 MB chunks, whole tiles
	const uint64_t n_chunk = (n_tile + CH_TILES - 1) / CH_TILES;
	const uint64_t line_cap = line_estimate(len), cap = tab_cap_for(line_cap);
	p.start = mab_alloc<uint64_t>(d, line_cap);
	p.ln = mab_alloc<PRec>(d, line_cap);
	p.tab = tab_alloc(d, cap, count_hits);
	unsigned *ctr = mab_alloc<unsigned>(d, n_chunk);                // tile counter of each launch
	MAB_CUDA(cudaMemsetAsync(ctr, 0, n_chunk * 4, d.stream));
	void *ts_mem = nullptr;
	const LineTileState ts = tiles_alloc(d, n_tile, &ts_mem);
	tiles_reset(d, ts, n_tile);
	d.zero_scal(SC_COUNT, PC_N);
	if (!d.copy_stream) MAB_CUDA(cudaStreamCreateWithFlags(&d.copy_stream, cudaStreamNonBlocking));
	std::vector<cudaEvent_t> ev(n_chunk);
	cudaEvent_t ready;
	MAB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
	MAB_CUDA(cudaEventRecord(ready, d.stream));                 // the copies may not overtake whatever still uses d_text on the main stream
	MAB_CUDA(cudaStreamWaitEvent(d.copy_stream, ready, 0));
	uint64_t t_done = 0;                                         // tiles [0, t_done) are parsed
	for (uint64_t k = 0; k < n_chunk; ++k) { // copy k is issued before the kernel of chunk k: a pageable source blocks the host per chunk, not for the whole text
		const uint64_t t0 = k * CH_TILES, t1 = (k + 1) * CH_TILES < n_tile ? (k + 1) * CH_TILES : n_tile;
		const uint64_t b0 = t0 * PT_TILE, b1 = t1 * PT_TILE < len ? t1 * PT_TILE : len;
		MAB_CUDA(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
		MAB_CUDA(cudaMemcpyAsync(d_text + b0, host_text + b0, b1 - b0, cudaMemcpyHostToDevice, d.copy_stream));
		MAB_CUDA(cudaEventRecord(ev[k], d.copy_stream));
		MAB_CUDA(cudaStreamWaitEvent(d.stream, ev[k], 0));
		const uint64_t t_hi = k + 1 == n_chunk ? n_tile : t1 - 1;
		MAB_LAUNCH(d, k_parse_tiles, (unsigned)(t_hi - t_done), PT_THREADS, 0, d_text, len, b1, t_done, ctr + k, ts, min_span, min_match, bi_dir, p.tab, p.ln,
		           p.start, line_cap, d.d_scal + SC_COUNT);
		t_done = t_hi;
	}
	p.n_parsed = d.get_scal(SC_COUNT + PC_PARSED);               // (synchronises)
	for (uint64_t k = 0; k < n_chunk; ++k) MAB_CUDA(cudaEventDestroy(ev[k]));
	MAB_CUDA(cudaEventDestroy(ready));
	d.free(ctr); d.free(ts_mem);
	p.n_lines = d.h_scal[SC_COUNT + PC_LINES];
	if (p.n_lines > line_cap || d.h_scal[SC_COUNT + PC_OVERFLOW] != 0 || d.h_scal[SC_COUNT + PC_CUT] != 0) {
		d.free(p.start); d.free(p.ln); tab_free(d, p.tab);
		p = Parsed();
		return false;
	}
	p.cap = cap;
	return true;
}

// mab_load_paf_text + mab_ingest in one call (same result): when the last byte of the text lands only the id ranking, the hit
// emission and the sort are left.
void ingest_paf_stream(MabDev &d, char *d_text, const char *host_text, size_t len, int min_span, int min_match, int bi_dir,
                       DHits &h, DNames &names, IngestStats &st)
{
	memset(&st, 0, sizeof(st));
	names = DNames();
	h.n = 0, h.n_seq = 0;
	if (len == 0) { dh_reserve(d, h, 1); return; }
	if (len >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of PAF on one GPU\n"); exit(73); }
	Parsed p;
	if (!stream_parse(d, d_text, host_text, len, min_span, min_match, bi_dir, true, p)) {
		ingest_paf(d, d_text, len, min_span, min_match, bi_dir, h, names, st, nullptr); // the text is resident now: the plain path parses it again
		++st.name_regrow;
		return;
	}
	st.n_parsed = p.n_parsed, st.n_lines = p.n_lines;
	d.trace("ingest:stream (copy + parse + dictionary + hit counts)");
	ingest_finish(d, d_text, len, p.start, p.ln, p.n_lines, p.tab, p.cap, bi_dir, nullptr, h, names, st);
}

static void ingest_finish(MabDev &d, const char *d_text, size_t len, uint64_t *start, PRec *ln, uint64_t n_lines, NameTab tab, uint64_t cap, int bi_dir,
                          const NoContParams *nocont, DHits &h, DNames &names, IngestStats &st)
{
	// the hit ordinals 2 * line + 1 and the bucket offsets are 32-bit
	if (2 * n_lines >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 PAF lines on one GPU\n"); exit(73); }
	d.trace("ingest:dictionary");
	if (nocont) { // -R: mark the contained reads, drop every line that names one, take the first appearances again
		uint8_t *excl = mab_alloc<uint8_t>(d, cap);
		MAB_CUDA(cudaMemsetAsync(excl, 0, cap, d.stream));
		MAB_LAUNCH(d, k_nocont_mark, mab_grid(n_lines, 256), 256, 0, ln, n_lines, d_text, start, nocont->max_hang, nocont->int_frac, excl);
		d.zero_scal(SC_AUX, 1);
		MAB_LAUNCH(d, k_count_u8, mab_grid(cap, 256), 256, 0, excl, cap, d.d_scal + SC_AUX);
		MAB_CUDA(cudaMemsetAsync(tab.first, 0xff, cap * 8, d.stream));
		MAB_CUDA(cudaMemsetAsync(tab.hits, 0, cap * 4, d.stream));
		MAB_LAUNCH(d, k_nocont_drop, mab_grid(n_lines, 256), 256, 0, ln, n_lines, excl, bi_dir, tab);
		st.n_dropped = d.get_scal(SC_AUX);
		d.free(excl);
		d.trace("ingest:-R prefilter");
	}
	// (4) ids = rank of the first occurrence; the hit counts of the slots become those of the reads (the bucket sizes of the sort)
	uint64_t *slots = mab_alloc<uint64_t>(d, cap);
	uint32_t n_seq;
	{
		cub::CountingInputIterator<uint64_t> pos(0);
		SlotUsed used{tab.first};
		size_t tb = 0;
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		cub::DeviceSelect::If(nullptr, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceSelect::If(tmp, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		++d.n_lib;
		uint64_t n = d.get_scal(SC_NSEL);
		if (n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 reads\n"); exit(73); }
		n_seq = (uint32_t)n;
	}
	names.n_seq = n_seq;
	names.off = mab_alloc<uint64_t>(d, n_seq); names.nlen = mab_alloc<uint32_t>(d, n_seq); names.slen = mab_alloc<uint32_t>(d, n_seq);
	uint32_t *read_cnt = mab_alloc<uint32_t>(d, (size_t)n_seq + 1), *first = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
	MAB_CUDA(cudaMemsetAsync(read_cnt + n_seq, 0, 4, d.stream));
	if (n_seq) {
		unsigned long long *fa = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq), *fb = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq);
		uint64_t *sb = mab_alloc<uint64_t>(d, n_seq);
		MAB_LAUNCH(d, k_dict_pairs, mab_grid(n_seq, 256), 256, 0, slots, n_seq, tab, fa);
		cub::DoubleBuffer<unsigned long long> dk(fa, fb);
		cub::DoubleBuffer<uint64_t> dv(slots, sb);
		size_t tb = 0;
		int end_bit = (int)bits_for(2 * n_lines + 1);
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)n_seq, 0, end_bit, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)n_seq, 0, end_bit, d.stream);
		++d.n_lib;
		d.zero_scal(SC_AUX, 1);
		MAB_LAUNCH(d, k_dict_rank, mab_grid(n_seq, 256), 256, 0, dk.Current(), dv.Current(), n_seq, tab, d_text, start, names.off, names.nlen, names.slen, d.d_scal + SC_AUX,
		           read_cnt);
		st.tot_len = d.get_scal(SC_AUX);
		d.free(fa); d.free(fb); d.free(sb);
	}
	d.free(slots);

	d.trace("ingest:rank_ids");
	// (5) every hit emitted straight into its read's bucket of h.a2
	dh_bucket_first(d, read_cnt, n_seq, first);
	MAB_CUDA(cudaMemsetAsync(read_cnt, 0, (size_t)n_seq * 4, d.stream)); // the counts become the buckets' fill cursors
	uint32_t n_hits;
	MAB_CUDA(cudaMemcpyAsync(&n_hits, first + n_seq, 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	dh_reserve(d, h, n_hits ? n_hits : 1);
	h.n = n_hits, h.n_seq = n_seq;
	if (n_hits) MAB_LAUNCH(d, k_hit_emit, mab_grid(n_lines, 256), 256, 0, ln, n_lines, bi_dir, tab, first, read_cnt, h.a2);
	st.n_hits = n_hits, st.n_seq = n_seq;
	d.free(ln); d.free(start);
	tab_free(d, tab);

	d.trace("ingest:emit_hits");
	// (6) ma_hit_sort: order every bucket (h.a2 -> h.a)
	dh_sort_buckets(d, h, first);
	d.free(read_cnt); d.free(first);
	d.trace("ingest:sort_hits");
}

// Host-side probe of the device parser (same source, compiled for the host): lets the CPU test tier compare the
// lockstep parser with the host reader on corner-case lines without a GPU.  out = nf ql qs qe rev tl ts te ml bl qnl tnl tdelta.
extern "C" int mab_test_parse_line(const char *line, size_t len, uint32_t *out)
{
	static uint32_t vals[11 * 32];
	PLine r;
	size_t eol = len;
	if (eol > 1 && line[eol - 1] == '\r') --eol;
	parse_line(line, line + eol, r, vals);
	out[0] = r.nf, out[1] = r.ql, out[2] = r.qs, out[3] = r.qe, out[4] = r.ml_rev >> 31, out[5] = r.tl, out[6] = r.ts, out[7] = r.te;
	out[8] = r.ml_rev & 0x7fffffffu, out[9] = r.bl, out[10] = r.qnl, out[11] = r.tnl, out[12] = r.tdelta;
	return 0;
}

// =============================================================================================================
// Sharded ingest (SURVEY.md 8e.1-2): every rank parses its own byte range of the PAF (ranges follow rank order, so
// "line i of rank r" has the global line number base[r] + i), the distinct names of all ranks are all-gathered and
// ranked by global first occurrence -- which reproduces the single-GPU ids exactly -- and every hit travels to the
// rank that owns its query read (id mod world) in one all-to-all; per-source order is file order, so the stable sort
// that follows sees the hits of a read in the same order as a single GPU would.
// =============================================================================================================
__global__ void k_last_bl(const PRec *ln, uint64_t n_lines, unsigned long long *out) // out[0] = 1 + index of the last line with an 11th field
{
	unsigned long long mx = 0; // per-thread maximum over its grid-stride share, one atomic per warp at the end
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x)
		if (ln[i].bl_f >> 31) mx = i + 1;
	#pragma unroll
	for (int o = 16; o; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, mx, o); mx = t > mx ? t : mx; }
	if ((threadIdx.x & 31) == 0 && mx) atomicMax(out, mx);
}

struct GEntry { unsigned long long hash, first; uint32_t slen, nlen; }; // a distinct name of one rank, 24 bytes

__global__ void k_local_entries(const uint64_t *slots, uint32_t n, NameTab t, const char *text, const uint64_t *start, uint64_t line_base, uint64_t seed,
                                GEntry *ent, uint32_t *name_sz, uint64_t *name_off)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint64_t occ = t.first[slots[i]];
		GEntry e;
		uint64_t no;
		occ_name(text, start, occ, &no, &e.nlen, &e.slen);
		e.hash = name_hash(text + no, 0, e.nlen, seed), e.first = 2 * line_base + occ;
		ent[i] = e;
		name_sz[i] = e.nlen, name_off[i] = no;
	}
}

__global__ void k_local_names(uint32_t n, const uint64_t *name_off, const uint32_t *name_sz, const char *text, const uint64_t *pos, char *out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const char *src = text + name_off[i];
		char *dst = out + pos[i];
		for (uint32_t k = 0; k < name_sz[i]; ++k) dst[k] = src[k];
	}
}

struct U32ToU64i { __host__ __device__ __forceinline__ uint64_t operator()(uint32_t x) const { return x; } };

struct GTab { unsigned long long *key, *first; uint32_t *win, *id; uint64_t mask; }; // global table: winner entry and read id per slot

__global__ void k_gtab_insert(const GEntry *ent, uint64_t n, GTab t, uint32_t *slot_of, unsigned long long *overflow)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long h = ent[i].hash;
		uint64_t s = h & t.mask;
		uint32_t found = 0xffffffffu;
		for (int probe = 0; probe < 1 << 14; ++probe, s = (s + 1) & t.mask) {
			unsigned long long k = t.key[s];
			if (k == 0) { k = atomicCAS(&t.key[s], 0ull, h); if (k == 0) k = h; }
			if (k == h) { atomicMin(&t.first[s], ent[i].first); found = (uint32_t)s; break; }
		}
		if (found == 0xffffffffu) atomicAdd(overflow, 1ull);
		slot_of[i] = found;
	}
}

// an entry that found no slot (slot_of = 0xffffffff, counted by k_gtab_insert) is skipped: the table is built again with another seed
__global__ void k_gtab_winner(const GEntry *ent, uint64_t n, GTab t, const uint32_t *slot_of)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t s = slot_of[i];
		if (s != 0xffffffffu && t.first[s] == ent[i].first) t.win[s] = (uint32_t)i; // first occurrences are unique: exactly one winner
	}
}

__global__ void k_gtab_verify(const GEntry *ent, uint64_t n, GTab t, const uint32_t *slot_of, const uint64_t *name_pos, const char *names, unsigned long long *n_bad)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		if (slot_of[i] == 0xffffffffu) continue;                         // (no slot: already an overflow, the table is redone)
		const uint32_t w = t.win[slot_of[i]];
		if (w == i) continue;
		bool ok = ent[w].nlen == ent[i].nlen;
		const char *a = names + name_pos[i], *b = names + name_pos[w];
		for (uint32_t k = 0; ok && k < ent[i].nlen; ++k) ok = a[k] == b[k];
		if (!ok) atomicAdd(n_bad, 1ull);
	}
}

struct GSlotUsed { const unsigned long long *key; __device__ __forceinline__ bool operator()(uint64_t s) const { return key[s] != 0; } };

__global__ void k_gtab_first(const uint64_t *slots, uint32_t n, GTab t, unsigned long long *first_out)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) first_out[i] = t.first[slots[i]];
}

__global__ void k_gtab_rank(const uint64_t *slot_sorted, uint32_t n, GTab t, const GEntry *ent, const uint64_t *name_pos,
                            uint64_t *noff, uint32_t *nlen, uint32_t *slen, unsigned long long *tot_len)
{
	unsigned long long sum = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint64_t s = slot_sorted[i];
		const uint32_t w = t.win[s];
		t.id[s] = i;
		noff[i] = name_pos[w], nlen[i] = ent[w].nlen, slen[i] = ent[w].slen;
		sum += ent[w].slen;
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long sm = BR(ts).Sum(sum);
	if (threadIdx.x == 0 && sm) atomicAdd(tot_len, sm);
}

// local dictionary slot -> global read id (entry i of this rank sits at slots[i] locally and at slot_of[i] in the global table)
__global__ void k_local_gid(const uint64_t *slots, uint32_t n, const uint32_t *slot_of, GTab gt, NameTab lt)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) lt.id[slots[i]] = gt.id[slot_of[i]];
}

// number of hits every line yields
__global__ void k_line_gids(const PRec *ln, uint64_t n_lines, NameTab lt, int bi_dir, uint32_t *cnt)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint2 sl = *reinterpret_cast<const uint2*>(&ln[i].slot_q);
		cnt[i] = sl.x != NOSLOT ? (bi_dir && lt.id[sl.x] != lt.id[sl.y] ? 2 : 1) : 0;
	}
}

__global__ void k_hit_emit_gid(const PRec *ln, uint64_t n_lines, const uint32_t *cnt, const uint64_t *off, NameTab lt, uint32_t carry_bl, uint32_t world,
                               DHit *out, uint32_t *dest)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t c = cnt[i];
		if (c == 0) continue;
		const PRec r = ln[i];
		const uint32_t qid = lt.id[r.slot_q], tid = lt.id[r.slot_t], bl = line_bl(ln, i, carry_bl);
		uint4 *o = reinterpret_cast<uint4*>(out + off[i]);
		o[0] = make_uint4(r.qs, qid, r.qe, tid);
		o[1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
		dest[off[i]] = qid % world;
		if (c == 2) {
			o[2] = make_uint4(r.ts, tid, r.te, qid);
			o[3] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
			dest[off[i] + 1] = tid % world;
		}
	}
}

// ---- emit + exchange fused: every hit is written straight into the receive buffer of the rank that owns its query read ------
// (over NVLink for remote owners).  Order inside a (source rank, destination) bucket must be file order, so positions come from a
// two-level count: per 256-line block and destination (k_push_count -> exclusive scan, destination-major), and inside a block the
// rank of a hit among the block's hits to the same destination (ballots per destination; a line's own hit precedes its mirror).
constexpr int PUSH_LINES = 256;

struct PushLine { bool has0, has1; uint32_t d0, d1, qid, tid; };

__device__ __forceinline__ PushLine push_line(const PRec *ln, uint64_t i, uint64_t n_lines, const NameTab &lt, int bi_dir, uint32_t world)
{
	PushLine p{false, false, 0, 0, 0, 0};
	if (i < n_lines) {
		const uint2 sl = *reinterpret_cast<const uint2*>(&ln[i].slot_q);
		if (sl.x != NOSLOT) {
			p.qid = lt.id[sl.x], p.tid = lt.id[sl.y];
			p.has0 = true, p.has1 = bi_dir && p.qid != p.tid;
			p.d0 = p.qid % world, p.d1 = p.tid % world;
		}
	}
	return p;
}

__global__ void __launch_bounds__(PUSH_LINES) k_push_count(const PRec *ln, uint64_t n_lines, NameTab lt, int bi_dir, uint32_t world, uint64_t n_blk, uint32_t *blk_cnt)
{
	__shared__ uint32_t s_cnt[32];
	for (uint64_t b = blockIdx.x; b < n_blk; b += gridDim.x) {
		if (threadIdx.x < 32) s_cnt[threadIdx.x] = 0;
		__syncthreads();
		const PushLine p = push_line(ln, b * PUSH_LINES + threadIdx.x, n_lines, lt, bi_dir, world);
		for (uint32_t g = 0; g < world; ++g) {
			const unsigned b0 = __ballot_sync(0xffffffffu, p.has0 && p.d0 == g), b1 = __ballot_sync(0xffffffffu, p.has1 && p.d1 == g);
			if ((threadIdx.x & 31) == 0 && (b0 | b1)) atomicAdd(&s_cnt[g], (uint32_t)(__popc(b0) + __popc(b1)));
		}
		__syncthreads();
		if (threadIdx.x < world) blk_cnt[(uint64_t)threadIdx.x * n_blk + b] = s_cnt[threadIdx.x];
		__syncthreads();
	}
}

// dst[g] = receive buffer of rank g (peer address); pos_base[g] = (offset of this rank's bucket in it) - blk_off[g * n_blk].
// The block's hits are first laid out in shared memory grouped by destination (in file order inside a group), then the whole
// staging area goes out with consecutive threads writing consecutive 16-byte halves: every destination receives one contiguous
// run per block (2 KB at 8 ranks) instead of isolated 32-byte stores -- isolated stores ran the NVLink at ~290 GB/s (11 ms at N=4).
__global__ void __launch_bounds__(PUSH_LINES) k_push_emit(const PRec *ln, uint64_t n_lines, NameTab lt, int bi_dir, uint32_t carry_bl, uint32_t world, uint64_t n_blk,
                                                          const uint64_t *__restrict__ blk_off, const long long *__restrict__ pos_base, DHit *const *__restrict__ dst)
{
	__shared__ uint32_t s_wc[PUSH_LINES / 32][32];
	__shared__ uint32_t s_seg[33];                                  // exclusive prefix of the block's per-destination totals
	__shared__ __align__(16) uint4 s_hit[2 * 2 * PUSH_LINES];        // up to two hits per line, two 16-byte halves per hit
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt_mask = (1u << lane) - 1u;
	for (uint64_t b = blockIdx.x; b < n_blk; b += gridDim.x) {
		const uint64_t i = b * PUSH_LINES + threadIdx.x;
		const PushLine p = push_line(ln, i, n_lines, lt, bi_dir, world);
		uint32_t r0 = 0, r1 = 0;                       // rank of my two hits inside the warp, among the hits to the same destination
		for (uint32_t g = 0; g < world; ++g) {
			const unsigned b0 = __ballot_sync(0xffffffffu, p.has0 && p.d0 == g), b1 = __ballot_sync(0xffffffffu, p.has1 && p.d1 == g);
			const uint32_t before = (uint32_t)(__popc(b0 & lt_mask) + __popc(b1 & lt_mask));
			if (p.has0 && p.d0 == g) r0 = before;
			if (p.has1 && p.d1 == g) r1 = before + (p.d0 == g ? 1u : 0u);
			if (lane == 0) s_wc[warp][g] = (uint32_t)(__popc(b0) + __popc(b1));
		}
		__syncthreads();
		if (warp == 0) { // per-destination totals of the block and their exclusive prefix
			uint32_t t = 0;
			if (lane < world) for (uint32_t w = 0; w < PUSH_LINES / 32; ++w) t += s_wc[w][lane];
			uint32_t inc = t;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if ((int)lane >= o) inc += y; }
			s_seg[lane + 1] = inc;
			if (lane == 0) s_seg[0] = 0;
		}
		__syncthreads();
		if (p.has0) {
			const PRec r = ln[i];
			const uint32_t bl = line_bl(ln, i, carry_bl);
			uint32_t w0 = 0, w1 = 0;
			for (uint32_t w = 0; w < warp; ++w) w0 += s_wc[w][p.d0], w1 += s_wc[w][p.d1];
			const uint32_t k0 = s_seg[p.d0] + w0 + r0;
			s_hit[2 * k0] = make_uint4(r.qs, p.qid, r.qe, p.tid);
			s_hit[2 * k0 + 1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
			if (p.has1) { // the same overlap seen from the target (hit.c:92-98)
				const uint32_t k1 = s_seg[p.d1] + w1 + r1;
				s_hit[2 * k1] = make_uint4(r.ts, p.tid, r.te, p.qid);
				s_hit[2 * k1 + 1] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
			}
		}
		__syncthreads();
		const uint32_t total = s_seg[world];
		for (uint32_t j = threadIdx.x; j < 2 * total; j += PUSH_LINES) {
			const uint32_t k = j >> 1;
			uint32_t g = 0;
			while (s_seg[g + 1] <= k) ++g;                // destination whose group holds staging slot k
			uint4 *o = reinterpret_cast<uint4*>(dst[g] + (pos_base[g] + (long long)blk_off[(uint64_t)g * n_blk + b] + (k - s_seg[g])));
			o[j & 1] = s_hit[j];
		}
		__syncthreads();
	}
	__threadfence_system();                            // the stores to peer memory are out before the grid reports completion
}

__global__ void k_gather_hits(const DHit *a, const uint32_t *pos, uint64_t n, DHit *out)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint4 *q = reinterpret_cast<const uint4*>(a + pos[i]);
		uint4 x = __ldg(q), y = __ldg(q + 1);
		uint4 *o = reinterpret_cast<uint4*>(out + i);
		o[0] = x, o[1] = y;
	}
}

__global__ void k_add_u64(uint64_t *a, uint64_t n, uint64_t add) { for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) a[i] += add; }

__global__ void k_iota32(uint32_t *a, uint64_t n) { for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) a[i] = (uint32_t)i; }

void ingest_paf_sharded(MabDev &d, ShardComm &sc, char *d_text, size_t len, int min_span, int min_match, int bi_dir,
                        DHits &h, DNames &names, char **name_text_out, IngestStats &st, const char *host_text)
{	// host_text != nullptr: this rank's bytes are still on the host; they are copied in chunks while the arrived chunks are parsed
	memset(&st, 0, sizeof(st));
	names = DNames();
	h.n = 0, h.n_seq = 0;
	const int G = sc.world;
	// (1)+(2) local line starts, parse + store filter + local dictionary (exact: occurrences are compared with a witness in the text)
	if (len >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of PAF on one GPU\n"); exit(73); }
	Parsed p;
	bool have = false;                                      // this rank holds a finished local parse
	if (host_text && len) {
		have = stream_parse(d, d_text, host_text, len, min_span, min_match, bi_dir, false, p);
		d.trace("shard-ingest:stream (copy + parse + dictionary)");
	}
	if (!have) parse_resident(d, d_text, len, min_span, min_match, bi_dir, false, p); // (local: the dictionary grows on this rank alone)
	st.name_regrow = p.regrow + (host_text && len && !have ? 1 : 0);
	uint64_t *start = p.start, n_lines = p.n_lines, cap = p.cap, n_parsed = p.n_parsed;
	PRec *ln = p.ln;
	NameTab tab = p.tab;
	st.n_parsed = n_parsed;
	std::vector<uint64_t> all_lines = sc_allgather_u64(d, sc, n_lines);
	uint64_t line_base = 0, n_lines_all = 0;
	for (int r = 0; r < G; ++r) { if (r < sc.rank) line_base += all_lines[r]; n_lines_all += all_lines[r]; }
	st.n_lines = n_lines_all;
	d.trace("shard-ingest:parse+filter+local dictionary");
	// bl carried over from earlier ranks for 10-field lines at the head of this range (applied when the hits are emitted)
	uint32_t carry = 0;
	{
		d.zero_scal(SC_TMP0, 1);
		if (n_lines) MAB_LAUNCH(d, k_last_bl, mab_grid(n_lines, 256), 256, 0, ln, n_lines, d.d_scal + SC_TMP0);
		uint64_t last11 = d.get_scal(SC_TMP0);
		uint32_t my_bl = 0;
		if (last11) { MAB_CUDA(cudaMemcpyAsync(&my_bl, &ln[last11 - 1].bl_f, 4, cudaMemcpyDeviceToHost, d.stream)); d.sync(); my_bl &= 0x7fffffffu; }
		std::vector<uint64_t> bls = sc_allgather_u64(d, sc, last11 ? ((uint64_t)1 << 32 | my_bl) : 0);
		for (int r = 0; r < sc.rank; ++r) if (bls[r] >> 32) carry = (uint32_t)bls[r];
	}
	// (3) distinct names of this rank -> entries + packed names, all-gathered; (4) global table (replicated).  Two different names
	// with one 64-bit hash would share a global slot: the byte comparison finds that and the entries are hashed again with another seed.
	uint32_t n_ent = 0;
	uint64_t *slots = mab_alloc<uint64_t>(d, cap);
	{
		cub::CountingInputIterator<uint64_t> pos(0);
		SlotUsed used{tab.first};
		size_t tb = 0;
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		cub::DeviceSelect::If(nullptr, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceSelect::If(tmp, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		++d.n_lib;
		n_ent = (uint32_t)d.get_scal(SC_NSEL);
	}
	GTab gt{nullptr, nullptr, nullptr, nullptr, 0};
	GEntry *g_ent = nullptr;
	char *g_names = nullptr;
	uint64_t *g_pos = nullptr;
	uint32_t *slot_of = nullptr;
	uint64_t n_ent_all = 0, name_bytes_all = 0, my_ent_off = 0;
	uint64_t seed = 0;
	for (int attempt = 0;; ++attempt) {
		GEntry *ent = mab_alloc<GEntry>(d, n_ent);
		uint32_t *nsz = mab_alloc<uint32_t>(d, (size_t)n_ent + 1);
		uint64_t *npos = mab_alloc<uint64_t>(d, (size_t)n_ent + 1), *nsrc = mab_alloc<uint64_t>(d, (size_t)n_ent + 1);
		uint64_t my_name_bytes = 0;
		char *my_names = nullptr;
		if (n_ent) {
			MAB_LAUNCH(d, k_local_entries, mab_grid(n_ent, 256), 256, 0, slots, n_ent, tab, d_text, start, line_base, seed, ent, nsz, nsrc);
			size_t tb = 0;
			cub::DeviceScan::ExclusiveSum(nullptr, tb, nsz, npos, (int)n_ent, d.stream);
			void *tmp = d.tmp(tb);
			cub::DeviceScan::ExclusiveSum(tmp, tb, nsz, npos, (int)n_ent, d.stream);
			++d.n_lib;
			uint64_t lp; uint32_t ls;
			MAB_CUDA(cudaMemcpyAsync(&lp, npos + n_ent - 1, 8, cudaMemcpyDeviceToHost, d.stream));
			MAB_CUDA(cudaMemcpyAsync(&ls, nsz + n_ent - 1, 4, cudaMemcpyDeviceToHost, d.stream));
			d.sync();
			my_name_bytes = lp + ls;
			my_names = (char*)d.alloc(my_name_bytes ? my_name_bytes : 1);
			MAB_LAUNCH(d, k_local_names, mab_grid(n_ent, 256), 256, 0, n_ent, nsrc, nsz, d_text, npos, my_names);
		}
		std::vector<uint64_t> ents = sc_allgather_u64(d, sc, n_ent), nbytes = sc_allgather_u64(d, sc, my_name_bytes);
		n_ent_all = name_bytes_all = 0;
		std::vector<uint64_t> ent_bytes(G), pos_bytes(G);
		for (int r = 0; r < G; ++r) {
			if (r == sc.rank) my_ent_off = n_ent_all;
			n_ent_all += ents[r], name_bytes_all += nbytes[r];
			ent_bytes[r] = ents[r] * sizeof(GEntry), pos_bytes[r] = ents[r] * 8;
		}
		g_ent = mab_alloc<GEntry>(d, n_ent_all);
		g_names = (char*)d.alloc(name_bytes_all ? name_bytes_all : 1);
		g_pos = mab_alloc<uint64_t>(d, n_ent_all);
		sc_allgather_v(d, sc, ent, ent_bytes, g_ent);
		sc_allgather_v(d, sc, my_names, nbytes, g_names);
		sc_allgather_v(d, sc, npos, pos_bytes, g_pos); // positions are local to each rank's block: rebased below
		{
			std::vector<uint64_t> eoff(G + 1, 0), noff(G + 1, 0);
			for (int r = 0; r < G; ++r) eoff[r + 1] = eoff[r] + ents[r], noff[r + 1] = noff[r] + nbytes[r];
			for (int r = 0; r < G; ++r) if (ents[r] && noff[r]) {
				MAB_LAUNCH(d, k_add_u64, mab_grid(ents[r], 256), 256, 0, g_pos + eoff[r], ents[r], noff[r]);
			}
		}
		d.free(ent); d.free(nsz); d.free(npos); d.free(nsrc); if (my_names) d.free(my_names);
		d.trace("shard-ingest:name all-gather");
		uint64_t gcap = 1ull << 16; while (gcap < 2 * n_ent_all + 2) gcap <<= 1;
		gt.key = (unsigned long long*)mab_alloc<uint64_t>(d, gcap); gt.first = (unsigned long long*)mab_alloc<uint64_t>(d, gcap);
		gt.win = mab_alloc<uint32_t>(d, gcap); gt.id = mab_alloc<uint32_t>(d, gcap); gt.mask = gcap - 1;
		MAB_CUDA(cudaMemsetAsync(gt.key, 0, gcap * 8, d.stream));
		MAB_CUDA(cudaMemsetAsync(gt.first, 0xff, gcap * 8, d.stream));
		slot_of = mab_alloc<uint32_t>(d, n_ent_all);
		d.zero_scal(SC_BIG, 1); d.zero_scal(SC_AUX2, 1);
		if (n_ent_all) {
			MAB_LAUNCH(d, k_gtab_insert, mab_grid(n_ent_all, 256), 256, 0, g_ent, n_ent_all, gt, slot_of, d.d_scal + SC_BIG);
			MAB_LAUNCH(d, k_gtab_winner, mab_grid(n_ent_all, 256), 256, 0, g_ent, n_ent_all, gt, slot_of);
			MAB_LAUNCH(d, k_gtab_verify, mab_grid(n_ent_all, 256), 256, 0, g_ent, n_ent_all, gt, slot_of, g_pos, g_names, d.d_scal + SC_AUX2);
		}
		const bool gbad = d.get_scal(SC_AUX2) != 0 || d.h_scal[SC_BIG] != 0; // identical on all ranks (replicated computation)
		if (!gbad) break;
		d.free(slot_of);
		d.free(gt.key); d.free(gt.first); d.free(gt.win); d.free(gt.id);
		d.free(g_ent); d.free(g_names); d.free(g_pos);
		seed = seed * 6364136223846793005ULL + 1442695040888963407ULL;
		++st.hash_retries, ++st.name_regrow;
		if (attempt > 16) { fprintf(stderr, "[E::miniasm_b200] read-name hashing keeps colliding\n"); exit(77); }
	}
	d.trace("shard-ingest:global table");
	// (5) global ids = rank of the global first occurrence
	uint32_t n_seq;
	{
		const uint64_t gcap = gt.mask + 1;
		uint64_t *slots = mab_alloc<uint64_t>(d, gcap);
		cub::CountingInputIterator<uint64_t> pos(0);
		GSlotUsed used{gt.key};
		size_t tb = 0;
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		cub::DeviceSelect::If(nullptr, tb, pos, slots, d_n, (int64_t)gcap, used, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceSelect::If(tmp, tb, pos, slots, d_n, (int64_t)gcap, used, d.stream);
		++d.n_lib;
		uint64_t n = d.get_scal(SC_NSEL);
		if (n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 reads\n"); exit(73); }
		n_seq = (uint32_t)n;
		names.n_seq = n_seq;
		names.off = mab_alloc<uint64_t>(d, n_seq); names.nlen = mab_alloc<uint32_t>(d, n_seq); names.slen = mab_alloc<uint32_t>(d, n_seq);
		if (n_seq) {
			unsigned long long *fa = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq), *fb = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq);
			uint64_t *sb = mab_alloc<uint64_t>(d, n_seq);
			MAB_LAUNCH(d, k_gtab_first, mab_grid(n_seq, 256), 256, 0, slots, n_seq, gt, fa);
			cub::DoubleBuffer<unsigned long long> dk(fa, fb);
			cub::DoubleBuffer<uint64_t> dv(slots, sb);
			size_t tb2 = 0;
			int end_bit = (int)bits_for(2 * n_lines_all + 1);
			cub::DeviceRadixSort::SortPairs(nullptr, tb2, dk, dv, (int)n_seq, 0, end_bit, d.stream);
			void *tmp2 = d.tmp(tb2);
			cub::DeviceRadixSort::SortPairs(tmp2, tb2, dk, dv, (int)n_seq, 0, end_bit, d.stream);
			++d.n_lib;
			d.zero_scal(SC_AUX, 1);
			MAB_LAUNCH(d, k_gtab_rank, mab_grid(n_seq, 256), 256, 0, dv.Current(), n_seq, gt, g_ent, g_pos, names.off, names.nlen, names.slen, d.d_scal + SC_AUX);
			st.tot_len = d.get_scal(SC_AUX);
			d.free(fa); d.free(fb); d.free(sb);
		}
		d.free(slots);
	}
	*name_text_out = g_names; // names.off points into this buffer (owned by the caller from now on)
	d.trace("shard-ingest:global ids");
	// (6) local hits with global ids go to the rank that owns their query read
	if (G > 32) { fprintf(stderr, "[E::miniasm_b200] more than 32 ranks\n"); exit(79); }
	if (n_ent) MAB_LAUNCH(d, k_local_gid, mab_grid(n_ent, 256), 256, 0, slots, n_ent, slot_of + my_ent_off, gt, tab);
	uint64_t n_recv = 0;
	std::vector<uint64_t> send_cnt(G, 0), recv_cnt(G, 0), mat((size_t)G * G, 0);
	auto counts_matrix = [&]() { // every rank learns how much it receives from whom
		uint64_t *m = mab_alloc<uint64_t>(d, (size_t)G * G + G);
		MAB_CUDA(cudaMemcpyAsync(m + (size_t)G * G, send_cnt.data(), 8 * (size_t)G, cudaMemcpyHostToDevice, d.stream));
		if (sc.active()) MAB_NCCL(ncclAllGather(m + (size_t)G * G, m, G, ncclUint64, sc.comm, d.stream));
		else MAB_CUDA(cudaMemcpyAsync(m, m + (size_t)G * G, 8 * (size_t)G, cudaMemcpyDeviceToDevice, d.stream));
		MAB_CUDA(cudaMemcpyAsync(mat.data(), m, 8 * (size_t)G * G, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		n_recv = 0;
		for (int r = 0; r < G; ++r) recv_cnt[r] = mat[(size_t)r * G + sc.rank], n_recv += recv_cnt[r];
		d.free(m);
		if (n_recv >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 hits on one GPU\n"); exit(73); }
	};
	// (6a) fused route: count per (256-line block, destination), scan, then ONE kernel emits every hit straight into its owner's
	// receive buffer over NVLink -- no send buffer, no bucket sort, no NCCL all-to-all.  Needs peer access to all receive buffers.
	const uint64_t n_blk = (n_lines + PUSH_LINES - 1) / PUSH_LINES;
	uint32_t *blk_cnt = mab_alloc<uint32_t>(d, (size_t)G * n_blk + 1);
	uint64_t *blk_off = mab_alloc<uint64_t>(d, (size_t)G * n_blk + 1);
	MAB_CUDA(cudaMemsetAsync(blk_cnt, 0, ((size_t)G * n_blk + 1) * 4, d.stream));
	if (n_blk) MAB_LAUNCH(d, k_push_count, mab_grid(n_blk, 1, MAB_SMS * 8u), PUSH_LINES, 0, ln, n_lines, tab, bi_dir, (uint32_t)G, n_blk, blk_cnt);
	{
		cub::TransformInputIterator<uint64_t, U32ToU64i, const uint32_t*> in(blk_cnt, U32ToU64i());
		size_t tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, in, blk_off, (int64_t)((size_t)G * n_blk + 1), d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, in, blk_off, (int64_t)((size_t)G * n_blk + 1), d.stream);
		++d.n_lib;
	}
	std::vector<uint64_t> bstart((size_t)G + 1, 0);
	for (int g = 0; g <= G; ++g) MAB_CUDA(cudaMemcpyAsync(&bstart[g], blk_off + (size_t)g * n_blk, 8, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	for (int g = 0; g < G; ++g) send_cnt[g] = bstart[g + 1] - bstart[g];
	const uint64_t n_loc = bstart[G];
	if (n_loc >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^32 hits parsed by one rank\n"); exit(73); }
	counts_matrix();
	dh_reserve(d, h, n_recv ? n_recv : 1);
	std::vector<void*> peer;
	const char *penv = getenv("MAB_SHARD_PUSH");
	const bool push = sc_peer_ptrs(d, sc, h.a, peer) && !(penv && atoi(penv) == 0); // (collective: also the barrier after which every receive buffer exists)
	d.trace("shard-ingest:count hits per owner");
	if (push) {
		std::vector<long long> pos_base((size_t)G);
		for (int g = 0; g < G; ++g) {
			uint64_t before = 0;                            // hits rank g receives from the ranks before this one
			for (int r = 0; r < sc.rank; ++r) before += mat[(size_t)r * G + g];
			pos_base[g] = (long long)before - (long long)bstart[g];
		}
		long long *d_pos = (long long*)d.alloc(sizeof(long long) * (size_t)G);
		DHit **d_dst = (DHit**)d.alloc(sizeof(void*) * (size_t)G);
		MAB_CUDA(cudaMemcpyAsync(d_pos, pos_base.data(), sizeof(long long) * (size_t)G, cudaMemcpyHostToDevice, d.stream));
		MAB_CUDA(cudaMemcpyAsync(d_dst, peer.data(), sizeof(void*) * (size_t)G, cudaMemcpyHostToDevice, d.stream));
		if (n_blk) MAB_LAUNCH(d, k_push_emit, mab_grid(n_blk, 1, MAB_SMS * 8u), PUSH_LINES, 0, ln, n_lines, tab, bi_dir, carry, (uint32_t)G, n_blk, blk_off, d_pos, d_dst);
		sc_allgather_u64(d, sc, 0); // nobody sorts before everybody has finished writing: a one-word all-gather, stream-ordered after the emit kernel on every rank
		d.free(d_pos); d.free((void*)d_dst);
		d.trace("shard-ingest:emit + push over NVLink");
	}
	d.free(blk_cnt); d.free(blk_off);
	if (!push) {
	// (6b) NCCL route: hits emitted locally, bucketed by owner with a stable one-pass radix sort, exchanged in an all-to-all
	uint32_t *cnt = mab_alloc<uint32_t>(d, n_lines + 1);
	uint64_t *off = mab_alloc<uint64_t>(d, n_lines + 1);
	if (n_lines) {
		MAB_LAUNCH(d, k_line_gids, mab_grid(n_lines, 256), 256, 0, ln, n_lines, tab, bi_dir, cnt);
		size_t tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, (int64_t)n_lines, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, off, (int64_t)n_lines, d.stream);
		++d.n_lib;
	}
	DHit *loc = mab_alloc<DHit>(d, n_loc), *snd = mab_alloc<DHit>(d, n_loc);
	uint32_t *dest = mab_alloc<uint32_t>(d, n_loc), *dest2 = mab_alloc<uint32_t>(d, n_loc), *ia = mab_alloc<uint32_t>(d, n_loc), *ib = mab_alloc<uint32_t>(d, n_loc);
	if (n_loc) {
		MAB_LAUNCH(d, k_hit_emit_gid, mab_grid(n_lines, 256), 256, 0, ln, n_lines, cnt, off, tab, carry, (uint32_t)G, loc, dest);
		MAB_LAUNCH(d, k_iota32, mab_grid(n_loc, 256), 256, 0, ia, n_loc);
		cub::DoubleBuffer<uint32_t> dk(dest, dest2), dv(ia, ib);
		size_t tb = 0;
		int eb = (int)bits_for((uint64_t)G - 1);
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int64_t)n_loc, 0, eb, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int64_t)n_loc, 0, eb, d.stream); // stable: file order kept inside every bucket
		++d.n_lib;
		MAB_LAUNCH(d, k_gather_hits, mab_grid(n_loc, 256), 256, 0, loc, dv.Current(), n_loc, snd);
	}
	d.trace("shard-ingest:emit+bucket hits");
	{
		std::vector<uint64_t> sb(G), rb(G);
		for (int r = 0; r < G; ++r) sb[r] = send_cnt[r] * sizeof(DHit), rb[r] = recv_cnt[r] * sizeof(DHit);
		if (sc.active()) sc_alltoall_v(d, sc, snd, sb, h.a, rb);
		else if (n_loc) MAB_CUDA(cudaMemcpyAsync(h.a, snd, n_loc * sizeof(DHit), cudaMemcpyDeviceToDevice, d.stream));
	}
	d.sync();
	d.free(loc); d.free(snd); d.free(dest); d.free(dest2); d.free(ia); d.free(ib); d.free(cnt); d.free(off);
	}
	h.n = n_recv, h.n_seq = n_seq;
	d.trace("shard-ingest:exchange");
	d.sync();
	d.free(ln); d.free(start);
	tab_free(d, tab);
	d.free(gt.key); d.free(gt.first); d.free(gt.win); d.free(gt.id);
	d.free(g_ent); d.free(g_pos); d.free(slots); d.free(slot_of);
	std::vector<uint64_t> hits_all = sc_allgather_u64(d, sc, n_recv), parsed_all = sc_allgather_u64(d, sc, st.n_parsed);
	st.n_hits = st.n_parsed = 0;
	for (int r = 0; r < G; ++r) st.n_hits += hits_all[r], st.n_parsed += parsed_all[r];
	st.n_seq = n_seq;
	dh_sort(d, h);
	d.trace("shard-ingest:sort");
}

// =============================================================================================================
// Windowed ingest: the text comes from a source that is read twice, one window at a time, so the device never holds more
// of it than two windows (DESIGN.md 3d).  A window is a run of whole lines: it is numbered, parsed and filtered the way
// k_parse_tiles does it (8 KB tiles staged in shared memory, decoupled look-back over the window's tiles), with the global
// number of the window's first line carried from window to window in device memory.
//   pass 1  enters the names of the stored lines into the dictionary and counts the hits per name; no record is kept.  A
//           name that is new is copied into the packed name store at once and its witness re-pointed there, so nothing
//           refers to a window after its launch; first[slot] carries the sequence-length column of the occurrence it names.
//   pass 2  parses the same windows again, looks the names up and writes every hit and its mirror straight into its read's
//           bucket with the ordinal 2 * line (+ 1), as k_hit_emit does.
// =============================================================================================================
// device words of a windowed run; the two pairs (line, bl) are adjacent so that one copy hands OUT to the next window's IN
enum { WS_PARSED = 0, WS_STORED, WS_TAB_FULL, WS_STORE_FULL, WS_STORE_USED, WS_BAD, WS_EMITTED,
       WS_LINE_IN, WS_BL_IN,    // global number of the window's first line; (1 + line) << 31 | bl of the last line with an 11th field before the window
       WS_LINE_OUT, WS_BL_OUT,  // the same after the window
       WS_N };

struct WinTab {
	NameTab t;                   // key: witness offsets count through the name store first, then through the current window;
	                             // first: (2 * line + role) << 32 | sequence-length column of that occurrence
	char *store;                 // names of the dictionary, each followed by a TAB
	uint64_t store_cap;
};

// (pass 1 reads witnesses past the L1: a name stored by another CTA of the same launch may share a line with bytes cached before)
template <bool CG>
__device__ __forceinline__ bool name_at(const char *w, const char *nm, uint32_t nl)
{
	for (uint32_t i = 0; i < nl; ++i) if ((CG ? __ldcg(w + i) : w[i]) != nm[i]) return false;
	return (CG ? __ldcg(w + nl) : w[nl]) == '\t';
}

// name = nm[0 .. nl), followed by a TAB, at byte woff of the window `win`; occ = 2 * line + role, slen = its length column
__device__ __forceinline__ uint32_t win_insert(const WinTab &t, const char *win, const char *nm, uint32_t nl, uint64_t woff, uint64_t occ, uint32_t slen,
                                               unsigned long long *ws)
{
	const uint64_t h = name_hash(nm, 0, nl, 0);
	const unsigned long long frag = (h >> 37) << NT_OFF_BITS, mine = frag | (t.store_cap + woff + 1);
	uint64_t s = h & t.t.mask;
	for (int probe = 0; probe < 1 << 14; ++probe, s = (s + 1) & t.t.mask) {
		unsigned long long k = t.t.key[s];
		bool fresh = false;
		if (k == 0) {
			k = atomicCAS(&t.t.key[s], 0ull, mine);
			if (k == 0) k = mine, fresh = true;
		}
		if ((k ^ mine) >> NT_OFF_BITS) continue;                      // another fragment
		if (fresh) { // a new name: into the store, then the witness points there (until then it points at this occurrence, which stays put for the launch)
			const unsigned long long at = atomicAdd(ws + WS_STORE_USED, (unsigned long long)nl + 1);
			if (at + nl + 1 <= t.store_cap) {
				for (uint32_t i = 0; i < nl; ++i) t.store[at + i] = nm[i];
				t.store[at + nl] = '\t';
				__threadfence();
				atomicExch(&t.t.key[s], frag | (at + 1));
			} else atomicAdd(ws + WS_STORE_FULL, 1ull);
		} else {
			const uint64_t off = (k & NT_OFF_MASK) - 1;
			if (!name_at<true>(off < t.store_cap ? t.store + off : win + (off - t.store_cap), nm, nl)) continue;
		}
		const unsigned long long v = occ << 32 | slen;
		if (t.t.first[s] > v) atomicMin(&t.t.first[s], v);
		return (uint32_t)s;
	}
	atomicAdd(ws + WS_TAB_FULL, 1ull);
	return 0;
}

// pass 2: the slot of a name, NOSLOT when the dictionary of pass 1 does not have it
__device__ __forceinline__ uint32_t win_find(const WinTab &t, const char *nm, uint32_t nl)
{
	const uint64_t h = name_hash(nm, 0, nl, 0);
	uint64_t s = h & t.t.mask;
	for (int probe = 0; probe < 1 << 14; ++probe, s = (s + 1) & t.t.mask) {
		const unsigned long long k = t.t.key[s];
		if (k == 0) break;
		if ((k >> NT_OFF_BITS) == (h >> 37) && name_at<false>(t.store + ((k & NT_OFF_MASK) - 1), nm, nl)) return (uint32_t)s;
	}
	return NOSLOT;
}

// bl of the 10-field line that starts at byte s of the window: the 11th column of the closest earlier line that has one
// (paf.c:47, hit.c:73), searched backwards through the window, then what the windows before left behind
__device__ uint32_t win_prev_bl(const char *text, uint64_t s, unsigned long long carry)
{
	while (s > 0) {
		uint64_t eol = s - 1, p = eol;                                // text[eol] is the '\n' that ends the line before
		while (p > 0 && text[p - 1] != '\n') --p;
		if (eol - p > 1 && text[eol - 1] == '\r') --eol;
		uint64_t q = p;
		int tabs = 0;
		for (; q < eol && tabs < 10; ++q) tabs += text[q] == '\t';
		if (tabs == 10) {
			uint64_t f = q;
			while (f < eol && text[f] != '\t') ++f;
			return num_field(text + q, 0, (uint32_t)(f - q)) & 0x7fffffffu;
		}
		s = p;
	}
	return (uint32_t)carry & 0x7fffffffu;
}

// One window [text, text + len) of whole lines (the last window may lack the final '\n'), one tile per CTA.
// PASS 2: bfirst = bucket starts per read id (n_seq + 1), cur = fill cursors, out = the hit buckets.
template <int PASS>
__global__ void __launch_bounds__(PT_THREADS)
k_win_tiles(const char *__restrict__ text, size_t len, unsigned *tile_ctr, LineTileState tstate, int min_span, int min_match, int bi_dir, WinTab tab,
            const uint32_t *__restrict__ bfirst, uint32_t *cur, DHit *out, unsigned long long *ws)
{
	typedef cub::BlockScan<uint32_t, PT_THREADS> BS;
	__shared__ __align__(16) char s_text[PT_TILE + PT_OVER + 16];
	__shared__ uint16_t s_start[PT_LIST + 1];
	__shared__ uint32_t s_vals[PT_THREADS / 32][11][32];
	__shared__ typename BS::TempStorage s_scan;
	__shared__ typename LinePrefixOp::TempStorage s_pref;
	__shared__ unsigned long long s_first, s_tile, s_eol;
	__shared__ uint32_t s_nl;
	const uint32_t lane = threadIdx.x & 31;
	if (threadIdx.x == 0) s_tile = atomicAdd(tile_ctr, 1u), s_nl = ~0u;
	__syncthreads();
	const uint64_t t = s_tile, b0 = t * PT_TILE, b1 = b0 + PT_TILE < len ? b0 + PT_TILE : len;
	const uint64_t w_end = b1 + PT_OVER < len ? b1 + PT_OVER : len;           // staged bytes: [b0, w_end)
	{
		const uint32_t n16 = (uint32_t)((w_end - b0 + 15) >> 4);  // the tail word may reach past `len` but stays inside the (padded) window
		for (uint32_t k = threadIdx.x; k < n16; k += PT_THREADS)
			reinterpret_cast<uint4*>(s_text)[k] = __ldg(reinterpret_cast<const uint4*>(text + b0) + k);
	}
	__syncthreads();
	const uint32_t my0 = threadIdx.x * 64, lim = (uint32_t)((b1 == len ? len - 1 : b1) - b0);
	uint64_t bits = 0;
	#pragma unroll
	for (int k = 0; k < 4; ++k) bits |= (uint64_t)nl_bits_u4(reinterpret_cast<const uint4*>(s_text + my0)[k]) << (16 * k);
	bits &= lim <= my0 ? 0ull : lim - my0 >= 64 ? ~0ull : (1ull << (lim - my0)) - 1;
	const bool line0 = t == 0 && threadIdx.x == 0;            // the window's first line starts at its byte 0
	uint32_t rank, n;
	BS(s_scan).ExclusiveSum((uint32_t)__popcll(bits) + line0, rank, n);
	for (uint32_t o = lim + threadIdx.x; o < (uint32_t)(w_end - b0); o += PT_THREADS)
		if (s_text[o] == '\n' && b0 + o < len) { atomicMin(&s_nl, o); break; }
	if (threadIdx.x < 32) {
		if (t == 0) {
			if (threadIdx.x == 0) tstate.SetInclusive(0, n), s_first = 0;
		} else {
			LinePrefixOp op(tstate, s_pref, ::cuda::std::plus<unsigned long long>(), (int)t);
			const unsigned long long ex = op(n);
			if (threadIdx.x == 0) s_first = ex;
		}
	}
	__syncthreads();
	const uint64_t first = ws[WS_LINE_IN] + s_first;          // global number of the tile's first line
	if (threadIdx.x == 0 && b1 == len) ws[WS_LINE_OUT] = first + n;
	if (n == 0) return;
	uint64_t last_eol = s_nl != ~0u ? b0 + s_nl : w_end >= len ? len : ~0ull; // ~0: the tile's last line ends past the overhang
	if (last_eol == ~0ull) {
		if (threadIdx.x < 32) {
			uint64_t e = len;
			for (uint64_t p = w_end; p < len; p += 32 * 16) {
				const uint64_t q = p + 16 * lane;
				uint32_t m = 0;
				for (uint32_t k = 0; k < 16 && q + k < len; ++k) m |= (uint32_t)(text[q + k] == '\n') << k;
				const unsigned hit = __ballot_sync(0xffffffffu, m != 0);
				if (hit) { e = __shfl_sync(0xffffffffu, q + __ffs(m) - 1, __ffs(hit) - 1); break; }
			}
			if (threadIdx.x == 0) s_eol = e;
		}
		__syncthreads();
		last_eol = s_eol;
	}
	unsigned n_parsed = 0, n_pass = 0, n_bad = 0, n_emit = 0;
	unsigned long long last11 = 0;                            // (1 + line) << 31 | bl of this thread's last line with an 11th field
	for (uint32_t r0 = 0; r0 < n; r0 += PT_LIST) {
		{
			uint32_t r = rank;
			uint64_t b = bits;
			if (line0) { if (r == r0) s_start[0] = 0; ++r; }
			for (; b && r <= r0 + PT_LIST; ++r, b &= b - 1)
				if (r >= r0) s_start[r - r0] = (uint16_t)(my0 + __ffsll((long long)b));
		}
		__syncthreads();
		const uint32_t cnt = n - r0 < PT_LIST ? n - r0 : PT_LIST;
		for (uint32_t j0 = 0; j0 < cnt; j0 += PT_THREADS) {
			const uint32_t j = j0 + threadIdx.x;
			const uint64_t i = first + r0 + j;
			uint32_t sq = NOSLOT, st = 0;
			if (j < cnt) {
				const uint64_t s = b0 + s_start[j];
				uint64_t eol = r0 + j + 1 < n ? b0 + s_start[j + 1] - 1 : last_eol;
				const char *base = eol <= w_end ? s_text - b0 : text; // base + window offset = address of that byte
				if (eol - s > 1 && base[eol - 1] == '\r') --eol;
				PLine r;
				parse_line(base + s, base + eol, r, &s_vals[threadIdx.x >> 5][0][lane]);
				if (r.nf >= 10) {
					++n_parsed;
					if (PASS == 2 && r.nf >= 11) last11 = (i + 1) << 31 | (r.bl & 0x7fffffffu);
					if (!(r.qe - r.qs < (uint32_t)min_span || r.te - r.ts < (uint32_t)min_span || (int)(r.ml_rev & 0x7fffffffu) < min_match)) {
						++n_pass;
						if (PASS == 1) {
							sq = win_insert(tab, text, base + s, r.qnl, s, 2 * i, r.ql, ws);
							st = win_insert(tab, text, base + s + r.tdelta, r.tnl, s + r.tdelta, 2 * i + 1, r.tl, ws);
						} else {
							sq = win_find(tab, base + s, r.qnl), st = win_find(tab, base + s + r.tdelta, r.tnl);
							if (sq == NOSLOT || st == NOSLOT) ++n_bad;  // a name pass 1 did not see: the source delivered other bytes
							else {
								const uint32_t qid = tab.t.id[sq], tid = tab.t.id[st], ord = (uint32_t)(2 * i);
								const uint32_t bl = r.nf >= 11 ? r.bl & 0x7fffffffu : win_prev_bl(text, s, ws[WS_BL_IN]);
								uint32_t at = atomicAdd(&cur[qid], 1u);
								if (at < bfirst[qid + 1] - bfirst[qid]) {
									uint4 *o = reinterpret_cast<uint4*>(out + bfirst[qid] + at);
									o[0] = make_uint4(r.qs, ord, r.qe, tid);
									o[1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
									++n_emit;
								} else ++n_bad;                            // more hits than pass 1 counted for the read
								if (bi_dir && qid != tid) { // the same overlap seen from the target (hit.c:92-98)
									at = atomicAdd(&cur[tid], 1u);
									if (at < bfirst[tid + 1] - bfirst[tid]) {
										uint4 *o = reinterpret_cast<uint4*>(out + bfirst[tid] + at);
										o[0] = make_uint4(r.ts, ord + 1, r.te, qid);
										o[1] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
										++n_emit;
									} else ++n_bad;
								}
							}
						}
					}
				}
			}
			if (PASS == 1) { // consecutive lines often share their query read: one add per distinct slot of the warp
				const unsigned grp = __match_any_sync(0xffffffffu, sq);
				if (sq != NOSLOT && lane == (uint32_t)__ffs(grp) - 1) atomicAdd(&tab.t.hits[sq], (uint32_t)__popc(grp));
				if (sq != NOSLOT && bi_dir && st != sq) atomicAdd(&tab.t.hits[st], 1u);
			}
		}
		__syncthreads(); // the list is rewritten by the next round
	}
	n_parsed = __reduce_add_sync(0xffffffffu, n_parsed), n_pass = __reduce_add_sync(0xffffffffu, n_pass);
	if (PASS == 2) {
		n_bad = __reduce_add_sync(0xffffffffu, n_bad), n_emit = __reduce_add_sync(0xffffffffu, n_emit);
		#pragma unroll
		for (int o = 16; o; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xffffffffu, last11, o); last11 = y > last11 ? y : last11; }
	}
	if (lane == 0) {
		if (n_parsed) atomicAdd(ws + WS_PARSED, (unsigned long long)n_parsed);
		if (n_pass) atomicAdd(ws + WS_STORED, (unsigned long long)n_pass);
		if (n_bad) atomicAdd(ws + WS_BAD, (unsigned long long)n_bad);
		if (n_emit) atomicAdd(ws + WS_EMITTED, (unsigned long long)n_emit);
		if (last11) atomicMax(ws + WS_BL_OUT, last11);
	}
}

// ids and per-read counts from the dictionary of pass 1 (k_dict_rank without a text to read back from: the witness is in the
// name store and first carries the length column)
__global__ void k_win_rank(const unsigned long long *first_sorted, const uint64_t *slot_sorted, uint32_t n, WinTab t, uint64_t *noff, uint32_t *nlen, uint32_t *slen,
                           unsigned long long *tot_len, uint32_t *read_cnt)
{
	unsigned long long sum = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint64_t s = slot_sorted[i], off = (t.t.key[s] & NT_OFF_MASK) - 1;
		t.t.id[s] = i;
		read_cnt[i] = t.t.hits[s];
		uint32_t l = 0;
		while (t.store[off + l] != '\t') ++l;
		noff[i] = off, nlen[i] = l, slen[i] = (uint32_t)first_sorted[i]; // the length kept for a read is the one of its first appearance (sdict.c:36)
		sum += slen[i];
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long s = BR(ts).Sum(sum);
	if (threadIdx.x == 0 && s) atomicAdd(tot_len, s);
}

// one past the last '\n' of p[0, n) (device memory), 0 if there is none
__global__ void k_last_nl(const char *p, uint64_t n, unsigned long long *out)
{
	unsigned long long best = 0;
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) if (p[i] == '\n') best = i + 1;
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage t;
	best = BR(t).Reduce(best, cub::Max());
	if (threadIdx.x == 0 && best) atomicMax(out, best);
}

// The two windows on both sides of PCIe and what a launch over one of them needs (a device source: the device windows only).
struct WinRun {
	MabDev &d;
	const TextSource &src;
	size_t cap;                                              // bytes of a window
	char *host[2] = {nullptr, nullptr}, *dev[2] = {nullptr, nullptr};
	cudaEvent_t copied[2], parsed[2];                        // window k & 1: its bytes have landed / its launch is done
	void *ts_mem = nullptr;
	LineTileState ts;
	unsigned *ctr = nullptr;
	unsigned long long *ws = nullptr, *nl = nullptr;

	WinRun(MabDev &dev_, const TextSource &s, size_t w) : d(dev_), src(s), cap(0)
	{
		for (int i = 0; i < 2; ++i) {
			MAB_CUDA(cudaEventCreateWithFlags(&copied[i], cudaEventDisableTiming));
			MAB_CUDA(cudaEventCreateWithFlags(&parsed[i], cudaEventDisableTiming));
		}
		ctr = mab_alloc<unsigned>(d, 1);
		ws = (unsigned long long*)mab_alloc<uint64_t>(d, WS_N);
		nl = (unsigned long long*)mab_alloc<uint64_t>(d, 1);
		if (!d.copy_stream) MAB_CUDA(cudaStreamCreateWithFlags(&d.copy_stream, cudaStreamNonBlocking));
		resize(w, 0, 0);
	}
	~WinRun()
	{
		d.sync();
		MAB_CUDA(cudaStreamSynchronize(d.copy_stream));
		for (int i = 0; i < 2; ++i) {
			if (host[i]) MAB_CUDA(cudaFreeHost(host[i]));
			d.free(dev[i]);
			MAB_CUDA(cudaEventDestroy(copied[i])); MAB_CUDA(cudaEventDestroy(parsed[i]));
		}
		d.free(ts_mem); d.free(ctr); d.free(ws); d.free(nl);
	}
	// windows of w bytes, keeping the first `keep` bytes of window b (host, or device for a device source; nothing is in flight
	// when it is called with cap != 0)
	void resize(size_t w, int b, size_t keep)
	{
		if (cap) { d.sync(); MAB_CUDA(cudaStreamSynchronize(d.copy_stream)); }
		for (int i = 0; i < 2; ++i) {
			if (!src.fill) {
				char *nh;
				MAB_CUDA(cudaMallocHost(&nh, w));
				if (i == b && keep) memcpy(nh, host[i], keep);
				if (host[i]) MAB_CUDA(cudaFreeHost(host[i]));
				host[i] = nh;
			}
			char *old = dev[i];
			if (!(src.fill && i == b && keep) && old) d.free(old), old = nullptr;
			dev[i] = (char*)d.alloc(w + 64);                      // (+64: the tiles are staged in whole 16-byte words)
			if (old) { MAB_CUDA(cudaMemcpyAsync(dev[i], old, keep, cudaMemcpyDeviceToDevice, d.stream)); d.free(old); }
		}
		if (ts_mem) d.free(ts_mem);
		ts = tiles_alloc(d, w / PT_TILE + 1, &ts_mem);
		cap = w;
	}
};

// One pass over the source: false when it cannot be rewound.  *n_bytes = bytes delivered.
template <int PASS>
static bool win_pass(WinRun &w, int min_span, int min_match, int bi_dir, const WinTab &tab, const uint32_t *bfirst, uint32_t *cur, DHit *out, uint64_t *n_bytes)
{
	MabDev &d = w.d;
	if (w.src.rewind(w.src.ud) != 0) return false;
	if (tab.store_cap + w.cap >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of read names and window\n"); exit(73); }
	MAB_CUDA(cudaMemsetAsync(w.ws, 0, WS_N * 8, d.stream));
	cudaEvent_t ready;
	MAB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
	MAB_CUDA(cudaEventRecord(ready, d.stream));                 // the copies may not overtake whatever still uses the windows' memory on the main stream
	MAB_CUDA(cudaStreamWaitEvent(d.copy_stream, ready, 0));
	const char *tail = nullptr;                                 // the unfinished line after the previous window, still in its host buffer
	size_t n_tail = 0, total = 0;
	bool eof = false;
	if (w.src.fill) { // a device source: the windows are filled on the device, the unfinished line moves device to device
		size_t tail_at = 0;
		for (int b = 0; !eof; b ^= 1) {
			if (n_tail) MAB_CUDA(cudaMemcpyAsync(w.dev[b], w.dev[b ^ 1] + tail_at, n_tail, cudaMemcpyDeviceToDevice, d.stream)); // (after window b's last launch: one stream)
			size_t have = n_tail, cut = 0;
			for (;;) {
				while (have < w.cap) {
					const int64_t r = w.src.fill(w.src.ud, w.dev[b] + have, w.cap - have);
					if (r == TS_FULL) break;
					if (r < 0) {
						if (PASS == 2) { fprintf(stderr, "[E::miniasm_b200] the PAF source failed when read again after %llu bytes\n", (unsigned long long)total); exit(78); }
						d.sync();
						MAB_CUDA(cudaEventDestroy(ready));
						return false;
					}
					if (r == 0) { eof = true; break; }
					have += (size_t)r, total += (size_t)r;
				}
				if (eof) { cut = have; break; }
				if (have) {
					MAB_CUDA(cudaMemsetAsync(w.nl, 0, 8, d.stream));
					const size_t look = have < (1u << 20) ? have : (1u << 20); // the last MB first, all of it if that has no line end
					MAB_LAUNCH(d, k_last_nl, mab_grid(look, 256), 256, 0, w.dev[b] + (have - look), (uint64_t)look, w.nl);
					unsigned long long nl = 0;
					MAB_CUDA(cudaMemcpyAsync(&nl, w.nl, 8, cudaMemcpyDeviceToHost, d.stream));
					d.sync();
					if (nl) nl += have - look;
					else if (look < have) {
						MAB_LAUNCH(d, k_last_nl, mab_grid(have - look, 256), 256, 0, w.dev[b], (uint64_t)(have - look), w.nl);
						MAB_CUDA(cudaMemcpyAsync(&nl, w.nl, 8, cudaMemcpyDeviceToHost, d.stream));
						d.sync();
					}
					if (nl) { cut = (size_t)nl; break; }
				}
				w.resize(2 * w.cap, b, have);                       // a line longer than the window: the windows grow
				if (tab.store_cap + w.cap >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of read names and window\n"); exit(73); }
			}
			tail_at = cut, n_tail = have - cut;
			if (cut == 0) break;
			const uint64_t n_tile = (cut + PT_TILE - 1) / PT_TILE;
			tiles_reset(d, w.ts, n_tile);
			MAB_CUDA(cudaMemsetAsync(w.ctr, 0, 4, d.stream));
			MAB_LAUNCH(d, k_win_tiles<PASS>, (unsigned)n_tile, PT_THREADS, 0, w.dev[b], cut, w.ctr, w.ts, min_span, min_match, bi_dir, tab, bfirst, cur, out, w.ws);
			MAB_CUDA(cudaMemcpyAsync(w.ws + WS_LINE_IN, w.ws + WS_LINE_OUT, 16, cudaMemcpyDeviceToDevice, d.stream));
			MAB_CUDA(cudaEventRecord(w.parsed[b], d.stream));
		}
	}
	for (int b = 0; !eof; b ^= 1) {
		MAB_CUDA(cudaEventSynchronize(w.copied[b]));            // the window that last used this host buffer has crossed
		if (n_tail) memcpy(w.host[b], tail, n_tail);
		size_t have = n_tail, cut = 0;
		for (;;) {
			while (have < w.cap) {
				const size_t r = w.src.read(w.src.ud, w.host[b] + have, w.cap - have);
				if (r == 0) { eof = true; break; }
				have += r, total += r;
			}
			if (eof) { cut = have; break; }
			const char *nl = (const char*)memrchr(w.host[b], '\n', have);
			if (nl) { cut = (size_t)(nl - w.host[b]) + 1; break; }
			w.resize(2 * w.cap, b, have);                       // a line longer than the window: the windows grow
			if (tab.store_cap + w.cap >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of read names and window\n"); exit(73); }
		}
		tail = w.host[b] + cut, n_tail = have - cut;
		if (cut == 0) break;                                    // (the end of the source, nothing left)
		MAB_CUDA(cudaStreamWaitEvent(d.copy_stream, w.parsed[b], 0)); // the launch that last read this device window is done
		MAB_CUDA(cudaMemcpyAsync(w.dev[b], w.host[b], cut, cudaMemcpyHostToDevice, d.copy_stream));
		MAB_CUDA(cudaEventRecord(w.copied[b], d.copy_stream));
		MAB_CUDA(cudaStreamWaitEvent(d.stream, w.copied[b], 0));
		const uint64_t n_tile = (cut + PT_TILE - 1) / PT_TILE;
		tiles_reset(d, w.ts, n_tile);
		MAB_CUDA(cudaMemsetAsync(w.ctr, 0, 4, d.stream));
		MAB_LAUNCH(d, k_win_tiles<PASS>, (unsigned)n_tile, PT_THREADS, 0, w.dev[b], cut, w.ctr, w.ts, min_span, min_match, bi_dir, tab, bfirst, cur, out, w.ws);
		MAB_CUDA(cudaMemcpyAsync(w.ws + WS_LINE_IN, w.ws + WS_LINE_OUT, 16, cudaMemcpyDeviceToDevice, d.stream));
		MAB_CUDA(cudaEventRecord(w.parsed[b], d.stream));
	}
	d.sync();
	MAB_CUDA(cudaEventDestroy(ready));
	*n_bytes = total;
	return true;
}

bool ingest_paf_windowed(MabDev &d, const TextSource &src, size_t window_bytes, size_t size_hint, int min_span, int min_match, int bi_dir,
                         DHits &h, DNames &names, char **name_text_out, IngestStats &st)
{
	memset(&st, 0, sizeof(st));
	names = DNames();
	h.n = 0, h.n_seq = 0;
	*name_text_out = nullptr;
	d.trace("ingest:begin");
	if (window_bytes < (64u << 10)) window_bytes = 64u << 10;
	WinRun w(d, src, (window_bytes + PT_TILE - 1) / PT_TILE * PT_TILE);
	// table and name store from the size of the input when it is known; either one overflowing runs pass 1 again with four times the room
	uint64_t cap = tab_cap_for(line_estimate(size_hint)), store_cap = size_hint / 32 > (8u << 20) ? size_hint / 32 : (8u << 20);
	unsigned long long ws[WS_N];
	uint64_t n_bytes = 0;
	WinTab tab;
	for (;;) {
		tab.t = tab_alloc(d, cap, true);
		tab.store = (char*)d.alloc(store_cap), tab.store_cap = store_cap;
		const bool ok = win_pass<1>(w, min_span, min_match, bi_dir, tab, nullptr, nullptr, nullptr, &n_bytes);
		if (ok) { MAB_CUDA(cudaMemcpyAsync(ws, w.ws, sizeof(ws), cudaMemcpyDeviceToHost, d.stream)); d.sync(); }
		if (ok && !ws[WS_TAB_FULL] && !ws[WS_STORE_FULL]) break;
		tab_free(d, tab.t); d.free(tab.store);
		if (!ok) return false;
		if (ws[WS_TAB_FULL]) cap <<= 2;
		if (ws[WS_STORE_FULL]) store_cap <<= 2;
		++st.name_regrow;
		if (cap > (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] read-name table overflow\n"); exit(77); }
	}
	const uint64_t n_lines = ws[WS_LINE_IN];
	st.n_lines = n_lines, st.n_parsed = ws[WS_PARSED];
	const uint64_t n_stored = ws[WS_STORED];
	if (2 * n_lines >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 PAF lines on one GPU\n"); exit(73); }
	d.trace("ingest:windowed pass 1 (parse + dictionary + hit counts)");
	if (n_bytes == 0) { // (as ingest_paf leaves an empty text)
		tab_free(d, tab.t); d.free(tab.store);
		dh_reserve(d, h, 1);
		return true;
	}
	// ids = rank of the first occurrence; the hit counts of the slots become those of the reads
	uint64_t *slots = mab_alloc<uint64_t>(d, cap);
	uint32_t n_seq;
	{
		cub::CountingInputIterator<uint64_t> pos(0);
		SlotUsed used{tab.t.first};
		size_t tb = 0;
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		cub::DeviceSelect::If(nullptr, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceSelect::If(tmp, tb, pos, slots, d_n, (int64_t)cap, used, d.stream);
		++d.n_lib;
		const uint64_t n = d.get_scal(SC_NSEL);
		if (n >= (1ull << 31)) { fprintf(stderr, "[E::miniasm_b200] more than 2^31 reads\n"); exit(73); }
		n_seq = (uint32_t)n;
	}
	names.n_seq = n_seq;
	names.off = mab_alloc<uint64_t>(d, n_seq); names.nlen = mab_alloc<uint32_t>(d, n_seq); names.slen = mab_alloc<uint32_t>(d, n_seq);
	uint32_t *read_cnt = mab_alloc<uint32_t>(d, (size_t)n_seq + 1), *first = mab_alloc<uint32_t>(d, (size_t)n_seq + 1);
	MAB_CUDA(cudaMemsetAsync(read_cnt + n_seq, 0, 4, d.stream));
	if (n_seq) {
		unsigned long long *fa = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq), *fb = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq);
		uint64_t *sb = mab_alloc<uint64_t>(d, n_seq);
		MAB_LAUNCH(d, k_dict_pairs, mab_grid(n_seq, 256), 256, 0, slots, n_seq, tab.t, fa);
		cub::DoubleBuffer<unsigned long long> dk(fa, fb);
		cub::DoubleBuffer<uint64_t> dv(slots, sb);
		size_t tb = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)n_seq, 32, 64, d.stream);   // by the occurrence number, the high half
		void *tmp = d.tmp(tb);
		cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)n_seq, 32, 64, d.stream);
		++d.n_lib;
		d.zero_scal(SC_AUX, 1);
		MAB_LAUNCH(d, k_win_rank, mab_grid(n_seq, 256), 256, 0, dk.Current(), dv.Current(), n_seq, tab, names.off, names.nlen, names.slen, d.d_scal + SC_AUX, read_cnt);
		st.tot_len = d.get_scal(SC_AUX);
		d.free(fa); d.free(fb); d.free(sb);
	}
	d.free(slots);
	d.trace("ingest:rank_ids");
	dh_bucket_first(d, read_cnt, n_seq, first);
	MAB_CUDA(cudaMemsetAsync(read_cnt, 0, (size_t)n_seq * 4, d.stream)); // the counts become the buckets' fill cursors
	uint32_t n_hits;
	MAB_CUDA(cudaMemcpyAsync(&n_hits, first + n_seq, 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	dh_reserve(d, h, n_hits ? n_hits : 1);
	h.n = n_hits, h.n_seq = n_seq;
	st.n_hits = n_hits, st.n_seq = n_seq;
	// pass 2: every hit straight into its read's bucket of h.a2
	uint64_t n_bytes2 = 0;
	const bool ok2 = win_pass<2>(w, min_span, min_match, bi_dir, tab, first, read_cnt, h.a2, &n_bytes2);
	if (ok2) { MAB_CUDA(cudaMemcpyAsync(ws, w.ws, sizeof(ws), cudaMemcpyDeviceToHost, d.stream)); d.sync(); }
	tab_free(d, tab.t);
	if (!ok2) {
		d.free(tab.store); d.free(read_cnt); d.free(first);
		names_free(d, names);
		h.n = 0, h.n_seq = 0;
		return false;
	}
	if (n_bytes2 != n_bytes || ws[WS_LINE_IN] != n_lines || ws[WS_PARSED] != st.n_parsed || ws[WS_STORED] != n_stored || ws[WS_BAD] || ws[WS_EMITTED] != n_hits) {
		fprintf(stderr, "[E::miniasm_b200] the PAF source delivered a different text after rewinding: %llu bytes, %llu lines, %llu hits first, "
		        "%llu bytes, %llu lines, %llu hits (%llu without a bucket) then\n", (unsigned long long)n_bytes, (unsigned long long)n_lines, (unsigned long long)n_hits,
		        (unsigned long long)n_bytes2, ws[WS_LINE_IN], ws[WS_EMITTED], ws[WS_BAD]);
		exit(78);
	}
	*name_text_out = tab.store;   // names.off points into it (owned by the caller from now on)
	d.trace("ingest:windowed pass 2 (parse + emit_hits)");
	dh_sort_buckets(d, h, first);
	d.free(read_cnt); d.free(first);
	d.trace("ingest:sort_hits");
	return true;
}
