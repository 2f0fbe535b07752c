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
// GPU shape: (1) line starts (newline count per tile, scan, positions), (2) one thread per line parses it, applies the store
// filter and enters both names into an exact open-addressing dictionary (slot word = hash fragment + byte offset of a witness
// occurrence: an occurrence with the same fragment compares its bytes with the witness's; value = smallest occurrence number,
// atomicMin) -- all in ONE pass that leaves a 32-byte record per line, (3) distinct names ranked by first occurrence = ids,
// (4) hits emitted at scanned offsets, (5) radix sort (hit_dev.cu).  ingest_paf_stream runs (1)-(2) chunk by chunk while the next
// chunks of the text are still crossing PCIe.
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

// Streaming variants (ingest_paf_stream): tiles [t0, t1) of the text have just arrived.  nl_state[0] = newline-started lines
// seen so far (line 0 starts at byte 0 and is not counted), nl_state[1] = capacity of `out`.
__global__ void __launch_bounds__(NL_THREADS) k_nl_count_range(const char *__restrict__ text, size_t len, uint64_t t0, uint64_t t1, uint64_t *cnt)
{
	typedef cub::BlockReduce<uint32_t, NL_THREADS> BR;
	__shared__ typename BR::TempStorage ts;
	for (uint64_t t = t0 + blockIdx.x; t < t1; t += gridDim.x) {
		uint32_t c = 0;
		#pragma unroll
		for (int k = 0; k < NL_PER_THREAD; ++k) c += __popc(nl_bits16(text, len, t * NL_TILE + ((uint64_t)k * NL_THREADS + threadIdx.x) * 16));
		c = BR(ts).Sum(c);
		if (threadIdx.x == 0) cnt[t - t0] = c;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(NL_THREADS) k_nl_write_range(const char *__restrict__ text, size_t len, uint64_t t0, uint64_t t1, const uint64_t *__restrict__ base,
                                                              const unsigned long long *nl_state, uint64_t *out)
{
	typedef cub::BlockScan<uint32_t, NL_THREADS> BS;
	__shared__ typename BS::TempStorage ts;
	const uint64_t seen = nl_state[0], cap = nl_state[1];
	for (uint64_t t = t0 + blockIdx.x; t < t1; t += gridDim.x) {
		uint64_t at = seen + base[t - t0];
		#pragma unroll
		for (int k = 0; k < NL_PER_THREAD; ++k) {
			const uint64_t off = t * NL_TILE + ((uint64_t)k * NL_THREADS + threadIdx.x) * 16;
			uint32_t bits = nl_bits16(text, len, off), rank, total;
			BS(ts).ExclusiveSum((uint32_t)__popc(bits), rank, total);
			uint64_t q = at + rank;
			while (bits) { const int b = __ffs(bits) - 1; if (q + 1 < cap) out[q + 1] = off + b + 1; ++q; bits &= bits - 1; }
			at += total;
			__syncthreads();
		}
	}
}

// after the tiles [t0, t1): lines whose END is known now are [rng[0], rng[1]); rng[2] = total number of lines once the text is complete
__global__ void k_nl_advance(unsigned long long *nl_state, const uint64_t *base, const uint64_t *cnt, uint64_t n_tiles, unsigned long long *rng, int last)
{
	if (blockIdx.x || threadIdx.x) return;
	const unsigned long long seen = nl_state[0] + (n_tiles ? base[n_tiles - 1] + cnt[n_tiles - 1] : 0);
	nl_state[0] = seen;
	const unsigned long long known_starts = seen + 1;                 // lines 0 .. seen have a start
	unsigned long long cap = nl_state[1];
	unsigned long long hi = last ? known_starts : known_starts - 1;   // the last known line's end is the next line's start, or the end of the text
	if (hi > cap - 1) hi = cap - 1;                                   // (overflow of the estimate: start[] is only filled below cap; the host notices and falls back)
	rng[0] = rng[1] > hi ? hi : rng[1];                               // previous upper bound becomes the lower one
	rng[1] = hi;
	rng[2] = last ? known_starts : ~0ull;
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

// One CTA parses PARSE_LINES consecutive lines.  Their bytes are contiguous in the file, so the CTA first copies
// the whole range into shared memory with coalesced 128-bit loads and the threads then walk their own line there:
// byte-wise walking of global memory makes every warp-level load touch ~16 cache lines (L1 wavefront bound).
// A range that does not fit (very long lines) is parsed straight from global memory.
// Fused into the same pass (round 1 ran them as three more sweeps over a 64-byte record): the store filter of
// hit.c:85 and the dictionary insert of both names, while the line is still in shared memory.
constexpr int PARSE_LINES = 128;
constexpr int PARSE_SMEM = 16 * 1024;

__global__ void __launch_bounds__(PARSE_LINES)
k_parse(const char *__restrict__ text, size_t len, const uint64_t *__restrict__ start, const unsigned long long *__restrict__ rng,
        int min_span, int min_match, NameTab tab, PRec *out, unsigned long long *counts)
{	// rng: lines [rng[0], rng[1]) are parsed; rng[2] = number of lines of the whole text, or ~0 while it is still arriving (then
	// line rng[1] exists and its start ends line rng[1]-1).  counts: [0] lines with >= 10 fields, [1] lines stored, [2] dictionary overflow
	__shared__ __align__(16) char s_text[PARSE_SMEM];
	__shared__ uint32_t s_vals[PARSE_LINES / 32][11][32];
	unsigned n_parsed = 0, n_pass = 0;
	const uint64_t line_lo = rng[0], line_hi = rng[1], n_lines = rng[2];
	const uint64_t n_blk = (line_hi - line_lo + PARSE_LINES - 1) / PARSE_LINES;
	for (uint64_t b = blockIdx.x; b < n_blk; b += gridDim.x) {
		const uint64_t l0 = line_lo + b * PARSE_LINES, l1 = l0 + PARSE_LINES < line_hi ? l0 + PARSE_LINES : line_hi;
		const uint64_t s0 = start[l0], s1 = l1 < n_lines ? start[l1] : len;
		const uint64_t a0 = s0 & ~(uint64_t)15;
		const bool staged = s1 - a0 <= PARSE_SMEM;
		__syncthreads(); // the previous range is no longer needed
		if (staged) {
			const uint64_t n16 = (s1 - a0 + 15) >> 4; // whole 16-byte words; the tail word may reach past `len` but stays inside the (padded) allocation
			for (uint64_t k = threadIdx.x; k < n16; k += PARSE_LINES)
				reinterpret_cast<uint4*>(s_text)[k] = __ldg(reinterpret_cast<const uint4*>(text + a0) + k);
		}
		__syncthreads();
		const uint64_t i = l0 + threadIdx.x;
		if (i < l1) {
			const uint64_t s = start[i];
			uint64_t eol = i + 1 < n_lines ? start[i + 1] - 1 : (text[len - 1] == '\n' ? len - 1 : len);
			const char *base = staged ? s_text - a0 : text; // base + file offset = address of that byte
			if (eol - s > 1 && base[eol - 1] == '\r') --eol;
			PLine r;
			parse_line(base + s, base + eol, r, &s_vals[threadIdx.x >> 5][0][threadIdx.x & 31]);
			PRec o;
			o.qs = r.qs, o.qe = r.qe, o.ts = r.ts, o.te = r.te, o.ml_rev = r.ml_rev;
			o.bl_f = (r.bl & 0x7fffffffu) | (r.nf >= 11 ? 0x80000000u : 0u);
			o.slot_q = NOSLOT, o.slot_t = 0;
			if (r.nf >= 10) {
				++n_parsed;
				if (!(r.qe - r.qs < (uint32_t)min_span || r.te - r.ts < (uint32_t)min_span || (int)(r.ml_rev & 0x7fffffffu) < min_match)) {
					++n_pass;
					o.slot_q = tab_insert(tab, text, base + s, r.qnl, s, 2 * i, counts + 2);
					o.slot_t = tab_insert(tab, text, base + s + r.tdelta, r.tnl, s + r.tdelta, 2 * i + 1, counts + 2);
				}
			}
			*reinterpret_cast<uint4*>(out + i) = make_uint4(o.qs, o.qe, o.ts, o.te);
			*(reinterpret_cast<uint4*>(out + i) + 1) = make_uint4(o.ml_rev, o.bl_f, o.slot_q, o.slot_t);
		}
	}
	n_parsed = __reduce_add_sync(0xffffffffu, n_parsed), n_pass = __reduce_add_sync(0xffffffffu, n_pass);
	if ((threadIdx.x & 31) == 0) {
		if (n_parsed) atomicAdd(counts, (unsigned long long)n_parsed);
		if (n_pass) atomicAdd(counts + 1, (unsigned long long)n_pass);
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

__global__ void k_nocont_drop(PRec *ln, uint64_t n_lines, const uint8_t *excl, NameTab t)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t sq = ln[i].slot_q, st = ln[i].slot_t;
		if (sq == NOSLOT) continue;
		if (excl[sq] || excl[st]) { ln[i].slot_q = NOSLOT; continue; }
		if (t.first[sq] > 2 * i) atomicMin(&t.first[sq], (unsigned long long)(2 * i));
		if (t.first[st] > 2 * i + 1) atomicMin(&t.first[st], (unsigned long long)(2 * i + 1));
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

__global__ void k_dict_rank(const unsigned long long *first_sorted, const uint64_t *slot_sorted, uint32_t n, NameTab t,
                            const char *text, const uint64_t *start, uint64_t *noff, uint32_t *nlen, uint32_t *slen, unsigned long long *tot_len)
{
	unsigned long long sum = 0;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		t.id[slot_sorted[i]] = i;
		occ_name(text, start, first_sorted[i], &noff[i], &nlen[i], &slen[i]); // the length kept for a read is the one of its first appearance (sdict.c:36)
		sum += slen[i];
	}
	typedef cub::BlockReduce<unsigned long long, 256> BR;
	__shared__ typename BR::TempStorage ts;
	unsigned long long s = BR(ts).Sum(sum);
	if (threadIdx.x == 0 && s) atomicAdd(tot_len, s);
}

// --------------------------------------------------------------------------------------------- hits
__global__ void k_hit_count(const PRec *ln, uint64_t n_lines, int bi_dir, uint32_t *cnt)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint2 sl = *reinterpret_cast<const uint2*>(&ln[i].slot_q);
		cnt[i] = sl.x != NOSLOT ? (bi_dir && sl.x != sl.y ? 2 : 1) : 0;
	}
}

__global__ void k_hit_emit(const PRec *ln, uint64_t n_lines, const uint32_t *cnt, const uint64_t *off, NameTab t, DHit *out, unsigned *max_qs)
{
	unsigned mx = 0;
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t c = cnt[i];
		if (c == 0) continue;
		const PRec r = ln[i];
		const uint32_t qid = t.id[r.slot_q], tid = t.id[r.slot_t], bl = line_bl(ln, i, 0);
		uint4 *o = reinterpret_cast<uint4*>(out + off[i]);
		o[0] = make_uint4(r.qs, qid, r.qe, tid);
		o[1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
		mx = r.qs > mx ? r.qs : mx;
		if (c == 2) { // the same overlap seen from the target (hit.c:92-98)
			o[2] = make_uint4(r.ts, tid, r.te, qid);
			o[3] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
			mx = r.ts > mx ? r.ts : mx;
		}
	}
	mx = __reduce_max_sync(0xffffffffu, mx);
	if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_qs, mx);
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

constexpr int SC_RNG = 40;   // d_scal[40..42]: the line range k_parse works on (lo, hi, total or ~0)

static void set_rng(MabDev &d, uint64_t lo, uint64_t hi, uint64_t total)
{
	const unsigned long long v[3] = { lo, hi, total };
	MAB_CUDA(cudaMemcpyAsync(d.d_scal + SC_RNG, v, sizeof(v), cudaMemcpyHostToDevice, d.stream));
}

static NameTab tab_alloc(MabDev &d, uint64_t cap)
{
	NameTab tab;
	tab.key = (unsigned long long*)mab_alloc<uint64_t>(d, cap);
	tab.first = (unsigned long long*)mab_alloc<uint64_t>(d, cap);
	tab.id = mab_alloc<uint32_t>(d, cap);
	tab.mask = cap - 1;
	MAB_CUDA(cudaMemsetAsync(tab.key, 0, cap * 8, d.stream));
	MAB_CUDA(cudaMemsetAsync(tab.first, 0xff, cap * 8, d.stream));
	return tab;
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

	d.trace("ingest:begin");
	// (1) line starts: count newlines per 16 KB tile, scan the tile counts, write the positions
	uint64_t n_lines;
	uint64_t *start = dev_line_starts(d, d_text, len, &n_lines);
	st.n_lines = n_lines;
	d.trace("ingest:line_starts");

	// (2) parse + store filter + dictionary insert in one pass; the table grows (and the pass repeats) until every name has a slot
	if (len >= (1ull << NT_OFF_BITS) - 1) { fprintf(stderr, "[E::miniasm_b200] more than 2^37 bytes of PAF on one GPU\n"); exit(73); }
	PRec *ln = mab_alloc<PRec>(d, n_lines);
	NameTab tab{nullptr, nullptr, nullptr, 0};
	uint64_t cap = 1ull << 20;
	while (cap < n_lines / 4) cap <<= 1;                 // ~50 lines name a read twice each: load <= 1/6 at that ratio; overflow quadruples it
	for (;;) {
		tab = tab_alloc(d, cap);
		d.zero_scal(SC_COUNT, 4);
		set_rng(d, 0, n_lines, n_lines);
		MAB_LAUNCH(d, k_parse, mab_grid((n_lines + PARSE_LINES - 1) / PARSE_LINES, 1, MAB_SMS * 16u), PARSE_LINES, 0, d_text, len, start, d.d_scal + SC_RNG, min_span, min_match, tab, ln, d.d_scal + SC_COUNT);
		st.n_parsed = d.get_scal(SC_COUNT);
		if (d.h_scal[SC_COUNT + 2] == 0) break;
		d.free(tab.key); d.free(tab.first); d.free(tab.id);
		cap <<= 2;
		if (cap > (1ull << 33)) { fprintf(stderr, "[E::miniasm_b200] read-name table overflow\n"); exit(77); }
	}
	ingest_finish(d, d_text, len, start, ln, n_lines, tab, cap, bi_dir, nocont, h, names, st);
}

// Front end of an ingest with the text still on the host: it crosses PCIe in 64 MB chunks on a copy stream while the chunks that
// have arrived are scanned for line starts and parsed (store filter, dictionary) on the context's stream -- k_parse needs nothing
// global any more.  host_text may be pageable or pinned (pinned overlaps fully); d_text has room for len + 64.  Capacities are
// estimates (a 12-column line has >= 24 bytes): false = the text broke them (or the dictionary overflowed), nothing is kept and the
// caller parses the now-resident text the plain way.  No collectives inside (the sharded ingest calls it rank by rank).
static bool stream_parse(MabDev &d, char *d_text, const char *host_text, size_t len, int min_span, int min_match,
                         uint64_t **start_out, PRec **ln_out, NameTab *tab_out, uint64_t *cap_out, uint64_t *n_lines_out, uint64_t *n_parsed_out)
{
	const uint64_t CH_TILES = (64ull << 20) / NL_TILE, n_tile = (len + NL_TILE - 1) / NL_TILE;       // 64 MB chunks, whole tiles
	const uint64_t n_chunk = (n_tile + CH_TILES - 1) / CH_TILES;
	const uint64_t line_cap = len / 24 + 1024;
	uint64_t cap = 1ull << 20;
	while (cap < line_cap / 8) cap <<= 1;
	uint64_t *start = mab_alloc<uint64_t>(d, line_cap + 1);
	PRec *ln = mab_alloc<PRec>(d, line_cap);
	uint64_t *cnt = mab_alloc<uint64_t>(d, CH_TILES + 1), *base = mab_alloc<uint64_t>(d, CH_TILES + 1);
	unsigned long long *state = (unsigned long long*)mab_alloc<uint64_t>(d, 8);   // [0] newline-started lines seen, [1] capacity; [4..6] = rng
	NameTab tab = tab_alloc(d, cap);
	{
		const unsigned long long init[8] = { 0, line_cap, 0, 0, 0, 0, ~0ull, 0 };
		MAB_CUDA(cudaMemcpyAsync(state, init, sizeof(init), cudaMemcpyHostToDevice, d.stream));
		MAB_CUDA(cudaMemsetAsync(start, 0, 8, d.stream));
	}
	d.zero_scal(SC_COUNT, 4);
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, base, (int64_t)CH_TILES, d.stream);
	void *tmp = d.tmp(tb);
	if (!d.copy_stream) MAB_CUDA(cudaStreamCreateWithFlags(&d.copy_stream, cudaStreamNonBlocking));
	std::vector<cudaEvent_t> ev(n_chunk);
	cudaEvent_t ready;
	MAB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
	MAB_CUDA(cudaEventRecord(ready, d.stream));                 // the copies may not overtake whatever still uses d_text on the main stream
	MAB_CUDA(cudaStreamWaitEvent(d.copy_stream, ready, 0));
	for (uint64_t k = 0; k < n_chunk; ++k) { // copy k is issued before the kernels of chunk k: a pageable source blocks the host per chunk, not for the whole text
		const uint64_t t0 = k * CH_TILES, t1 = (k + 1) * CH_TILES < n_tile ? (k + 1) * CH_TILES : n_tile;
		const uint64_t b0 = t0 * NL_TILE, b1 = t1 * NL_TILE < len ? t1 * NL_TILE : len;
		MAB_CUDA(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
		MAB_CUDA(cudaMemcpyAsync(d_text + b0, host_text + b0, b1 - b0, cudaMemcpyHostToDevice, d.copy_stream));
		MAB_CUDA(cudaEventRecord(ev[k], d.copy_stream));
		MAB_CUDA(cudaStreamWaitEvent(d.stream, ev[k], 0));
		MAB_LAUNCH(d, k_nl_count_range, mab_grid(t1 - t0, 1, MAB_SMS * 8u), NL_THREADS, 0, d_text, len, t0, t1, cnt);
		cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, base, (int64_t)(t1 - t0), d.stream);
		++d.n_lib;
		MAB_LAUNCH(d, k_nl_write_range, mab_grid(t1 - t0, 1, MAB_SMS * 8u), NL_THREADS, 0, d_text, len, t0, t1, base, state, start);
		MAB_LAUNCH(d, k_nl_advance, 1, 32, 0, state, base, cnt, t1 - t0, state + 4, (int)(k + 1 == n_chunk));
		MAB_LAUNCH(d, k_parse, MAB_SMS * 8u, PARSE_LINES, 0, d_text, len, start, state + 4, min_span, min_match, tab, ln, d.d_scal + SC_COUNT);
	}
	unsigned long long fin[8];
	MAB_CUDA(cudaMemcpyAsync(fin, state, sizeof(fin), cudaMemcpyDeviceToHost, d.stream));
	*n_parsed_out = d.get_scal(SC_COUNT);                       // (synchronises)
	for (uint64_t k = 0; k < n_chunk; ++k) MAB_CUDA(cudaEventDestroy(ev[k]));
	MAB_CUDA(cudaEventDestroy(ready));
	d.free(cnt); d.free(base); d.free(state);
	const uint64_t n_lines = fin[0] + 1;
	if (n_lines >= line_cap || d.h_scal[SC_COUNT + 2] != 0) {   // estimates broken (very short lines / more names than slots)
		d.free(start); d.free(ln); d.free(tab.key); d.free(tab.first); d.free(tab.id);
		return false;
	}
	*start_out = start, *ln_out = ln, *tab_out = tab, *cap_out = cap, *n_lines_out = n_lines;
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
	uint64_t *start; PRec *ln; NameTab tab; uint64_t cap, n_lines, n_parsed;
	if (!stream_parse(d, d_text, host_text, len, min_span, min_match, &start, &ln, &tab, &cap, &n_lines, &n_parsed)) {
		ingest_paf(d, d_text, len, min_span, min_match, bi_dir, h, names, st, nullptr); // the text is resident now: the plain path sizes exactly
		return;
	}
	st.n_parsed = n_parsed, st.n_lines = n_lines;
	d.trace("ingest:stream (copy + line starts + parse + dictionary)");
	ingest_finish(d, d_text, len, start, ln, n_lines, tab, cap, bi_dir, nullptr, h, names, st);
}

static void ingest_finish(MabDev &d, const char *d_text, size_t len, uint64_t *start, PRec *ln, uint64_t n_lines, NameTab tab, uint64_t cap, int bi_dir,
                          const NoContParams *nocont, DHits &h, DNames &names, IngestStats &st)
{
	uint32_t *cnt = nullptr;
	uint64_t *off = nullptr;
	d.trace("ingest:dictionary");
	if (nocont) { // -R: mark the contained reads, drop every line that names one, take the first appearances again
		uint8_t *excl = mab_alloc<uint8_t>(d, cap);
		MAB_CUDA(cudaMemsetAsync(excl, 0, cap, d.stream));
		MAB_LAUNCH(d, k_nocont_mark, mab_grid(n_lines, 256), 256, 0, ln, n_lines, d_text, start, nocont->max_hang, nocont->int_frac, excl);
		d.zero_scal(SC_AUX, 1);
		MAB_LAUNCH(d, k_count_u8, mab_grid(cap, 256), 256, 0, excl, cap, d.d_scal + SC_AUX);
		MAB_CUDA(cudaMemsetAsync(tab.first, 0xff, cap * 8, d.stream));
		MAB_LAUNCH(d, k_nocont_drop, mab_grid(n_lines, 256), 256, 0, ln, n_lines, excl, tab);
		st.n_dropped = d.get_scal(SC_AUX);
		d.free(excl);
		d.trace("ingest:-R prefilter");
	}
	// (4) ids = rank of the first occurrence
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
		MAB_LAUNCH(d, k_dict_rank, mab_grid(n_seq, 256), 256, 0, dk.Current(), dv.Current(), n_seq, tab, d_text, start, names.off, names.nlen, names.slen, d.d_scal + SC_AUX);
		st.tot_len = d.get_scal(SC_AUX);
		d.free(fa); d.free(fb); d.free(sb);
	}
	d.free(slots);

	d.trace("ingest:rank_ids");
	// (5) hits at scanned offsets (file order, mirrored hit right after its original)
	cnt = mab_alloc<uint32_t>(d, n_lines);
	off = mab_alloc<uint64_t>(d, n_lines + 1);
	MAB_LAUNCH(d, k_hit_count, mab_grid(n_lines, 256), 256, 0, ln, n_lines, bi_dir, cnt);
	{
		size_t tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, (int64_t)n_lines, d.stream);
		void *tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, off, (int64_t)n_lines, d.stream);
		++d.n_lib;
	}
	uint64_t last_off;
	uint32_t last_cnt;
	MAB_CUDA(cudaMemcpyAsync(&last_off, off + n_lines - 1, 8, cudaMemcpyDeviceToHost, d.stream));
	MAB_CUDA(cudaMemcpyAsync(&last_cnt, cnt + n_lines - 1, 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	const uint64_t n_hits = last_off + last_cnt;
	dh_reserve(d, h, n_hits ? n_hits : 1);
	h.n = n_hits, h.n_seq = n_seq;
	d.zero_scal(SC_AUX, 1);
	if (n_hits) MAB_LAUNCH(d, k_hit_emit, mab_grid(n_lines, 256), 256, 0, ln, n_lines, cnt, off, tab, h.a, (unsigned*)(d.d_scal + SC_AUX));
	uint32_t max_qs = (uint32_t)(d.get_scal(SC_AUX) & 0xffffffffu);
	st.n_hits = n_hits, st.n_seq = n_seq, st.max_qs_bits = bits_for(max_qs);
	d.free(cnt); d.free(off); d.free(ln); d.free(start);
	d.free(tab.key); d.free(tab.first); d.free(tab.id);

	d.trace("ingest:emit_hits");
	// (6) ma_hit_sort
	dh_sort(d, h, st.max_qs_bits);
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

__global__ void k_gtab_winner(const GEntry *ent, uint64_t n, GTab t, const uint32_t *slot_of)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
		if (t.first[slot_of[i]] == ent[i].first) t.win[slot_of[i]] = (uint32_t)i; // first occurrences are unique: exactly one winner
}

__global__ void k_gtab_verify(const GEntry *ent, uint64_t n, GTab t, const uint32_t *slot_of, const uint64_t *name_pos, const char *names, unsigned long long *n_bad)
{
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
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
                               DHit *out, uint32_t *dest, unsigned *max_qs)
{
	unsigned mx = 0;
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t c = cnt[i];
		if (c == 0) continue;
		const PRec r = ln[i];
		const uint32_t qid = lt.id[r.slot_q], tid = lt.id[r.slot_t], bl = line_bl(ln, i, carry_bl);
		uint4 *o = reinterpret_cast<uint4*>(out + off[i]);
		o[0] = make_uint4(r.qs, qid, r.qe, tid);
		o[1] = make_uint4(r.ts, r.te, r.ml_rev, bl);
		dest[off[i]] = qid % world;
		mx = r.qs > mx ? r.qs : mx;
		if (c == 2) {
			o[2] = make_uint4(r.ts, tid, r.te, qid);
			o[3] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
			dest[off[i] + 1] = tid % world;
			mx = r.ts > mx ? r.ts : mx;
		}
	}
	mx = __reduce_max_sync(0xffffffffu, mx);
	if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_qs, mx);
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
                                                          const uint64_t *__restrict__ blk_off, const long long *__restrict__ pos_base, DHit *const *__restrict__ dst, unsigned *max_qs)
{
	__shared__ uint32_t s_wc[PUSH_LINES / 32][32];
	__shared__ uint32_t s_seg[33];                                  // exclusive prefix of the block's per-destination totals
	__shared__ __align__(16) uint4 s_hit[2 * 2 * PUSH_LINES];        // up to two hits per line, two 16-byte halves per hit
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt_mask = (1u << lane) - 1u;
	unsigned mx = 0;
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
			mx = r.qs > mx ? r.qs : mx;
			if (p.has1) { // the same overlap seen from the target (hit.c:92-98)
				const uint32_t k1 = s_seg[p.d1] + w1 + r1;
				s_hit[2 * k1] = make_uint4(r.ts, p.tid, r.te, p.qid);
				s_hit[2 * k1 + 1] = make_uint4(r.qs, r.qe, r.ml_rev, bl);
				mx = r.ts > mx ? r.ts : mx;
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
	mx = __reduce_max_sync(0xffffffffu, mx);
	if (lane == 0 && mx) atomicMax(max_qs, mx);
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
	uint64_t *start = nullptr, n_lines = 0, cap = 1ull << 20, n_parsed = 0;
	PRec *ln = nullptr;
	NameTab tab{nullptr, nullptr, nullptr, 0};
	bool have = false;                                      // this rank holds a finished local parse
	if (host_text && len) {
		have = stream_parse(d, d_text, host_text, len, min_span, min_match, &start, &ln, &tab, &cap, &n_lines, &n_parsed);
		if (!have) cap = 1ull << 20;
		d.trace("shard-ingest:stream (copy + line starts + parse + dictionary)");
	}
	if (!have) {
		if (len) start = dev_line_starts(d, d_text, len, &n_lines);
		ln = mab_alloc<PRec>(d, n_lines);
		while (cap < n_lines / 4) cap <<= 1;
	}
	for (;;) {
		bool overflow = false;
		if (!have) {
			tab = tab_alloc(d, cap);
			d.zero_scal(SC_COUNT, 4);
			set_rng(d, 0, n_lines, n_lines);
			if (n_lines) MAB_LAUNCH(d, k_parse, mab_grid((n_lines + PARSE_LINES - 1) / PARSE_LINES, 1, MAB_SMS * 16u), PARSE_LINES, 0, d_text, len, start, d.d_scal + SC_RNG, min_span, min_match, tab, ln, d.d_scal + SC_COUNT);
			n_parsed = d.get_scal(SC_COUNT);
			overflow = d.h_scal[SC_COUNT + 2] != 0;
		}
		// every rank must take the same branch: agree on the outcome
		std::vector<uint64_t> f = sc_allgather_u64(d, sc, overflow);
		bool any = false;
		for (int r = 0; r < G; ++r) any |= f[r] != 0;
		if (!any) break;
		d.free(tab.key); d.free(tab.first); d.free(tab.id);   // (a rank whose own table was fine parses again too: same branch everywhere)
		have = false;
		cap <<= 2;
		if (cap > (1ull << 33)) { fprintf(stderr, "[E::miniasm_b200] read-name table overflow\n"); exit(77); }
	}
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
		++st.hash_retries;
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
	uint32_t max_qs = 0;
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
		d.zero_scal(SC_AUX, 1);
		if (n_blk) MAB_LAUNCH(d, k_push_emit, mab_grid(n_blk, 1, MAB_SMS * 8u), PUSH_LINES, 0, ln, n_lines, tab, bi_dir, carry, (uint32_t)G, n_blk, blk_off, d_pos, d_dst, (unsigned*)(d.d_scal + SC_AUX));
		max_qs = (uint32_t)(d.get_scal(SC_AUX) & 0xffffffffu);
		{ // nobody sorts before everybody has finished writing: a one-word all-reduce, stream-ordered after the emit kernel on every rank
			std::vector<uint64_t> mq = sc_allgather_u64(d, sc, max_qs);
			for (int r = 0; r < G; ++r) if (mq[r] > max_qs) max_qs = (uint32_t)mq[r];
		}
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
	d.zero_scal(SC_AUX, 1);
	if (n_loc) {
		MAB_LAUNCH(d, k_hit_emit_gid, mab_grid(n_lines, 256), 256, 0, ln, n_lines, cnt, off, tab, carry, (uint32_t)G, loc, dest, (unsigned*)(d.d_scal + SC_AUX));
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
	max_qs = (uint32_t)(d.get_scal(SC_AUX) & 0xffffffffu);
	{
		std::vector<uint64_t> sb(G), rb(G);
		for (int r = 0; r < G; ++r) sb[r] = send_cnt[r] * sizeof(DHit), rb[r] = recv_cnt[r] * sizeof(DHit);
		if (sc.active()) sc_alltoall_v(d, sc, snd, sb, h.a, rb);
		else if (n_loc) MAB_CUDA(cudaMemcpyAsync(h.a, snd, n_loc * sizeof(DHit), cudaMemcpyDeviceToDevice, d.stream));
	}
	{ // sort key width must cover the largest query start of any rank
		std::vector<uint64_t> mq = sc_allgather_u64(d, sc, max_qs);
		for (int r = 0; r < G; ++r) if (mq[r] > max_qs) max_qs = (uint32_t)mq[r];
	}
	d.sync();
	d.free(loc); d.free(snd); d.free(dest); d.free(dest2); d.free(ia); d.free(ib); d.free(cnt); d.free(off);
	}
	h.n = n_recv, h.n_seq = n_seq;
	d.trace("shard-ingest:exchange");
	d.sync();
	d.free(ln); d.free(start);
	d.free(tab.key); d.free(tab.first); d.free(tab.id);
	d.free(gt.key); d.free(gt.first); d.free(gt.win); d.free(gt.id);
	d.free(g_ent); d.free(g_pos); d.free(slots); d.free(slot_of);
	std::vector<uint64_t> hits_all = sc_allgather_u64(d, sc, n_recv), parsed_all = sc_allgather_u64(d, sc, st.n_parsed);
	st.n_hits = st.n_parsed = 0;
	for (int r = 0; r < G; ++r) st.n_hits += hits_all[r], st.n_parsed += parsed_all[r];
	st.n_seq = n_seq, st.max_qs_bits = bits_for(max_qs);
	dh_sort(d, h, st.max_qs_bits);
	d.trace("shard-ingest:sort");
}
