// inflate.cuh -- DEFLATE (RFC 1951) / gzip (RFC 1952) decoding core shared by the CUDA kernels of gunzip_dev.cu and the
// host build of tests/hostsim/inflate_host.cpp.  Everything here is __host__ __device__ and bounded: a decode can start at
// any bit of any byte string (a false guess of a block start decodes garbage) and must neither read nor write out of bounds
// nor run forever.  Every table built from a block header is validated before use, every input read past the end is caught
// at the next symbol, and every back-reference is checked against the output the decoder is allowed to see.
//
// The parallel scheme (DESIGN.md section 3c) decodes one "unit" per guessed block start, twice:
//   pass 1 (InfOutMark): unknown history.  Output goes to a 32 KiB ring of 16-bit cells; a byte copied from before the
//     unit's own first output byte is stored as a marker 256 + w, naming byte w of the 32 KiB window that precedes the unit.
//   pass 2 (InfOutByte): the resolved window of the predecessor is known; bytes go straight to their final place.
// Both passes stop at the first block boundary that lands exactly on a later unit's start (INF_LAND), or at the end of the
// input right after a gzip trailer (INF_END).  A fault found only after reading past the end of the input is INF_SHORT: with
// the whole file that is truncation, with a piece of it (the streaming decoder of gzstream.cuh) it asks for more bytes.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define INF_HD __host__ __device__ __forceinline__
#define INF_HD_NOINL __host__ __device__
#else
#define INF_HD inline
#define INF_HD_NOINL inline
#endif

enum { INF_END = 1, INF_LAND = 2, INF_ERR = -1, INF_SHORT = -2 };
enum { INF_WIN = 32768, INF_WMASK = INF_WIN - 1 };
#define INF_CRC_POLY 0xEDB88320u

// ---- bit reader: LSB-first over in[0, nbytes); bytes past the end read as zero and are caught by over() -------------------
struct InfIn {
	const uint8_t *p;
	uint64_t nbytes, byte; // next byte to load (may pass nbytes: virtual zeros)
	uint64_t buf;
	int cnt;
	INF_HD void init(const uint8_t *in, uint64_t n, uint64_t bit)
	{
		p = in, nbytes = n, byte = bit >> 3, buf = 0, cnt = 0;
		refill();
		drop((int)(bit & 7));
	}
	INF_HD void refill()
	{
		while (cnt <= 56) {
			const uint64_t v = byte < nbytes ? p[byte] : 0;
			buf |= v << cnt, ++byte, cnt += 8;
		}
	}
	INF_HD uint64_t pos() const { return byte * 8 - (uint64_t)cnt; }
	INF_HD bool over() const { return pos() > nbytes * 8; }
	INF_HD uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1)); }
	INF_HD void drop(int n) { buf >>= n, cnt -= n; }
	INF_HD uint32_t bits(int n) { if (cnt < n) refill(); uint32_t v = peek(n); drop(n); return v; } // n <= 32
	INF_HD void align() { drop(cnt & 7); }
};

// ---- canonical Huffman code: counts per length, symbols in code order, and an LB-bit first-level lookup --------------------
// lut entry: sym | len << 9 (len 1..LB); 0 = the next LB bits start a longer (or unassigned) code -> bit-serial walk
template <int NSYM, int LB>
struct InfHuff {
	uint16_t cnt[16];
	uint16_t sym[NSYM];
	uint16_t lut[1 << LB];
	int nsym;
	// returns the Kraft slack: 0 complete, > 0 incomplete, < 0 over-subscribed (the table is unusable then)
	INF_HD int build(const uint8_t *len, int n, bool with_lut)
	{
		uint16_t offs[16];
		for (int l = 0; l < 16; ++l) cnt[l] = 0;
		for (int s = 0; s < n; ++s) ++cnt[len[s]];
		int left = 1;
		for (int l = 1; l < 16; ++l) {
			left = left * 2 - cnt[l];
			if (left < 0) return left;
		}
		offs[1] = 0;
		for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + cnt[l]);
		for (int s = 0; s < n; ++s) if (len[s]) sym[offs[len[s]]++] = (uint16_t)s;
		nsym = n;
		if (with_lut) {
			for (int i = 0; i < (1 << LB); ++i) lut[i] = 0;
			uint32_t code = 0;
			int k = 0;
			for (int l = 1; l <= LB; ++l) {
				for (int c = 0; c < cnt[l]; ++c, ++code, ++k) {
					uint32_t r = 0;
					for (int b = 0; b < l; ++b) r |= ((code >> b) & 1u) << (l - 1 - b);
					const uint16_t e = (uint16_t)(sym[k] | (l << 9));
					for (uint32_t f = r; f < (1u << LB); f += 1u << l) lut[f] = e;
				}
				code <<= 1;
			}
		}
		return left;
	}
	// bit-serial walk over the canonical code; -1 for an unassigned code
	INF_HD int walk(InfIn &in) const
	{
		int code = 0, first = 0, index = 0;
		for (int l = 1; l < 16; ++l) {
			code |= (int)in.bits(1);
			const int c = cnt[l];
			if (code - first < c) return sym[index + code - first];
			index += c, first += c, first <<= 1, code <<= 1;
		}
		return -1;
	}
	INF_HD int decode(InfIn &in, bool with_lut) const
	{
		if (with_lut) {
			const uint16_t e = lut[in.peek(LB)];
			if (e) { in.drop(e >> 9); return e & 511; }
		}
		return walk(in);
	}
};

typedef InfHuff<288, 10> InfLit;
typedef InfHuff<32, 8> InfDist;
typedef InfHuff<19, 7> InfCL;

struct InfTables {
	InfLit lit;
	InfDist dist;
	int kind; // 0 none, 1 fixed, 2 dynamic
};

INF_HD void inf_len_code(int s, int &base, int &extra) // s = symbol - 257, 0..28
{
	if (s < 8) base = 3 + s, extra = 0;
	else if (s < 28) extra = (s >> 2) - 1, base = ((4 + (s & 3)) << extra) + 3;
	else base = 258, extra = 0;
}

INF_HD void inf_dist_code(int s, int &base, int &extra) // 0..29
{
	if (s < 4) base = 1 + s, extra = 0;
	else extra = (s >> 1) - 1, base = ((2 + (s & 1)) << extra) + 1;
}

INF_HD bool inf_single_code(const uint16_t *cnt) // zlib-compatible exception to completeness: one code of length 1
{
	for (int l = 2; l < 16; ++l) if (cnt[l]) return false;
	return cnt[1] == 1;
}

// Fixed codes of BTYPE=01 (RFC 1951 3.2.6)
INF_HD void inf_build_fixed(InfTables &t, bool with_lut)
{
	uint8_t l[288];
	for (int i = 0; i < 288; ++i) l[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
	t.lit.build(l, 288, with_lut);
	for (int i = 0; i < 32; ++i) l[i] = 5;
	t.dist.build(l, 32, with_lut);
	t.kind = 1;
}

// Header of a BTYPE=10 block (after BFINAL/BTYPE).  strict: both codes complete (the block-start test); otherwise the rules a
// conforming decoder applies (a single one-bit code is allowed, and a distance code may be empty).  Returns false on any fault.
INF_HD_NOINL bool inf_read_dynamic(InfIn &in, InfTables &t, bool strict, bool with_lut)
{
	static const uint8_t ord[19] = { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };
	in.refill();
	const int nlen = (int)in.bits(5) + 257, ndist = (int)in.bits(5) + 1, ncode = (int)in.bits(4) + 4;
	if (nlen > 286 || ndist > 30) return false;
	uint8_t l[286 + 30];
	for (int i = 0; i < 19; ++i) l[i] = 0;
	for (int i = 0; i < ncode; ++i) l[ord[i]] = (uint8_t)in.bits(3);
	InfCL cl;
	if (cl.build(l, 19, true) != 0) return false; // the code-length code must be complete
	const int n = nlen + ndist;
	for (int i = 0; i < n;) {
		in.refill();
		const int s = cl.decode(in, true);
		if (s < 0) return false;
		if (s < 16) { l[i++] = (uint8_t)s; continue; }
		int rep, v = 0;
		if (s == 16) { if (i == 0) return false; v = l[i - 1], rep = 3 + (int)in.bits(2); }
		else if (s == 17) rep = 3 + (int)in.bits(3);
		else rep = 11 + (int)in.bits(7);
		if (i + rep > n) return false;
		while (rep--) l[i++] = (uint8_t)v;
	}
	if (in.over() || l[256] == 0) return false;
	const int ll = t.lit.build(l, nlen, with_lut);
	if (ll < 0 || (ll > 0 && (strict || !inf_single_code(t.lit.cnt)))) return false;
	const int dl = t.dist.build(l + nlen, ndist, with_lut);
	if (dl < 0) return false;
	if (dl > 0) { // incomplete: only one one-bit code, or none at all (a block of literals only)
		bool empty = true;
		for (int k = 1; k < 16; ++k) if (t.dist.cnt[k]) empty = false;
		if (strict || (!empty && !inf_single_code(t.dist.cnt))) return false;
	}
	t.kind = 2;
	return true;
}

// ---- CRC-32 (RFC 1952 8) -----------------------------------------------------------------------------------------------
INF_HD uint32_t inf_crc_bitwise(uint32_t crc, const uint8_t *p, uint64_t n) // standard pre/post-inverted CRC, no table
{
	crc = ~crc;
	for (uint64_t i = 0; i < n; ++i) {
		crc ^= p[i];
		for (int k = 0; k < 8; ++k) crc = (crc >> 1) ^ (crc & 1 ? INF_CRC_POLY : 0);
	}
	return ~crc;
}

INF_HD void inf_crc_table(uint32_t *t) // t[b] = raw CRC register after feeding byte b into a zero register
{
	for (uint32_t b = 0; b < 256; ++b) {
		uint32_t c = b;
		for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (c & 1 ? INF_CRC_POLY : 0);
		t[b] = c;
	}
}

// raw CRC register of a byte string (zero start, no final inversion): linear in the data, so for strings A, B
// raw(A B) = raw(A) * x^(8|B|) + raw(B) over GF(2) modulo the CRC polynomial
INF_HD uint32_t inf_crc_raw(const uint32_t *t, uint32_t c, const uint8_t *p, uint64_t n)
{
	for (uint64_t i = 0; i < n; ++i) c = t[(c ^ p[i]) & 255] ^ (c >> 8);
	return c;
}

// product of two polynomials modulo the CRC polynomial, in the reflected bit order of the CRC register (bit 31 = x^0)
INF_HD uint32_t inf_gf2_mul(uint32_t a, uint32_t b)
{
	uint32_t p = 0;
	for (int i = 0; i < 32; ++i) {
		if (a & (0x80000000u >> i)) p ^= b;
		b = (b >> 1) ^ (b & 1 ? INF_CRC_POLY : 0); // b * x
	}
	return p;
}

INF_HD void inf_x2k_table(uint32_t *x2k) // x2k[k] = x^(2^k), k < 64
{
	x2k[0] = 0x40000000u; // x^1
	for (int k = 1; k < 64; ++k) x2k[k] = inf_gf2_mul(x2k[k - 1], x2k[k - 1]);
}

INF_HD uint32_t inf_x8n(const uint32_t *x2k, uint64_t n) // x^(8n)
{
	uint32_t r = 0x80000000u; // x^0
	for (int k = 0; n && k < 61; ++k, n >>= 1) if (n & 1) r = inf_gf2_mul(r, x2k[k + 3]);
	return r;
}

INF_HD uint32_t inf_crc_join(const uint32_t *x2k, uint32_t raw_a, uint32_t raw_b, uint64_t len_b)
{
	return inf_gf2_mul(raw_a, inf_x8n(x2k, len_b)) ^ raw_b;
}

// the standard CRC-32 of a string of n bytes from its raw register
INF_HD uint32_t inf_crc_final(const uint32_t *x2k, uint32_t raw, uint64_t n)
{
	return ~(raw ^ inf_gf2_mul(0xffffffffu, inf_x8n(x2k, n)));
}

// ---- gzip member header (RFC 1952 2.3) at byte `at`: returns the byte offset of the deflate data, -1 for a bad header or -2
// for one the input ends inside (every byte present so far is a valid header prefix)
INF_HD int64_t inf_gzip_header(const uint8_t *p, uint64_t n, uint64_t at)
{
	uint64_t i = at;
	if (at >= n) return -2;
	if (p[i] != 0x1f || (n - i > 1 && p[i + 1] != 0x8b) || (n - i > 2 && p[i + 2] != 8) || (n - i > 3 && (p[i + 3] & 0xe0))) return -1;
	if (n < 10 || at > n - 10) return -2;
	const uint8_t flg = p[i + 3];
	i += 10;
	if (flg & 4) { // FEXTRA
		if (i + 2 > n) return -2;
		const uint64_t xlen = p[i] | (uint64_t)p[i + 1] << 8;
		i += 2;
		if (xlen > n - i) return -2;
		i += xlen;
	}
	for (int f = 8; f <= 16; f <<= 1) if (flg & f) { // FNAME, FCOMMENT: zero-terminated
		while (i < n && p[i]) ++i;
		if (i >= n) return -2;
		++i;
	}
	if (flg & 2) { // FHCRC: the two low bytes of the CRC-32 of the header up to here
		if (i + 2 > n) return -2;
		const uint32_t c = inf_crc_bitwise(0, p + at, i - at);
		if ((c & 0xffff) != (uint32_t)(p[i] | p[i + 1] << 8)) return -1;
		i += 2;
	}
	return (int64_t)i;
}

// ---- output policies ----------------------------------------------------------------------------------------------------
// pass 1: unknown history.  lim is the lowest output position a distance may reach: -INF_WIN before the unit meets a member
// start (then a marker is written), the member's first position after it.
struct InfOutMark {
	uint16_t *ring;  // INF_WIN cells, indexed by position & INF_WMASK
	uint64_t p;
	int64_t lim;
	int64_t member_at; // output position of the last member start in this unit, -1 = none
	uint32_t n_members;
	INF_HD void begin(uint16_t *r) { ring = r, p = 0, lim = -INF_WIN, member_at = -1, n_members = 0; }
	INF_HD bool lit(uint32_t b) { ring[p & INF_WMASK] = (uint16_t)b, ++p; return true; }
	INF_HD bool copy(int len, int dist)
	{
		const int64_t src = (int64_t)p - dist;
		if (src < lim) return false;
		for (int k = 0; k < len; ++k) {
			const int64_t s = src + k;
			ring[p & INF_WMASK] = s >= 0 ? ring[(uint64_t)s & INF_WMASK] : (uint16_t)(256 + (s + INF_WIN));
			++p;
		}
		return true;
	}
	INF_HD void member_start() { lim = (int64_t)p, member_at = (int64_t)p; }
	INF_HD bool member_end(uint32_t, uint32_t) { ++n_members; return true; }
};

// pass 2: bytes to out[0, cap), history = the 32 KiB that precede the unit (win, of which the last `valid` bytes exist)
struct InfOutByte {
	uint8_t *out;
	const uint8_t *win;
	uint64_t p, cap;
	int64_t lim;
	// member trailers met, in order: end position (relative to the unit), CRC-32 and ISIZE
	uint64_t *m_end; uint32_t *m_crc, *m_isize;
	uint32_t n_members, m_cap;
	INF_HD bool lit(uint32_t b) { if (p >= cap) return false; out[p++] = (uint8_t)b; return true; }
	INF_HD bool copy(int len, int dist)
	{
		const int64_t src = (int64_t)p - dist;
		if (src < lim || p + (uint64_t)len > cap) return false;
		for (int k = 0; k < len; ++k) {
			const int64_t s = src + k;
			out[p] = s >= 0 ? out[s] : win[INF_WIN + s];
			++p;
		}
		return true;
	}
	INF_HD void member_start() { lim = (int64_t)p; }
	INF_HD bool member_end(uint32_t crc, uint32_t isize)
	{
		if (n_members >= m_cap) return false;
		if (m_end) m_end[n_members] = p, m_crc[n_members] = crc, m_isize[n_members] = isize;
		++n_members;
		return true;
	}
};

// literal bytes a PAF, FASTA or FASTQ file holds: printable ASCII, tab, CR, LF (used only to pick guesses)
INF_HD bool inf_plausible(uint32_t b) { return (b >= 0x20 && b < 0x7f) || b == '\t' || b == '\n' || b == '\r'; }

// ---- the decode loop ----------------------------------------------------------------------------------------------------
// Decodes from `bit` (at_header: a gzip member header starts at byte bit/8) until the first block boundary that equals
// starts[j] for some j >= *j (INF_LAND, *j = that unit), or the end of input right after a trailer (INF_END).  starts[] is
// ascending.  Any fault gives INF_ERR.
template <class Out>
INF_HD_NOINL int inf_run(const uint8_t *gz, uint64_t n, uint64_t bit, bool at_header, const uint64_t *starts, uint32_t n_starts,
                         uint32_t *j, InfTables &t, Out &o)
{
	InfIn in;
	in.init(gz, n, bit);
	bool header = at_header, first = true;
	t.kind = 0;
#define INF_FAIL return in.over() ? INF_SHORT : INF_ERR
	for (;;) {
		if (header) { // byte-aligned here
			const uint64_t at = in.pos() >> 3;
			const int64_t d = inf_gzip_header(gz, n, at);
			if (d < 0) return d == -2 ? INF_SHORT : INF_ERR;
			in.init(gz, n, (uint64_t)d * 8);
			o.member_start();
			header = false;
		}
		if (!first) {
			const uint64_t b = in.pos();
			while (*j < n_starts && starts[*j] < b) ++*j;
			if (*j < n_starts && starts[*j] == b) return INF_LAND;
		}
		first = false;
		in.refill();
		const uint32_t bfinal = in.bits(1), btype = in.bits(2);
		if (btype == 0) {
			in.align();
			const uint32_t len = in.bits(16), nlen = in.bits(16);
			if (in.over()) return INF_SHORT;
			if ((len ^ 0xffffu) != nlen) return INF_ERR;
			const uint64_t at = in.pos() >> 3;
			if (at > n || len > n - at) return INF_SHORT;
			for (uint32_t k = 0; k < len; ++k) if (!o.lit(gz[at + k])) return INF_ERR;
			in.init(gz, n, (at + len) * 8);
		} else if (btype == 3) {
			INF_FAIL;
		} else {
			if (btype == 1) { if (t.kind != 1) inf_build_fixed(t, true); }
			else if (!inf_read_dynamic(in, t, false, true)) INF_FAIL;
			for (;;) {
				in.refill();
				const int s = t.lit.decode(in, true);
				if (s < 256) {
					if (s < 0 || !o.lit((uint32_t)s)) INF_FAIL;
				} else if (s == 256) {
					break;
				} else {
					if (s > 285) INF_FAIL;
					int base, extra, dbase, dextra;
					inf_len_code(s - 257, base, extra);
					const int len = base + (int)in.bits(extra);
					const int ds = t.dist.decode(in, true);
					if (ds < 0 || ds > 29) INF_FAIL;
					inf_dist_code(ds, dbase, dextra);
					const int dist = dbase + (int)in.bits(dextra);
					if (in.over() || !o.copy(len, dist)) INF_FAIL;
				}
				if (in.over()) return INF_SHORT;
			}
			if (btype == 2) t.kind = 0;
		}
		if (in.over()) return INF_SHORT;
		if (bfinal) { // trailer: CRC-32, ISIZE; then the end of the input or the next member
			in.align();
			const uint64_t at = in.pos() >> 3;
			if (at > n || n - at < 8) return INF_SHORT;
			const uint8_t *q = gz + at;
			const uint32_t crc = q[0] | q[1] << 8 | q[2] << 16 | (uint32_t)q[3] << 24;
			const uint32_t isz = q[4] | q[5] << 8 | q[6] << 16 | (uint32_t)q[7] << 24;
			if (!o.member_end(crc, isz)) return INF_ERR;
			if (at + 8 == n) return INF_END;
			in.init(gz, n, (at + 8) * 8);
			header = true;
		}
	}
#undef INF_FAIL
}

// ---- window step: byte k of the 32 KiB window that follows a unit, from its pass-1 ring and the window that precedes it -----
// A marker the preceding window cannot back (it sits before a member start) reads an arbitrary window byte: no valid distance
// reaches it, and pass 2 checks every distance exactly.
INF_HD uint8_t inf_window_byte(const uint16_t *ring, uint64_t out_len, const uint8_t *win_in, uint32_t k)
{
	const int64_t pos = (int64_t)out_len - INF_WIN + (int64_t)k;
	if (pos < 0) return win_in[out_len + k];
	const uint32_t v = ring[(uint64_t)pos & INF_WMASK];
	return v < 256 ? (uint8_t)v : win_in[(v - 256) & INF_WMASK];
}

INF_HD uint32_t inf_window_valid(uint32_t valid_in, uint64_t out_len, int64_t member_at)
{
	const uint64_t v = member_at >= 0 ? out_len - (uint64_t)member_at : valid_in + out_len;
	return v < INF_WIN ? (uint32_t)v : (uint32_t)INF_WIN;
}

// ---- block-start test: is there a plausible BTYPE=10 block header at `bit`? ------------------------------------------------
// Both codes complete, end-of-block coded, and a trial decode of up to `trial` symbols (or to the end of the block) with
// unknown history emits only plausible literals.  Only picks guesses: correctness never depends on it.
INF_HD_NOINL bool inf_guess_test(const uint8_t *gz, uint64_t n, uint64_t bit, InfTables &t, int trial)
{
	InfIn in;
	in.init(gz, n, bit);
	const uint32_t h = in.peek(3);
	if ((h >> 1) != 2) return false;
	const uint32_t nl = (in.buf >> 3) & 31, nd = (in.buf >> 8) & 31;
	if (nl > 29 || nd > 29) return false;
	in.drop(3);
	if (!inf_read_dynamic(in, t, true, false)) return false;
	for (int k = 0; k < trial; ++k) {
		in.refill();
		const int s = t.lit.decode(in, false);
		if (s < 0 || s > 285) return false;
		if (s < 256) { if (!inf_plausible((uint32_t)s)) return false; continue; }
		if (s == 256) break;
		int base, extra;
		inf_len_code(s - 257, base, extra);
		in.bits(extra);
		const int ds = t.dist.decode(in, false);
		if (ds < 0 || ds > 29) return false;
		inf_dist_code(ds, base, extra);
		in.bits(extra);
		if (in.over()) return false;
	}
	return !in.over();
}
