// gzstream_host.cpp -- TEST INFRASTRUCTURE (never linked into the product): the streaming gzip decoder of
// miniasm_b200/csrc/gunzip_dev.cu (GzStream) run on the host over the very same inflate.cuh and gzstream.cuh.  Each fill takes a
// compressed segment from the carried bit position (copied into a buffer of exactly its length, so a sanitizer sees any read
// past it), guesses block starts per chunk, decodes every unit with unknown history, chains them by gzs_chain, propagates the
// 32 KiB windows from the carried history, decodes the chained units again into the caller's buffer and checks the CRC-32 and
// ISIZE of every member that ends in the segment, joined to the carried raw CRC.  tests/test_gzstream_cpu.py drives it.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../miniasm_b200/csrc/gzstream.cuh"

namespace {
struct Stream {
	const uint8_t *gz;
	uint64_t len, seg_fixed, chunk_fixed;
	uint64_t pos = 0, carry_len = 0, need = 0, next_seg = 0, in_used = 0, out_made = 0;
	bool hdr = true, done = false;
	uint32_t valid = 0, carry_raw = 0;
	std::vector<uint8_t> hist = std::vector<uint8_t>(INF_WIN, 0);
	uint64_t n_seg = 0, n_grow = 0, n_units = 0, n_chain = 0;
	void rewind()
	{
		pos = 0, carry_len = 0, need = 0, next_seg = 0, hdr = true, done = false, valid = 0, carry_raw = 0;
		memset(hist.data(), 0, INF_WIN);
	}
};

enum { R_REJECT = -2, R_SMALL = -3, R_GROW = -4 };

int64_t step(Stream &s, uint8_t *dst, uint64_t cap, uint64_t base, uint64_t n, bool final, uint64_t *need)
{
	++s.n_seg;
	std::vector<uint8_t> gz(s.gz + base, s.gz + base + n); // exactly the segment
	const uint8_t *g = gz.data();
	InfTables t;
	const uint64_t chunk = s.chunk_fixed ? s.chunk_fixed : gzs_chunk_for(n), n_chunks = (n + chunk - 1) / chunk;
	std::vector<uint64_t> starts(1, s.pos & 7);
	for (uint64_t i = 1; i < n_chunks; ++i) {
		const uint64_t b0 = i * chunk * 8, b1 = (i + 1 < n_chunks ? (i + 1) * chunk : n) * 8;
		for (uint64_t b = b0; b < b1; ++b)
			if (inf_guess_test(g, n, b, t, 256)) { starts.push_back(b); break; }
	}
	const uint32_t nu = (uint32_t)starts.size();
	s.n_units += nu;
	std::vector<int> st(nu);
	std::vector<uint32_t> land(nu), nmem(nu);
	std::vector<uint64_t> olen(nu);
	std::vector<int64_t> mat(nu);
	std::vector<uint16_t> ring((size_t)nu * INF_WIN);
	for (uint32_t u = 0; u < nu; ++u) {
		InfOutMark o;
		o.begin(&ring[(size_t)u * INF_WIN]);
		uint32_t j = u + 1;
		st[u] = inf_run(g, n, starts[u], u == 0 && s.hdr, starts.data(), nu, &j, t, o);
		land[u] = j, olen[u] = o.p, mat[u] = o.member_at, nmem[u] = o.n_members;
	}
	std::vector<uint32_t> chain(nu), mbase(nu);
	std::vector<uint64_t> off(nu);
	GzsChain r;
	gzs_chain(st.data(), land.data(), olen.data(), nmem.data(), final, cap, chain.data(), off.data(), mbase.data(), r);
	if (r.kind == GZS_BAD) return R_REJECT;
	if (r.kind == GZS_GROW) return R_GROW;
	if (r.kind == GZS_SMALL) { *need = olen[0]; return R_SMALL; }
	const uint64_t need_next = r.kind == GZS_STOP && st[r.stop] == INF_LAND ? olen[r.stop] : 0;
	const uint32_t nc = r.nc;
	s.n_chain += nc;
	std::vector<uint8_t> win((size_t)(nc + 1) * INF_WIN);
	std::vector<uint32_t> valid(nc + 1);
	memcpy(win.data(), s.hist.data(), INF_WIN), valid[0] = s.valid;
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		for (uint32_t k = 0; k < INF_WIN; ++k)
			win[(size_t)(c + 1) * INF_WIN + k] = inf_window_byte(&ring[(size_t)u * INF_WIN], olen[u], &win[(size_t)c * INF_WIN], k);
		valid[c + 1] = inf_window_valid(valid[c], olen[u], mat[u]);
	}
	const uint64_t members = r.members;
	std::vector<uint64_t> m_end(members + 1);
	std::vector<uint32_t> m_crc(members + 1), m_isz(members + 1);
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		InfOutByte o;
		o.out = dst + off[c], o.win = &win[(size_t)c * INF_WIN], o.p = 0, o.cap = olen[u], o.lim = -(int64_t)valid[c];
		o.m_end = &m_end[mbase[c]], o.m_crc = &m_crc[mbase[c]], o.m_isize = &m_isz[mbase[c]], o.n_members = 0, o.m_cap = nmem[u];
		uint32_t j = u + 1;
		const int q = inf_run(g, n, starts[u], u == 0 && s.hdr, starts.data(), nu, &j, t, o);
		if (q != st[u] || o.p != olen[u] || o.n_members != nmem[u] || (q == INF_LAND && j != land[u])) return R_REJECT;
		for (uint32_t k = 0; k < nmem[u]; ++k) m_end[mbase[c] + k] += off[c];
	}
	uint32_t tab[256], x2k[64];
	inf_crc_table(tab), inf_x2k_table(x2k);
	uint32_t carry_raw = 0;
	uint64_t carry_len = 0;
	for (uint32_t m = 0; m <= members; ++m) {
		const uint64_t a = m ? m_end[m - 1] : 0, b = m < members ? m_end[m] : r.total;
		uint32_t raw = inf_crc_raw(tab, 0, dst + a, b - a);
		uint64_t len = b - a;
		gzs_piece(x2k, s.carry_raw, s.carry_len, m, raw, len);
		if (m == members) carry_raw = raw, carry_len = len;
		else if (!gzs_member_ok(x2k, raw, len, m_crc[m], m_isz[m])) return R_REJECT;
	}
	memcpy(s.hist.data(), &win[(size_t)nc * INF_WIN], INF_WIN);
	s.valid = valid[nc], s.carry_raw = carry_raw, s.carry_len = carry_len, s.hdr = false;
	s.need = gzs_need_after(need_next, cap, r.total);
	const uint64_t pos = r.kind == GZS_LAST ? s.len * 8 : gzs_next_bit(base * 8, starts.data(), r.stop);
	s.in_used += (pos - s.pos) / 8, s.out_made += r.total;
	s.next_seg = gzs_seg_len(cap, s.in_used, s.out_made);
	s.pos = pos;
	if (r.kind == GZS_LAST) s.done = true;
	return (int64_t)r.total;
}
}

extern "C" {

void *gzs_open(const uint8_t *gz, uint64_t len, uint64_t seg, uint64_t chunk)
{
	Stream *s = new Stream();
	s->gz = gz, s->len = len, s->seg_fixed = seg, s->chunk_fixed = chunk;
	return s;
}

void gzs_close(void *h) { delete (Stream*)h; }
void gzs_rewind(void *h) { ((Stream*)h)->rewind(); }

// the next at most cap inflated bytes into dst: their number (0 at the end), -2 rejected, -3 the next piece alone is *need bytes.
// seg = 0 (at open): segment lengths as GzStream picks them (gzs_seg_len, the room memo)
int64_t gzs_fill(void *h, uint8_t *dst, uint64_t cap, uint64_t *need)
{
	Stream &s = *(Stream*)h;
	if (s.len < 18) return R_REJECT;
	if (!s.seg_fixed && !s.done && gzs_room_short(s.need, cap)) { *need = s.need; return R_SMALL; }
	while (!s.done) {
		const uint64_t base = s.pos >> 3;
		uint64_t seg = s.seg_fixed ? s.seg_fixed : s.next_seg ? s.next_seg : gzs_seg_len(cap, s.in_used, s.out_made);
		for (;;) {
			const uint64_t n = seg < s.len - base ? seg : s.len - base;
			const int64_t r = step(s, dst, cap, base, n, base + n == s.len, need);
			if (r == R_GROW) { seg *= 2, ++s.n_grow; continue; }
			if (r != 0 || s.done) return r;
			break; // nothing but empty output: the next segment
		}
	}
	return 0;
}

void gzs_counts(void *h, uint64_t *out) // segments decoded, of them grown, units, chained units
{
	Stream &s = *(Stream*)h;
	out[0] = s.n_seg, out[1] = s.n_grow, out[2] = s.n_units, out[3] = s.n_chain;
}

}
