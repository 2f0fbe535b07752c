// inflate_host.cpp -- TEST INFRASTRUCTURE (never linked into the product): the chunked gzip decoder of
// miniasm_b200/csrc/gunzip_dev.cu run on the host, one chunk after another, over the very same inflate.cuh: find a guessed
// block start per chunk, decode every unit with unknown history (pass 1), chain the units from the true start, propagate
// the 32 KiB windows, decode the chained units again into their final place (pass 2), and check every member's CRC-32
// (per-segment raw CRCs joined by GF(2) shifts, as the CRC kernels do) and ISIZE.  tests/test_inflate_cpu.py drives it.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../miniasm_b200/csrc/inflate.cuh"

extern "C" {

// info[]: 0 units, 1 chained units, 2 chained units that are guesses (i.e. confirmed guesses), 3 members, 4 chunks
// mode: 0 guesses from the block-start test, 1 every guess forced to a wrong bit, 2 no guesses at all
int gzh_inflate(const uint8_t *gz, size_t n, size_t chunk, int mode, size_t seg, uint8_t **out, size_t *out_len, uint32_t *info)
{
	*out = nullptr, *out_len = 0;
	if (n < 2 || gz[0] != 0x1f || gz[1] != 0x8b) return -2;
	InfTables t;
	// find
	const size_t n_chunks = (n + chunk - 1) / chunk;
	std::vector<uint64_t> starts(1, 0);
	for (size_t i = 1; i < n_chunks; ++i) {
		const uint64_t b0 = (uint64_t)i * chunk * 8, b1 = (uint64_t)(i + 1 < n_chunks ? (i + 1) * chunk : n) * 8;
		if (mode == 1) { starts.push_back(b0 + 5); continue; }
		if (mode == 2) continue;
		for (uint64_t b = b0; b < b1; ++b)
			if (inf_guess_test(gz, n, b, t, 256)) { starts.push_back(b); break; }
	}
	const uint32_t nu = (uint32_t)starts.size();
	// pass 1
	std::vector<int> st(nu);
	std::vector<uint32_t> land(nu), nmem(nu);
	std::vector<uint64_t> olen(nu);
	std::vector<int64_t> mat(nu);
	std::vector<uint16_t> ring((size_t)nu * INF_WIN);
	for (uint32_t u = 0; u < nu; ++u) {
		InfOutMark o;
		o.begin(&ring[(size_t)u * INF_WIN]);
		uint32_t j = u + 1;
		st[u] = inf_run(gz, n, starts[u], u == 0, starts.data(), nu, &j, t, o);
		land[u] = j, olen[u] = o.p, mat[u] = o.member_at, nmem[u] = o.n_members;
	}
	// chain
	std::vector<uint32_t> chain;
	std::vector<uint64_t> off;
	std::vector<uint32_t> mbase;
	uint64_t total = 0;
	uint32_t members = 0;
	for (uint32_t u = 0;;) {
		if (st[u] < 0) return -2;
		chain.push_back(u), off.push_back(total), mbase.push_back(members);
		total += olen[u], members += nmem[u];
		if (st[u] == INF_END) break;
		u = land[u];
	}
	const uint32_t nc = (uint32_t)chain.size();
	// window
	std::vector<uint8_t> win((size_t)(nc + 1) * INF_WIN, 0);
	std::vector<uint32_t> valid(nc + 1, 0);
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		for (uint32_t k = 0; k < INF_WIN; ++k)
			win[(size_t)(c + 1) * INF_WIN + k] = inf_window_byte(&ring[(size_t)u * INF_WIN], olen[u], &win[(size_t)c * INF_WIN], k);
		valid[c + 1] = inf_window_valid(valid[c], olen[u], mat[u]);
	}
	// resolve
	uint8_t *txt = (uint8_t*)malloc(total ? total : 1);
	std::vector<uint64_t> m_end(members ? members : 1);
	std::vector<uint32_t> m_crc(members ? members : 1), m_isz(members ? members : 1);
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		InfOutByte o;
		o.out = txt + off[c], o.win = &win[(size_t)c * INF_WIN], o.p = 0, o.cap = olen[u], o.lim = -(int64_t)valid[c];
		o.m_end = &m_end[mbase[c]], o.m_crc = &m_crc[mbase[c]], o.m_isize = &m_isz[mbase[c]], o.n_members = 0, o.m_cap = nmem[u];
		uint32_t j = u + 1;
		const int r = inf_run(gz, n, starts[u], u == 0, starts.data(), nu, &j, t, o);
		if (r != st[u] || o.p != olen[u] || o.n_members != nmem[u] || (r == INF_LAND && j != land[u])) { free(txt); return -2; }
		for (uint32_t k = 0; k < nmem[u]; ++k) m_end[mbase[c] + k] += off[c];
	}
	// crc: raw CRCs of fixed segments of the text, joined per member (head piece, whole segments, tail piece)
	uint32_t tab[256], x2k[64];
	inf_crc_table(tab), inf_x2k_table(x2k);
	const uint64_t n_seg = (total + seg - 1) / seg;
	std::vector<uint32_t> sc(n_seg ? n_seg : 1);
	for (uint64_t s = 0; s < n_seg; ++s) sc[s] = inf_crc_raw(tab, 0, txt + s * seg, (s + 1) * seg < total ? seg : total - s * seg);
	const uint32_t xs = inf_x8n(x2k, seg);
	for (uint32_t m = 0; m < members; ++m) {
		const uint64_t a = m ? m_end[m - 1] : 0, b = m_end[m];
		uint64_t A = (a + seg - 1) / seg * seg, B = b / seg * seg;
		if (A > b) A = b;
		if (B < A) B = A;
		uint32_t raw = inf_crc_raw(tab, 0, txt + a, A - a);
		for (uint64_t s = A / seg; s < B / seg; ++s) raw = inf_gf2_mul(raw, xs) ^ sc[s];
		raw = inf_crc_join(x2k, raw, inf_crc_raw(tab, 0, txt + B, b - B), b - B);
		if (inf_crc_final(x2k, raw, b - a) != m_crc[m] || (uint32_t)(b - a) != m_isz[m]) { free(txt); return -2; }
	}
	uint32_t confirmed = 0;
	for (uint32_t c = 1; c < nc; ++c) confirmed += chain[c] != 0;
	info[0] = nu, info[1] = nc, info[2] = confirmed, info[3] = members, info[4] = (uint32_t)n_chunks;
	*out = txt, *out_len = total;
	return 0;
}

void gzh_free(uint8_t *p) { free(p); }

// pass 1 from an arbitrary bit of an arbitrary byte string, with every later chunk start of `chunk` bytes as a landing point;
// returns the status (and the output length through *out_len)
int gzh_decode_at(const uint8_t *gz, size_t n, uint64_t bit, int at_header, size_t chunk, uint64_t *out_len)
{
	static uint16_t ring[INF_WIN];
	InfTables t;
	std::vector<uint64_t> starts;
	for (uint64_t b = (bit / 8 / chunk + 1) * chunk * 8; b < (uint64_t)n * 8; b += chunk * 8) starts.push_back(b + 3);
	InfOutMark o;
	o.begin(ring);
	uint32_t j = 0;
	const int r = inf_run(gz, n, bit, at_header != 0, starts.data(), (uint32_t)starts.size(), &j, t, o);
	*out_len = o.p;
	return r;
}

int gzh_guess_at(const uint8_t *gz, size_t n, uint64_t bit)
{
	InfTables t;
	return inf_guess_test(gz, n, bit, t, 256);
}

uint32_t gzh_crc32(const uint8_t *p, size_t n, size_t seg) // the CRC-32 through the segment join
{
	uint32_t tab[256], x2k[64];
	inf_crc_table(tab), inf_x2k_table(x2k);
	uint32_t raw = 0;
	for (size_t s = 0; s < n; s += seg) {
		const size_t l = n - s < seg ? n - s : seg;
		raw = inf_crc_join(x2k, raw, inf_crc_raw(tab, 0, p + s, l), l);
	}
	return inf_crc_final(x2k, raw, n);
}

}
