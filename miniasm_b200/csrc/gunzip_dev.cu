// gunzip_dev.cu -- the kernels of the GPU gzip decoder (gunzip_dev.cuh, DESIGN.md section 3c) over the inflate.cuh core:
//   k_gz_find     one block per chunk of compressed bytes: the first bit offset that passes the block-start test
//   k_gz_compact  unit starts = the true start (bit 0) + the chunks' guesses, ascending
//   k_gz_decode   pass 1, one thread per unit: decode with unknown history into a 32 KiB ring of bytes and window markers
//   k_gz_chain    walk the units from the true start along the confirmed landings; output offsets and member slots
//   k_gz_window   in chain order, the resolved 32 KiB window after each chained unit
//   k_gz_resolve  pass 2, one thread per chained unit: decode again with the true window, bytes straight into place
//   k_gz_crc_seg / k_gz_crc_member   raw CRC-32 per fixed segment, joined per member by GF(2) shifts, checked with ISIZE
#include "gunzip_dev.cuh"
#include "inflate.cuh"
#include <cstdio>
#include <cstdlib>
#include <vector>

#define GZ_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
	fprintf(stderr, "[E::miniasm_b200] %s failed at %s:%d: %s\n", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); \
	exit(70); } } while (0)

static const size_t GZ_CHUNK = 64u << 10;   // compressed bytes per chunk (DESIGN.md 3c: measured on config 3)
static const size_t GZ_SEG = 16u << 10;     // output bytes per CRC segment
static const int GZ_TRIAL = 256;            // symbols of the block-start test's trial decode
static const uint64_t GZ_NONE = ~0ull;

// device scalars
enum { GS_NU = 0, GS_NC, GS_TOTAL, GS_MEMBERS, GS_ERR, GS_CONF, GS_N };

__global__ void __launch_bounds__(256) k_gz_find(const uint8_t *gz, uint64_t n, uint64_t chunk, uint64_t *guess)
{
	__shared__ unsigned long long found;
	const uint64_t i = blockIdx.x + 1, b0 = i * chunk * 8, b1 = (i + 1) * chunk < n ? (i + 1) * chunk * 8 : n * 8;
	if (threadIdx.x == 0) found = GZ_NONE;
	__syncthreads();
	InfTables t;
	for (uint64_t base = b0; base < b1; base += blockDim.x) {
		const uint64_t b = base + threadIdx.x;
		if (b < b1 && inf_guess_test(gz, n, b, t, GZ_TRIAL)) atomicMin(&found, (unsigned long long)b);
		__syncthreads();
		if (found != GZ_NONE) break;
	}
	if (threadIdx.x == 0) guess[i] = found;
}

__global__ void k_gz_compact(const uint64_t *guess, uint64_t n_chunks, uint64_t *starts, unsigned long long *sc)
{
	uint64_t k = 0;
	starts[k++] = 0;
	for (uint64_t i = 1; i < n_chunks; ++i) if (guess[i] != GZ_NONE) starts[k++] = guess[i];
	sc[GS_NU] = k;
}

__global__ void __launch_bounds__(32) k_gz_decode(const uint8_t *gz, uint64_t n, const uint64_t *starts, uint32_t nu, uint16_t *ring,
                                                  int *st, uint32_t *land, uint64_t *olen, int64_t *mat, uint32_t *nmem)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= nu) return;
	InfTables t;
	InfOutMark o;
	o.begin(ring + (size_t)u * INF_WIN);
	uint32_t j = u + 1;
	st[u] = inf_run(gz, n, starts[u], u == 0, starts, nu, &j, t, o);
	land[u] = j, olen[u] = o.p, mat[u] = o.member_at, nmem[u] = o.n_members;
}

__global__ void k_gz_chain(const int *st, const uint32_t *land, const uint64_t *olen, const uint32_t *nmem, uint32_t nu,
                           uint32_t *chain, uint64_t *off, uint32_t *mbase, unsigned long long *sc)
{
	uint64_t total = 0, members = 0, c = 0;
	for (uint32_t u = 0;; ++c) {
		if (st[u] < 0) { sc[GS_ERR] = 1; return; }
		chain[c] = u, off[c] = total, mbase[c] = (uint32_t)members;
		total += olen[u], members += nmem[u];
		if (st[u] == INF_END) break;
		u = land[u]; // > u: the chain always moves on
	}
	sc[GS_NC] = c + 1, sc[GS_TOTAL] = total, sc[GS_MEMBERS] = members, sc[GS_CONF] = c;
}

__global__ void __launch_bounds__(1024) k_gz_window(const uint32_t *chain, uint32_t nc, const uint16_t *ring, const uint64_t *olen,
                                                    const int64_t *mat, uint8_t *win, uint32_t *valid)
{
	for (uint32_t c = 0; c < nc; ++c) {
		const uint32_t u = chain[c];
		const uint8_t *wi = win + (size_t)c * INF_WIN;
		uint8_t *wo = win + (size_t)(c + 1) * INF_WIN;
		for (uint32_t k = threadIdx.x; k < INF_WIN; k += blockDim.x) wo[k] = inf_window_byte(ring + (size_t)u * INF_WIN, olen[u], wi, k);
		if (threadIdx.x == 0) valid[c + 1] = inf_window_valid(valid[c], olen[u], mat[u]);
		__syncthreads();
	}
}

__global__ void __launch_bounds__(32) k_gz_resolve(const uint8_t *gz, uint64_t n, const uint64_t *starts, uint32_t nu, const uint32_t *chain,
                                                   uint32_t nc, const uint64_t *off, const uint32_t *mbase, const int *st, const uint32_t *land,
                                                   const uint64_t *olen, const uint32_t *nmem, const uint8_t *win, const uint32_t *valid,
                                                   uint8_t *out, uint64_t *m_end, uint32_t *m_crc, uint32_t *m_isize, unsigned long long *sc)
{
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= nc) return;
	const uint32_t u = chain[c];
	InfTables t;
	InfOutByte o;
	o.out = out + off[c], o.win = win + (size_t)c * INF_WIN, o.p = 0, o.cap = olen[u], o.lim = -(int64_t)valid[c];
	o.m_end = m_end + mbase[c], o.m_crc = m_crc + mbase[c], o.m_isize = m_isize + mbase[c], o.n_members = 0, o.m_cap = nmem[u];
	uint32_t j = u + 1;
	const int r = inf_run(gz, n, starts[u], u == 0, starts, nu, &j, t, o);
	if (r != st[u] || o.p != olen[u] || o.n_members != nmem[u] || (r == INF_LAND && j != land[u])) { sc[GS_ERR] = 1; return; }
	for (uint32_t k = 0; k < o.n_members; ++k) o.m_end[k] += off[c];
}

__global__ void k_gz_crc_seg(const uint8_t *txt, uint64_t total, uint64_t seg, uint32_t *sc)
{
	__shared__ uint32_t tab[256];
	if (threadIdx.x < 256) {
		uint32_t c = threadIdx.x;
		for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (c & 1 ? INF_CRC_POLY : 0);
		tab[threadIdx.x] = c;
	}
	__syncthreads();
	const uint64_t n_seg = (total + seg - 1) / seg;
	for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_seg; s += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t a = s * seg, l = total - a < seg ? total - a : seg;
		const uint32_t *w = (const uint32_t*)(txt + a);
		uint32_t c = 0;
		uint64_t i = 0;
		if (((uintptr_t)txt & 3) == 0) for (; i + 4 <= l; i += 4) { // segments start at multiples of 16 KiB
			const uint32_t v = w[i >> 2];
			c = tab[(c ^ v) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 8)) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 16)) & 255] ^ (c >> 8);
			c = tab[(c ^ (v >> 24)) & 255] ^ (c >> 8);
		}
		for (; i < l; ++i) c = tab[(c ^ txt[a + i]) & 255] ^ (c >> 8);
		sc[s] = c;
	}
}

// one block per member [a, b): its head piece up to the first segment boundary, the whole segments, its tail piece; each
// thread joins a contiguous run of them, then the block joins the runs in order
__global__ void __launch_bounds__(128) k_gz_crc_member(const uint8_t *txt, uint64_t seg, const uint32_t *seg_crc, const uint64_t *m_end,
                                                       const uint32_t *m_crc, const uint32_t *m_isize, unsigned long long *sc)
{
	__shared__ uint32_t tab[256], x2k[64], r_crc[128];
	__shared__ uint64_t r_len[128];
	const uint32_t m = blockIdx.x, tid = threadIdx.x;
	for (uint32_t e = tid; e < 256; e += blockDim.x) {
		uint32_t c = e;
		for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (c & 1 ? INF_CRC_POLY : 0);
		tab[e] = c;
	}
	if (tid == 0) inf_x2k_table(x2k);
	__syncthreads();
	const uint64_t a = m ? m_end[m - 1] : 0, b = m_end[m];
	uint64_t A = (a + seg - 1) / seg * seg, B = b / seg * seg;
	if (A > b) A = b;
	if (B < A) B = A;
	const uint64_t n_full = (B - A) / seg, n_items = n_full + 2; // head, full segments, tail
	const uint64_t per = (n_items + blockDim.x - 1) / blockDim.x;
	const uint32_t xs = inf_x8n(x2k, seg);
	uint32_t raw = 0;
	uint64_t len = 0;
	for (uint64_t it = tid * per; it < n_items && it < (tid + 1) * per; ++it) {
		if (it == 0) raw = inf_crc_raw(tab, 0, txt + a, A - a), len = A - a;
		else if (it <= n_full) raw = inf_gf2_mul(raw, xs) ^ seg_crc[A / seg + it - 1], len += seg;
		else raw = inf_crc_join(x2k, raw, inf_crc_raw(tab, 0, txt + B, b - B), b - B), len += b - B;
	}
	r_crc[tid] = raw, r_len[tid] = len;
	__syncthreads();
	for (uint32_t s = 1; s < blockDim.x; s <<= 1) {
		if (tid % (2 * s) == 0 && tid + s < blockDim.x) {
			r_crc[tid] = inf_crc_join(x2k, r_crc[tid], r_crc[tid + s], r_len[tid + s]);
			r_len[tid] += r_len[tid + s];
		}
		__syncthreads();
	}
	if (tid == 0 && (inf_crc_final(x2k, r_crc[0], b - a) != m_crc[m] || (uint32_t)(b - a) != m_isize[m])) sc[GS_ERR] = 1;
}

namespace {
struct Scratch { // every allocation of one inflate, freed together; tracks the peak
	GzMem &mem;
	std::vector<std::pair<void*, size_t>> live;
	size_t now = 0, peak = 0;
	explicit Scratch(GzMem &m) : mem(m) {}
	template <typename T> T *get(size_t n)
	{
		const size_t bytes = (n ? n : 1) * sizeof(T);
		void *p = mem.alloc(bytes);
		live.push_back({p, bytes});
		now += bytes, peak = now > peak ? now : peak;
		return (T*)p;
	}
	void put(void *p)
	{
		for (size_t i = 0; i < live.size(); ++i) if (live[i].first == p) { now -= live[i].second; live.erase(live.begin() + i); break; }
		mem.free(p);
	}
	~Scratch() { for (auto &e : live) mem.free(e.first); }
};
}

int gz_inflate_dev(cudaStream_t st, GzMem &mem, const uint8_t *gz, size_t len, char *(*out)(void *ctx, size_t n), void *ctx,
                   size_t *out_len, GzStats *stats, size_t chunk)
{
	*out_len = 0;
	if (len < 18) return GZ_REJECT; // shorter than a header and a trailer
	if (!chunk) chunk = GZ_CHUNK;
	Scratch s(mem);
	cudaEvent_t ev[7];
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventCreate(&ev[i]));
	unsigned long long *d_sc = s.get<unsigned long long>(GS_N), h_sc[GS_N];
	GZ_CUDA(cudaMemsetAsync(d_sc, 0, GS_N * sizeof(unsigned long long), st));
	auto fetch = [&]() {
		GZ_CUDA(cudaMemcpyAsync(h_sc, d_sc, sizeof(h_sc), cudaMemcpyDeviceToHost, st));
		GZ_CUDA(cudaStreamSynchronize(st));
	};
	int rc = GZ_REJECT;
	const uint64_t n_chunks = (len + chunk - 1) / chunk;
	GZ_CUDA(cudaEventRecord(ev[0], st));
	// find + compact
	uint64_t *guess = s.get<uint64_t>(n_chunks), *starts = s.get<uint64_t>(n_chunks);
	if (n_chunks > 1) { k_gz_find<<<(unsigned)(n_chunks - 1), 256, 0, st>>>(gz, len, chunk, guess); GZ_CUDA(cudaGetLastError()); }
	k_gz_compact<<<1, 1, 0, st>>>(guess, n_chunks, starts, d_sc);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[1], st));
	fetch();
	const uint32_t nu = (uint32_t)h_sc[GS_NU];
	s.put(guess);
	// pass 1
	uint16_t *ring = s.get<uint16_t>((size_t)nu * INF_WIN);
	int *ust = s.get<int>(nu);
	uint32_t *land = s.get<uint32_t>(nu), *nmem = s.get<uint32_t>(nu);
	uint64_t *olen = s.get<uint64_t>(nu);
	int64_t *mat = s.get<int64_t>(nu);
	k_gz_decode<<<(nu + 31) / 32, 32, 0, st>>>(gz, len, starts, nu, ring, ust, land, olen, mat, nmem);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[2], st));
	// chain
	uint32_t *chain = s.get<uint32_t>(nu), *mbase = s.get<uint32_t>(nu);
	uint64_t *off = s.get<uint64_t>(nu);
	k_gz_chain<<<1, 1, 0, st>>>(ust, land, olen, nmem, nu, chain, off, mbase, d_sc);
	GZ_CUDA(cudaGetLastError());
	GZ_CUDA(cudaEventRecord(ev[3], st));
	fetch();
	const uint32_t nc = (uint32_t)h_sc[GS_NC];
	const uint64_t total = h_sc[GS_TOTAL], members = h_sc[GS_MEMBERS];
	float ms[6] = { 0, 0, 0, 0, 0, 0 };
	if (!h_sc[GS_ERR]) {
		// window
		uint8_t *win = s.get<uint8_t>((size_t)(nc + 1) * INF_WIN);
		uint32_t *valid = s.get<uint32_t>(nc + 1);
		GZ_CUDA(cudaMemsetAsync(win, 0, INF_WIN, st));
		GZ_CUDA(cudaMemsetAsync(valid, 0, sizeof(uint32_t), st));
		k_gz_window<<<1, 1024, 0, st>>>(chain, nc, ring, olen, mat, win, valid);
		GZ_CUDA(cudaGetLastError());
		GZ_CUDA(cudaEventRecord(ev[4], st));
		// resolve
		char *dst = out(ctx, total);
		uint64_t *m_end = s.get<uint64_t>(members);
		uint32_t *m_crc = s.get<uint32_t>(members), *m_isize = s.get<uint32_t>(members);
		k_gz_resolve<<<(nc + 31) / 32, 32, 0, st>>>(gz, len, starts, nu, chain, nc, off, mbase, ust, land, olen, nmem, win, valid,
		                                            (uint8_t*)dst, m_end, m_crc, m_isize, d_sc);
		GZ_CUDA(cudaGetLastError());
		GZ_CUDA(cudaEventRecord(ev[5], st));
		// crc
		const uint64_t n_seg = (total + GZ_SEG - 1) / GZ_SEG;
		uint32_t *seg_crc = s.get<uint32_t>(n_seg);
		if (n_seg) { k_gz_crc_seg<<<(unsigned)((n_seg + 255) / 256), 256, 0, st>>>((const uint8_t*)dst, total, GZ_SEG, seg_crc); GZ_CUDA(cudaGetLastError()); }
		if (members) { k_gz_crc_member<<<(unsigned)members, 128, 0, st>>>((const uint8_t*)dst, GZ_SEG, seg_crc, m_end, m_crc, m_isize, d_sc); GZ_CUDA(cudaGetLastError()); }
		GZ_CUDA(cudaEventRecord(ev[6], st));
		fetch();
		if (!h_sc[GS_ERR]) rc = GZ_OK, *out_len = total;
		for (int i = 0; i < 6; ++i) GZ_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
	}
	if (stats) {
		stats->ms_find = ms[0], stats->ms_decode = ms[1], stats->ms_chain = ms[2], stats->ms_window = ms[3], stats->ms_resolve = ms[4], stats->ms_crc = ms[5];
		stats->n_chunks = n_chunks, stats->n_units = nu, stats->n_chain = nc, stats->n_confirmed = h_sc[GS_CONF];
		stats->n_members = members, stats->out_len = rc == GZ_OK ? total : 0, stats->scratch_peak = s.peak;
	}
	for (int i = 0; i < 7; ++i) GZ_CUDA(cudaEventDestroy(ev[i]));
	return rc;
}
