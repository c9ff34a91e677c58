// abb_graph.cuh -- neighbourhoods of de Bruijn graph vertices for the two GraphViz dumps: the out-edge chains of `abyss-bloom-dbg -g`
// (outputGraph, BloomDBG/bloom-dbg.h:1171-1242) and the in- and out-edges of `abyss-bloom graph` (Bloom/bloom.cc:984-1153).
// Shared by the CUDA kernels k_successors (abb_insert.cuh) and k_graph_neighbors (below) and the CPU test harnesses
// (tests/host_graph, tests/host_bloom_graph).
#pragma once
#include "../../include/abyss_b200.h"
#include "abb_device.cuh"
#include <type_traits>

namespace abb {

/** the part of a k-mer's ntHash that positions first, first + stride, ... contribute.  The hash is XOR-linear in the positions
 *  (abb_device.cuh): forward XOR_t R^{k-1-t}(seed(c_t)), reverse complement XOR_t R^t(seed(comp c_t)), so the XOR of the parts
 *  over first = 0..stride-1 is NTC64 (nthash.hpp:268-272); stride 1 computes it whole. */
ABB_HD HashPair kmer_hash_part(const uint8_t* km, unsigned k, unsigned first, unsigned stride)
{
	HashPair h = { 0, 0 };
	for (unsigned t = first; t < k; t += stride) {
		const unsigned c = base_code(km[t]) & 3u;
		h.fh ^= srol_n(seed_of(c), k - 1 - t);
		h.rh ^= srol_n(seed_of(3 - c), t);
	}
	return h;
}

/** canonical hash of neighbour j of the k-mer u with hash state h (first / last = codes of u's first and last base): j < 4 the
 *  successor u[1:] + "ACGT"[j] (out_edge_iterator, BloomDBG/RollingBloomDBG.h:300-360), j >= 4 the predecessor "ACGT"[j - 4] +
 *  u[:-1] (in_edge_iterator, :365-427).  Vertex identity: RollingBloomDBGVertex compares canonical k-mers. */
ABB_HD uint64_t neighbor_hash(const HashPair& h, const RollTab& rt, unsigned first, unsigned last, unsigned j)
{
	return (j < 4 ? roll_right(h, rt, first, j) : roll_left(h, rt, last, j - 4)).canonical();
}

/** one byte of a filter, read past L1 on the device (the graph queries touch each line about once) */
ABB_HD unsigned ld_filter(const uint8_t* p)
{
#if defined(__CUDA_ARCH__)
	return __ldcg(p);
#else
	return *p;
#endif
}
/** bit `pos` of a bit array (BloomFilter::contains, vendor/btl_bloomfilter/BloomFilter.hpp:249-259, one hash) */
ABB_HD bool bit_at(const uint8_t* bits, uint64_t pos) { return (ld_filter(bits + (pos >> 3)) >> (pos & 7)) & 1; }

/** RollingBloomDBG::out_edge_iterator (BloomDBG/RollingBloomDBG.h:300-360): shift the k-mer left, try A, C, G, T as the last base,
 *  keep those the filter contains (`probe(canonical hash)`).  While a vertex has exactly one out-edge the walk moves on to that
 *  successor, up to max_chain (<= 128) vertices: unbranched paths -- nearly all of a genome's graph -- cost one query per
 *  max_chain vertices instead of one per vertex.  out[s] = out-edges of the s-th vertex of the chain (s = 0: the k-mer itself):
 *  mask bit b = the successor with base b exists, hash[b] = its canonical hash (vertex identity: RollingBloomDBGVertex compares
 *  canonical k-mers).  *self = canonical hash of the start k-mer.  Returns the number of vertices expanded. */
template <typename Probe>
ABB_HD unsigned successors_chain(const uint8_t* km, unsigned k, unsigned max_chain, const Probe& probe, abb_succ_info* out, uint64_t* self)
{
	const RollTab rt = make_rolltab(k);
	HashPair h = kmer_hash_part(km, k, 0, 1);
	*self = h.canonical();
	unsigned appended[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }; // bases appended so far, 2 bits each
	unsigned s = 0;
	while (s < max_chain) {
		// the base that leaves on this shift: from the start k-mer while it lasts, then from the appended bases
		const unsigned first = s < k ? base_code(km[s]) & 3u : (appended[(s - k) >> 4] >> (2 * ((s - k) & 15))) & 3u;
		unsigned mask = 0;
		for (unsigned b = 0; b < 4; ++b) {
			const uint64_t h0 = neighbor_hash(h, rt, first, 0, b);
			out[s].hash[b] = h0;
			if (probe(h0))
				mask |= 1u << b;
		}
		out[s].mask = (uint8_t)mask;
		++s;
		if ((mask & (mask - 1)) != 0 || mask == 0 || s == max_chain)
			break;
		unsigned nb = 0;
		while (!((mask >> nb) & 1))
			++nb;
		h = roll_right(h, rt, first, nb);
		appended[(s - 1) >> 4] |= nb << (2 * ((s - 1) & 15));
	}
	return s;
}

// ---- abyss-bloom graph: in- and out-edges and attribute filters, one warp per vertex ---------------------------------------------

constexpr unsigned kMaxAttrFilters = 32;
/** most probes one lane makes: ceil(32 / 4) graph hashes of its neighbour plus the 32 hashes of an attribute filter */
constexpr unsigned kMaxLaneProbes = kMaxHashes / 4 + kMaxHashes;

/** the filters of one abb_graph_neighbors call.  The graph is the last level of a bit or cascading filter; an attribute filter (-A)
 *  is a bit filter tested, as the reference's RollingBloomDBGVisitor::discover_vertex does, with the first H_a of the graph's hash
 *  values modulo its own size (its H_a <= the graph's H). */
struct NbrQuery {
	HashCfg cfg;         // the graph's: H, k, size, hash multipliers
	RollTab rt;          // the graph's k (no spaced seed); a kernel parameter, so rt.rk[base] is a constant-bank load
	const uint8_t* bits; // the graph's last level
	unsigned n_attr;
	struct Attr {
		const uint8_t* bits;
		FastMod mod;
		unsigned H;
	} attr[kMaxAttrFilters];
};

/** probes per lane of a query: ceil(H / 4) graph hashes, plus the most hashes of an attribute filter; <= kMaxLaneProbes */
inline unsigned nbr_lane_probes(const NbrQuery& q)
{
	unsigned ha = 0;
	for (unsigned a = 0; a < q.n_attr; ++a)
		ha = q.attr[a].H > ha ? q.attr[a].H : ha;
	return (q.cfg.H + 3) / 4 + ha;
}

/** f(std::integral_constant<unsigned, P>()) for the smallest probe bound P the kernel is built for (1, 2, 4, 8, 16,
 *  kMaxLaneProbes) that holds `probes` */
template <typename F>
inline void with_lane_probes(unsigned probes, F&& f)
{
	if (probes <= 1)
		f(std::integral_constant<unsigned, 1>());
	else if (probes <= 2)
		f(std::integral_constant<unsigned, 2>());
	else if (probes <= 4)
		f(std::integral_constant<unsigned, 4>());
	else if (probes <= 8)
		f(std::integral_constant<unsigned, 8>());
	else if (probes <= 16)
		f(std::integral_constant<unsigned, 16>());
	else
		f(std::integral_constant<unsigned, kMaxLaneProbes>());
}

/** One lane's share of the probes of a vertex with hash state h: graph(K) out_edges + in_edges + vertex_exists
 *  (RollingBloomDBG.h:302-445) and the -A tests.  Lane = 4 * neighbour + hash slot, as in the assembler's WarpCtx: lane l tests
 *  hashes l & 3, (l & 3) + 4, ... of neighbour l >> 2 (neighbour_hash order) in the graph; lane a < n_attr also tests the vertex
 *  itself in attribute filter a.  P >= nbr_lane_probes(q) bounds the lane's probes: the first loop computes every position and
 *  issues every load, the second reads the bytes, so a lane waits for one memory round trip whatever H and the attribute filters
 *  are.  Returns the neighbour's canonical hash; *graph_ok / *attr_ok = the lane's tests all passed. */
template <unsigned P>
ABB_HD uint64_t nbr_lane(const NbrQuery& q, const HashPair& h, unsigned first, unsigned last, unsigned lane, bool* graph_ok,
                         bool* attr_ok)
{
	const uint64_t hn = neighbor_hash(h, q.rt, first, last, lane >> 2), hs = h.canonical();
	const unsigned slot = lane & 3;
	const unsigned ng = slot < q.cfg.H ? (q.cfg.H - slot + 3) / 4 : 0; // graph probes of this lane
	const bool attr = lane < q.n_attr;
	const unsigned na = attr ? q.attr[lane].H : 0;
	unsigned byte[P], bit[P];
#pragma unroll
	for (unsigned j = 0; j < P; ++j) {
		byte[j] = 1;
		bit[j] = 0;
		if (j < ng) {
			const uint64_t p = nth_pos(hn, q.cfg, slot + 4 * j);
			byte[j] = ld_filter(q.bits + (p >> 3));
			bit[j] = p & 7;
		} else if (j < ng + na) {
			const NbrQuery::Attr& f = q.attr[lane];
			const uint64_t p = fastmod_u64(nth_hash(hs, q.cfg, j - ng), f.mod);
			byte[j] = ld_filter(f.bits + (p >> 3));
			bit[j] = p & 7;
		}
	}
	bool g = true, a = attr;
#pragma unroll
	for (unsigned j = 0; j < P; ++j) {
		const bool b = (byte[j] >> bit[j]) & 1;
		if (j < ng)
			g &= b;
		else
			a &= b; // past ng + na: byte 1, bit 0
	}
	*graph_ok = g;
	*attr_ok = a;
	return hn;
}

/** the 8-bit neighbour mask from the 32 lanes' graph_ok bits (bit l = lane l): neighbour j exists when lanes 4j..4j+3 all pass */
ABB_HD unsigned nbr_mask(unsigned lanes)
{
	lanes &= lanes >> 1;
	lanes &= lanes >> 2; // bit 4j = AND of the four lanes of neighbour j
	unsigned m = 0;
	for (unsigned j = 0; j < 8; ++j)
		m |= ((lanes >> (4 * j)) & 1u) << j;
	return m;
}

#if defined(__CUDACC__)
/** abb_graph_neighbors: one warp per k-mer, grid-stride.  The lanes hash the k-mer together (positions lane, lane + 32, ...,
 *  XOR-reduced), probe as nbr_lane says, and the ballots give the neighbour mask and the attribute bits.  P: nbr_lane's bound,
 *  chosen by the caller from nbr_lane_probes. */
template <unsigned P>
__global__ void __launch_bounds__(256)
k_graph_neighbors(const uint8_t* __restrict__ kmers, uint64_t n, const __grid_constant__ NbrQuery q, abb_nbr_info* __restrict__ out)
{
	const unsigned lane = threadIdx.x & 31, k = q.cfg.k;
	const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
	for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n; w += warps) {
		const uint8_t* km = kmers + w * k;
		HashPair h = kmer_hash_part(km, k, lane, 32);
		for (unsigned d = 16; d >= 1; d >>= 1) {
			h.fh ^= __shfl_xor_sync(0xffffffffu, h.fh, d);
			h.rh ^= __shfl_xor_sync(0xffffffffu, h.rh, d);
		}
		bool g, a;
		const uint64_t hn = nbr_lane<P>(q, h, base_code(km[0]) & 3u, base_code(km[k - 1]) & 3u, lane, &g, &a);
		const unsigned gl = __ballot_sync(0xffffffffu, g), al = __ballot_sync(0xffffffffu, a);
		abb_nbr_info& o = out[w];
		if ((lane & 3) == 0)
			o.hash[lane >> 2] = hn;
		if (lane == 0) {
			o.self = h.canonical();
			o.attr = al;
			o.mask = (uint8_t)nbr_mask(gl);
		}
	}
}
#endif

} // namespace abb
