// tests/host_walk/host_walk.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// Single-thread emulation harness for the pass-2 graph logic: instantiates the SAME templates
// the CUDA kernels use (abyss_b200/csrc/abb_walk.cuh) over a trivial one-lane context, drives
// them sequentially exactly like BloomDBG::assemble at -j1 (bloom-dbg.h:783-882,972-1089), and
// prints the unitig FASTA.  It lets the traversal logic be debugged against the reference's
// golden FASTA on a machine without a GPU.  The counting filter is built with the C oracle.
//
//   host_walk K KC H COUNTERS TRIM reads.fq [readlog.tsv] > out.fa
//   host_walk markerset                 checks marker_set_insert on sets it fills up
//
// HOST_WALK_TILES=1 splices tiles as the kernels do; HOST_WALK_DROP_TILES=SEED then leaves out a seeded subset of the tiles,
// as a full tile store does on the GPU: one of the four tiles of some markers, all four of others.
#include "../../abyss_b200/csrc/abb_walk.cuh"
extern "C" {
#include "../../oracle/abyss_oracle.h"
}
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

using namespace abb;

struct HostCtx {
	unsigned k, trim, H, threshold;
	RollTab rt;
	const char* mask = nullptr; // spaced seed (HOST_WALK_MASK)
	HashCfg cfg;
	const uint8_t* counters;
	Frame* frames;
	uint64_t* look;
	std::vector<std::unique_ptr<uint8_t[]>> allocs;
	bool fail_ = false;
	unsigned long long probes = 0;

	bool contains(uint64_t h0) const
	{
		for (unsigned i = 0; i < H; ++i)
			if (counters[nth_pos(h0, cfg, i)] < threshold)
				return false;
		return true;
	}
	template <int KW>
	unsigned neighbors(const Vtx<KW>& v)
	{
		++probes;
		unsigned m = 0;
		for (unsigned n = 0; n < 8; ++n) {
			if (contains(neighbor_bloom(v, k, rt, n < 4 ? FWD : REV, n & 3)))
				m |= 1u << n;
		}
		return m;
	}
	template <int KW>
	unsigned neighbors_dir(const Vtx<KW>& v, Dir d)
	{
		const unsigned m = neighbors(v);
		return d == FWD ? (m & 15) : (m >> 4);
	}
	struct Probe {
		unsigned mask;
	};
	template <int KW>
	Probe neighbors_issue(const Vtx<KW>& v) { return Probe{ neighbors(v) }; }
	unsigned neighbors_finish(const Probe& p) { return p.mask; }
	// tiles
	std::vector<TileRec> tile_recs;
	std::vector<std::unique_ptr<uint8_t[]>> tile_mem;
	std::unordered_map<uint64_t, uint32_t> tile_map; // (key mixed with class) -> index, verified on lookup
	bool use_tiles = false;
	unsigned long long tile_splices = 0;
	static uint64_t tkey(uint64_t key, unsigned cls) { return key * 4 + cls; } // exact for the emulation: 64-bit wrap is fine with verification
	bool tiles_enabled() const { return use_tiles; }
	const TileRec* tile_lookup(uint64_t key, unsigned cls)
	{
		auto range = tile_multi.equal_range(tkey(key, cls));
		for (auto it = range.first; it != range.second; ++it)
			if (tile_recs[it->second].key == key && tile_recs[it->second].cls == cls) {
				++tile_splices;
				return &tile_recs[it->second];
			}
		return nullptr;
	}
	std::unordered_multimap<uint64_t, uint32_t> tile_multi;
	uint32_t tile_index(const TileRec* t) const { return (uint32_t)(t - tile_recs.data()); }
	const TileRec* tile_at(uint32_t idx) const { return &tile_recs[idx]; }
	void prefetch(const void*) const {}
	void wr32(uint32_t* p, uint32_t v) { *p = v; }
	uint64_t rd64(const uint64_t* p) { return *p; }
	void wr64(uint64_t* p, uint64_t v) { *p = v; }
	uint8_t rd8(const uint8_t* p) { return *p; }
	void wr8(uint8_t* p, uint8_t v) { *p = v; }
	void sync() {}
	bool find64(const uint64_t* a, unsigned n, uint64_t key, unsigned stride)
	{
		for (unsigned i = 0; i < n; ++i)
			if (a[(size_t)i * stride] == key)
				return true;
		return false;
	}
	uint8_t* alloc(uint64_t bytes, bool zero)
	{
		allocs.emplace_back(new uint8_t[bytes + 8]);
		if (zero)
			memset(allocs.back().get(), 0, bytes);
		return allocs.back().get();
	}
	bool tile_cycle = false;
	void fail(unsigned why)
	{
		fail_ = true;
		if (why == abb::WALK_FAIL_TILE_CYCLE)
			tile_cycle = true;
		else
			fprintf(stderr, "host_walk: scratch overflow %u\n", why);
	}
	bool failed() const { return fail_; }
	void copy8(uint8_t* d, const uint8_t* s, unsigned n) { if (n) memcpy(d, s, n); }
	void copy8_rev(uint8_t* d, const uint8_t* s, unsigned n) { for (unsigned i = 0; i < n; ++i) d[i] = s[n - 1 - i]; }
	void rehash(const uint64_t* o, unsigned ocap, uint64_t* n, unsigned ncap)
	{
		for (unsigned s = 0; s < ocap; ++s)
			if (o[s]) {
				uint64_t t = pathset_slot(o[s], ncap);
				while (n[t])
					t = (t + 1) & (ncap - 1);
				n[t] = o[s];
			}
	}
	void mark_covered(const PathSet& ps, const uint64_t* rh, uint8_t* cov, unsigned nk, const ContigOut& o, const uint8_t* = nullptr, unsigned = 0)
	{
		std::unordered_set<uint64_t> tilev;
		for (int side = 0; side < 2; ++side) {
			const U32Vec& tv = side ? o.tiles_right : o.tiles_left;
			for (unsigned ti = 0; ti < tv.n; ++ti) {
				const TileRec& T = tile_recs[tv.p[ti]];
				tilev.insert(T.hashes, T.hashes + T.n);
			}
		}
		for (unsigned j = 0; j < nk; ++j) {
			if (cov[j] || !(pathset_contains(*this, ps, rh[j]) || tilev.count(rh[j])))
				continue;
			if (o.popped_front && rh[j] == o.front_h)
				continue;
			if (o.popped_back && rh[j] == o.back_h)
				continue;
			cov[j] = 1;
		}
	}
};

struct Assembly {
	HostCtx* c;
	std::vector<uint8_t> assembled; // bit filter, size() bits = #counters (bloom-dbg.h:910-911)
	uint64_t mbits;
	std::unordered_set<uint64_t> contigEnd;
	size_t contigID = 0;
	const std::string* readID = nullptr;

	bool inAssembled(uint64_t h0) const
	{
		for (unsigned i = 0; i < c->H; ++i) {
			uint64_t p = nth_pos(h0, c->cfg, i);
			if (!(assembled[p >> 3] & (1u << (p & 7))))
				return false;
		}
		return true;
	}
	void addAssembled(uint64_t h0)
	{
		for (unsigned i = 0; i < c->H; ++i) {
			uint64_t p = nth_pos(h0, c->cfg, i);
			assembled[p >> 3] |= (uint8_t)(1u << (p & 7));
		}
	}
	unsigned minCount(uint64_t h0) const
	{
		unsigned mn = 255;
		for (unsigned i = 0; i < c->H; ++i) {
			unsigned v = c->counters[nth_pos(h0, c->cfg, i)];
			if (v < mn)
				mn = v;
		}
		return mn;
	}
	struct Collected {
		std::string seq;
		bool pushed_front, pushed_back, popped_front, popped_back;
		uint64_t front_h, back_h;
	};
	std::vector<Collected> collected;
	void operator()(HostCtx&, unsigned, const ContigOut& o)
	{
		Collected x;
		if (getenv("HOST_WALK_DEBUG"))
			fprintf(stderr, "contig: len %u psize %u left %u right %u tip %d\n", o.len, o.psize, (unsigned)o.left, (unsigned)o.right, (int)o.tip);
		x.seq.assign(o.len, 'N');
		for (unsigned i = 0; i < o.len; ++i)
			if (column_written(c->rt, c->k, o.len - c->k + 1, i))
				x.seq[i] = "ACGT"[o.seq[i]];
		x.pushed_front = o.pushed_front; x.pushed_back = o.pushed_back;
		x.popped_front = o.popped_front; x.popped_back = o.popped_back;
		x.front_h = o.front_h; x.back_h = o.back_h;
		collected.push_back(x);
	}
	std::vector<uint64_t> hashes_of(const std::string& seq) const
	{
		const unsigned k = c->k;
		std::vector<uint64_t> tmp((seq.size() - k + 1) * c->H), hs(seq.size() - k + 1);
		size_t n = abo_hash_seq(seq.data(), seq.size(), k, c->H, c->mask, tmp.data(), NULL);
		if (n != hs.size()) { fprintf(stderr, "host_walk: contig hashing mismatch\n"); exit(3); }
		for (size_t i = 0; i < n; ++i)
			hs[i] = tmp[i * c->H];
		return hs;
	}
	/** a vertex occurs twice in the (untrimmed) path: the tile splice skipped an ER_CYCLE */
	bool has_repeat(const Collected& x) const
	{
		std::vector<uint64_t> hs = hashes_of(x.seq);
		std::unordered_set<uint64_t> seen;
		size_t b = x.pushed_front ? 1 : 0, e = hs.size() - (x.pushed_back ? 1 : 0);
		for (size_t i = b; i < e; ++i)
			if (!seen.insert(hs[i]).second)
				return true;
		if (x.popped_front && !seen.insert(x.front_h).second)
			return true;
		if (x.popped_back && !seen.insert(x.back_h).second)
			return true;
		return false;
	}
	/** identity of outputContig's end vertices v1/v2 (bloom-dbg.h:556-564): the k-mer string is canonicalized as a
	 *  string ('N' columns included), and operator== then compares the '1' positions */
	uint64_t end_identity(const std::string& kmer, uint64_t h0) const
	{
		if (!c->mask)
			return h0;
		const unsigned k = c->k;
		std::string rc(kmer.rbegin(), kmer.rend());
		for (auto& ch : rc)
			ch = ch == 'A' ? 'T' : ch == 'C' ? 'G' : ch == 'G' ? 'C' : ch == 'T' ? 'A' : ch;
		const std::string& cs = rc < kmer ? rc : kmer;
		uint64_t f = 0;
		for (unsigned i = 0; i < k; ++i)
			if (c->mask[i] == '1')
				f ^= srol_n(seed_of(base_code((uint8_t)cs[i])), k - 1 - i);
		return f;
	}
	// outputContig (bloom-dbg.h:538-620)
	void output(const Collected& x)
	{
		const unsigned k = c->k;
		const std::string& seq = x.seq;
		struct { unsigned len; } o = { (unsigned)seq.size() };
		std::vector<uint64_t> hs(o.len - k + 1);
		std::vector<uint64_t> tmp(hs.size() * c->H);
		size_t n = abo_hash_seq(seq.data(), seq.size(), k, c->H, c->mask, tmp.data(), NULL);
		if (n != hs.size()) { fprintf(stderr, "host_walk: contig hashing mismatch\n"); exit(3); }
		for (size_t i = 0; i < n; ++i)
			hs[i] = tmp[i * c->H];
		bool redundant = false;
		if (o.len < k + kFpTrim - 1) {
			const uint64_t e1 = end_identity(seq.substr(0, k), hs.front()), e2 = end_identity(seq.substr(seq.size() - k), hs.back());
			if (contigEnd.count(e1) && contigEnd.count(e2))
				redundant = true;
			else {
				contigEnd.insert(e1);
				contigEnd.insert(e2);
			}
		} else {
			redundant = true;
			for (uint64_t h : hs)
				if (!inAssembled(h)) {
					redundant = false;
					break;
				}
		}
		if (redundant)
			return;
		for (uint64_t h : hs)
			addAssembled(h);
		unsigned cov = 0;
		for (uint64_t h : hs)
			cov += minCount(h);
		printf(">%zu %u %u read:%s\n%s\n", contigID, o.len, cov, readID->c_str(), seq.c_str());
		++contigID;
	}
};

static uint64_t splitmix64(uint64_t x)
{
	x += 0x9E3779B97F4A7C15ULL;
	x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
	x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
	return x ^ (x >> 31);
}

template <int KW>
static int run(unsigned k, unsigned kc, unsigned H, uint64_t m, unsigned trim, const char* path, const char* logpath)
{
	std::vector<std::string> ids, seqs;
	{
		std::ifstream in(path);
		std::string l1, l2, l3, l4;
		while (std::getline(in, l1) && std::getline(in, l2)) {
			if (l1[0] == '@') {
				std::getline(in, l3);
				std::getline(in, l4);
			}
			std::string id = l1.substr(1, l1.find_first_of(" \t") == std::string::npos ? std::string::npos : l1.find_first_of(" \t") - 1);
			ids.push_back(id);
			for (auto& ch : l2)
				ch = (char)toupper(ch);
			seqs.push_back(l2);
		}
	}
	const char* mask = getenv("HOST_WALK_MASK");
	if (mask && !mask[0])
		mask = nullptr;
	if (mask && strlen(mask) != k) {
		fprintf(stderr, "host_walk: HOST_WALK_MASK must have k characters\n");
		return 2;
	}
	std::vector<uint8_t> counters(m, 0);
	for (auto& s : seqs)
		abo_cbf_load_seq(counters.data(), m, s.data(), s.size(), k, H, mask);

	HostCtx c;
	c.k = k; c.trim = trim; c.H = H; c.threshold = kc;
	c.rt = make_rolltab(k);
	c.mask = mask;
	std::vector<uint8_t> mpos;
	for (unsigned i = 0; mask && i < k; ++i)
		if (mask[i] == '0')
			mpos.push_back((uint8_t)i);
	c.rt.nmask = (unsigned)mpos.size();
	c.rt.mpos = mpos.data();
	c.cfg.H = H; c.cfg.k = k; c.cfg.mod = make_fastmod(m);
	for (unsigned i = 0; i < kMaxHashes; ++i)
		c.cfg.mult[i] = (uint64_t)i ^ ((uint64_t)k * kMultiSeed);
	c.counters = counters.data();
	std::vector<Frame> frames(kFrameCap);
	std::vector<uint64_t> look(kLookCap);
	c.frames = frames.data();
	c.look = look.data();

	if (getenv("HOST_WALK_TILES")) {
		// markers = solid k-mers of the reads whose canonical hash has its low bits clear; 4 tiles each
		std::vector<uint8_t> sb(kTileCap);
		std::vector<uint64_t> sh(kTileCap);
		// the marker set sized as ensure_tile_store would for every window being solid: it never fills here
		uint64_t windows = 0;
		for (auto& s : seqs)
			windows += s.size() >= k ? s.size() - k + 1 : 0;
		unsigned mset_cap = 1;
		while (mset_cap < (windows / (kMarkerMask + 1) * 2 + 4096) * 4)
			mset_cap <<= 1;
		std::vector<unsigned long long> mset(mset_cap, 0);
		const char* drop = getenv("HOST_WALK_DROP_TILES");
		const uint64_t drop_seed = drop ? strtoull(drop, nullptr, 10) : 0;
		size_t n_markers = 0, dropped = 0, lost_one = 0, lost_all = 0;
		for (auto& s : seqs) {
			if (s.size() < k)
				continue;
			size_t bad = s.find_first_not_of("ACGT"); // the first non-ACGT base at or after j: one scan per read, not per window
			for (size_t j = 0; j + k <= s.size(); ++j) {
				if (bad < j)
					bad = s.find_first_not_of("ACGT", j);
				if (bad < j + k)
					continue;
				Vtx<KW> v = vtx_from_codes<KW>((const uint8_t*)s.data() + j, k, true, c.rt);
				if (!is_marker(v.canon()) || !c.contains(v.bloom()))
					continue;
				const unsigned ins = marker_set_insert(mset.data(), mset_cap - 1, v.canon());
				if (ins == MARKER_NO_ROOM) {
					fprintf(stderr, "host_walk: marker set full\n");
					return 4;
				}
				if (ins != MARKER_FRESH)
					continue;
				++n_markers;
				// 1 marker in 8 loses one of its tiles, 1 in 8 all four
				const uint64_t r = drop ? splitmix64(drop_seed ^ v.canon()) : 0;
				const unsigned drop_mask = !drop ? 0u : (r & 7) == 0 ? 15u : (r & 7) == 1 ? 1u << ((r >> 3) & 3) : 0u;
				lost_one += drop_mask && drop_mask != 15u;
				lost_all += drop_mask == 15u;
				const Vtx<KW> rc = vtx_revcomp(v, k);
				for (int w = 0; w < 4; ++w) {
					if (drop_mask >> w & 1) {
						++dropped;
						continue;
					}
					TileRec t;
					memset(&t, 0, sizeof t);
					make_tile(c, (w & 2) ? rc : v, (w & 1) ? REV : FWD, &t, sb.data(), sh.data());
					c.tile_mem.emplace_back(new uint8_t[t.n * 9 + 16]);
					uint8_t* mem = c.tile_mem.back().get();
					t.hashes = (uint64_t*)mem;
					t.bases = mem + 8 * (size_t)t.n;
					memcpy(t.hashes, sh.data(), 8 * (size_t)t.n);
					memcpy(t.bases, sb.data(), t.n);
					c.tile_recs.push_back(t);
				}
			}
		}
		for (uint32_t i = 0; i < c.tile_recs.size(); ++i)
			c.tile_multi.emplace(HostCtx::tkey(c.tile_recs[i].key, c.tile_recs[i].cls), i);
		c.use_tiles = true;
		size_t linked = 0;
		for (auto& t : c.tile_recs)
			if (t.stop_kind == TS_MARKER && t.n) {
				const TileRec* o = c.tile_lookup(t.end_key, ((unsigned)t.end_orient << 1) | (t.cls & 1u));
				if (o) {
					t.next = c.tile_index(o) + 1;
					++linked;
				}
			}
		c.tile_splices = 0;
		fprintf(stderr, "host_walk: %zu tiles from %zu markers, %zu linked, %zu dropped (%zu markers lost one tile, %zu all four)\n",
		        c.tile_recs.size(), n_markers, linked, dropped, lost_one, lost_all);
	}

	Assembly as;
	as.c = &c;
	as.mbits = m;
	as.assembled.assign(m / 8, 0);
	FILE* log = logpath ? fopen(logpath, "w") : nullptr;
	if (log)
		fprintf(log, "read_id\tresult\n");
	static const char* names[] = { "SHORTER_THAN_K", "NON_ACGT", "BLUNT_END", "NOT_SOLID", "ALL_KMERS_VISITED", "GENERATED_CONTIGS" };
	size_t fallbacks = 0;
	for (size_t r = 0; r < seqs.size(); ++r) {
		const std::string& s = seqs[r];
		int code;
		std::vector<uint64_t> hs;
		if (s.size() < k)
			code = RC_SHORTER_THAN_K;
		else if (s.find_first_not_of("ACGT") != std::string::npos)
			code = RC_NON_ACGT;
		else {
			// hasBluntEnd (bloom-dbg.h:494-532)
			Vtx<KW> first = vtx_from_codes<KW>((const uint8_t*)s.data(), k, true, c.rt);
			Vtx<KW> last = vtx_from_codes<KW>((const uint8_t*)s.data() + s.size() - k, k, true, c.rt);
			bool blunt = !look_ahead(c, first, REV, kFpTrim) || !look_ahead(c, vtx_revcomp(last, k), REV, kFpTrim);
			if (blunt)
				code = RC_BLUNT_END;
			else {
				std::vector<uint64_t> tmp((s.size() - k + 1) * H);
				size_t n = abo_hash_seq(s.data(), s.size(), k, H, c.mask, tmp.data(), NULL);
				hs.resize(n);
				for (size_t i = 0; i < n; ++i)
					hs[i] = tmp[i * H];
				bool solid = true, visited = true;
				for (uint64_t h : hs)
					if (!c.contains(h)) {
						solid = false;
						break;
					}
				if (!solid)
					code = RC_NOT_SOLID;
				else {
					for (uint64_t h : hs)
						if (!as.inAssembled(h)) {
							visited = false;
							break;
						}
					if (visited)
						code = RC_ALL_KMERS_VISITED;
					else {
						code = RC_GENERATED_CONTIGS;
						as.readID = &ids[r];
						as.collected.clear();
						bool repeat = false;
						if (!walk_read<KW>(c, (const uint8_t*)s.data(), (unsigned)s.size(), as)) {
							if (!c.use_tiles || !c.tile_cycle) {
								fprintf(stderr, "host_walk: walk failed on read %zu\n", r);
								return 4;
							}
							repeat = true; // tile chain cycled: exact fallback below
							c.fail_ = false;
							c.tile_cycle = false;
						}
						if (c.use_tiles && !repeat)
							for (auto& x : as.collected)
								repeat |= as.has_repeat(x);
						if (repeat) { // exact fallback: walk this read again vertex by vertex
							++fallbacks;
							c.use_tiles = false;
							as.collected.clear();
							c.allocs.clear();
							if (!walk_read<KW>(c, (const uint8_t*)s.data(), (unsigned)s.size(), as))
								return 4;
							c.use_tiles = true;
						}
						for (auto& x : as.collected)
							as.output(x);
						c.allocs.clear();
					}
				}
			}
		}
		if (log)
			fprintf(log, "%s\t%s\n", ids[r].c_str(), names[code]);
	}
	if (log)
		fclose(log);
	fprintf(stderr, "host_walk: %zu reads, %zu contigs, %llu neighbour probes, %llu tile splices, %zu serial fallbacks\n", seqs.size(),
	        as.contigID, c.probes, c.tile_splices, fallbacks);
	return 0;
}

/** marker_set_insert on sets it fills: every key is fresh exactly once, a full set answers MARKER_NO_ROOM (the loop is bounded
 *  by construction, so the check is that the answer is right), and keys stored before the set filled up are still found */
static int markerset_check()
{
	int bad = 0;
	for (unsigned cap : { 64u, 128u, 4096u }) {
		std::vector<unsigned long long> set(cap, 0);
		std::unordered_set<uint64_t> fresh;
		std::vector<uint64_t> keys;
		unsigned no_room = 0, seen_twice = 0;
		for (uint64_t i = 0; i < 4ull * cap; ++i) {
			const uint64_t key = splitmix64(i) & ~kMarkerMask; // markers; key 0 (stored as 1) comes first
			keys.push_back(i == 0 ? 0 : key);
			const unsigned r = marker_set_insert(set.data(), cap - 1, keys.back());
			if (r == MARKER_FRESH && !fresh.insert(keys.back()).second)
				++seen_twice;
			no_room += r == MARKER_NO_ROOM;
			if (cap <= kMarkerProbes && r == MARKER_NO_ROOM && fresh.size() < cap) {
				fprintf(stderr, "markerset: cap %u: no room with %zu of %u entries taken\n", cap, fresh.size(), cap);
				++bad;
			}
		}
		// a second pass: nothing is fresh any more, every key stored before is found
		unsigned refound = 0;
		for (uint64_t key : keys) {
			const unsigned r = marker_set_insert(set.data(), cap - 1, key);
			if (r == MARKER_FRESH)
				++seen_twice;
			refound += r == MARKER_SEEN && fresh.count(key);
		}
		const bool full = fresh.size() == cap || (cap > kMarkerProbes && no_room > 0);
		printf("cap %u fresh %zu no_room %u refound %u twice %u\n", cap, fresh.size(), no_room, refound, seen_twice);
		if (seen_twice || !full || fresh.size() > cap || refound < fresh.size() || !no_room) {
			fprintf(stderr, "markerset: cap %u failed\n", cap);
			++bad;
		}
	}
	return bad ? 1 : 0;
}

int main(int argc, char** argv)
{
	if (argc == 2 && !strcmp(argv[1], "markerset"))
		return markerset_check();
	if (argc < 7) {
		fprintf(stderr, "usage: host_walk K KC H COUNTERS TRIM reads.fq [readlog]\n");
		return 2;
	}
	unsigned k = atoi(argv[1]), kc = atoi(argv[2]), H = atoi(argv[3]);
	uint64_t m = strtoull(argv[4], 0, 10);
	unsigned trim = atoi(argv[5]);
	const char* log = argc > 7 ? argv[7] : nullptr;
	const unsigned kw = (2 * k + 63) / 64;
	switch (kw) {
	case 1: return run<1>(k, kc, H, m, trim, argv[6], log);
	case 2: return run<2>(k, kc, H, m, trim, argv[6], log);
	case 3: return run<3>(k, kc, H, m, trim, argv[6], log);
	case 4: return run<4>(k, kc, H, m, trim, argv[6], log);
	default: return run<6>(k, kc, H, m, trim, argv[6], log);
	}
}
