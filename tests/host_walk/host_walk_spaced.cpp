// tests/host_walk/host_walk_spaced.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// host_walk with tiles under a spaced seed, built the way the kernels build them: a marker is a read window, all of whose k
// bases are ACGT, whose tile_key (the canonical hash of the full k-mer, abb_walk.cuh) has its low bits clear and whose Bloom
// hash is solid (k_find_markers); and the repeat check that guards the splices enters the trimmed-off end vertices with
// their Bloom hashes, as k_repeat_check does.  It reuses host_walk.cpp's single-lane context and -j1 driver pieces (HostCtx,
// Assembly); without a mask it computes what `HOST_WALK_TILES=1 host_walk` computes.
//
//   host_walk_spaced K KC H COUNTERS TRIM MASK reads.fq readlog.tsv [DROP_SEED] > out.fa
//
// MASK is the spaced seed ('-' for none).  DROP_SEED leaves out a seeded subset of the tiles, as a full tile store does on the
// GPU: one of the four tiles of some markers, all four of others.
#define main host_walk_main
#include "host_walk.cpp"
#undef main

namespace {

/** Assembly whose repeat check sees the trimmed-off end vertices as the Bloom hashes it hashes the rest of the contig with */
struct SpacedAssembly : Assembly {
	void operator()(HostCtx& c, unsigned seed_i, const ContigOut& o)
	{
		Assembly::operator()(c, seed_i, o);
		collected.back().front_h = o.front_b;
		collected.back().back_h = o.back_b;
	}
};

template <int KW>
int run_spaced(unsigned k, unsigned kc, unsigned H, uint64_t m, unsigned trim, const char* mask, const char* path, const char* logpath,
               const char* drop)
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
			const size_t sp = l1.find_first_of(" \t");
			ids.push_back(l1.substr(1, sp == std::string::npos ? std::string::npos : sp - 1));
			for (auto& ch : l2)
				ch = (char)toupper(ch);
			seqs.push_back(l2);
		}
	}
	if (mask && strlen(mask) != k) {
		fprintf(stderr, "host_walk_spaced: the mask must have k characters\n");
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

	{ // markers and their four tiles each
		std::vector<uint8_t> sb(kTileCap);
		std::vector<uint64_t> sh(kTileCap);
		uint64_t windows = 0;
		for (auto& s : seqs)
			windows += s.size() >= k ? s.size() - k + 1 : 0;
		unsigned mset_cap = 1;
		while (mset_cap < (windows / (kMarkerMask + 1) * 2 + 4096) * 4)
			mset_cap <<= 1;
		std::vector<unsigned long long> mset(mset_cap, 0);
		const uint64_t drop_seed = drop ? strtoull(drop, nullptr, 10) : 0;
		size_t n_markers = 0, dropped = 0, lost_one = 0, lost_all = 0;
		for (auto& s : seqs) {
			if (s.size() < k)
				continue;
			size_t bad = s.find_first_not_of("ACGT");
			for (size_t j = 0; j + k <= s.size(); ++j) {
				if (bad < j)
					bad = s.find_first_not_of("ACGT", j);
				if (bad < j + k) // the full k-mer, don't-care positions included, must be ACGT
					continue;
				const Vtx<KW> v = vtx_from_codes<KW>((const uint8_t*)s.data() + j, k, true, c.rt);
				const uint64_t key = tile_key(v, c.rt);
				if (!is_marker(key) || !c.contains(v.bloom()))
					continue;
				const unsigned ins = marker_set_insert(mset.data(), mset_cap - 1, key);
				if (ins == MARKER_NO_ROOM) {
					fprintf(stderr, "host_walk_spaced: marker set full\n");
					return 4;
				}
				if (ins != MARKER_FRESH)
					continue;
				++n_markers;
				const uint64_t r = drop ? splitmix64(drop_seed ^ key) : 0;
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
		fprintf(stderr, "host_walk_spaced: %zu tiles from %zu markers, %zu linked, %zu dropped (%zu markers lost one tile, %zu all four)\n",
		        c.tile_recs.size(), n_markers, linked, dropped, lost_one, lost_all);
	}

	SpacedAssembly as;
	as.c = &c;
	as.mbits = m;
	as.assembled.assign(m / 8, 0);
	FILE* log = fopen(logpath, "w");
	if (!log)
		return 2;
	fprintf(log, "read_id\tresult\n");
	static const char* names[] = { "SHORTER_THAN_K", "NON_ACGT", "BLUNT_END", "NOT_SOLID", "ALL_KMERS_VISITED", "GENERATED_CONTIGS" };
	size_t fallbacks = 0;
	for (size_t r = 0; r < seqs.size(); ++r) {
		const std::string& s = seqs[r];
		int code;
		if (s.size() < k)
			code = RC_SHORTER_THAN_K;
		else if (s.find_first_not_of("ACGT") != std::string::npos)
			code = RC_NON_ACGT;
		else if (!look_ahead(c, vtx_from_codes<KW>((const uint8_t*)s.data(), k, true, c.rt), REV, kFpTrim) ||
		         !look_ahead(c, vtx_revcomp(vtx_from_codes<KW>((const uint8_t*)s.data() + s.size() - k, k, true, c.rt), k), REV, kFpTrim))
			code = RC_BLUNT_END; // hasBluntEnd (bloom-dbg.h:494-532)
		else {
			std::vector<uint64_t> tmp((s.size() - k + 1) * H);
			const size_t n = abo_hash_seq(s.data(), s.size(), k, H, c.mask, tmp.data(), NULL);
			bool solid = true, visited = true;
			for (size_t i = 0; i < n; ++i) {
				solid &= c.contains(tmp[i * H]);
				visited &= as.inAssembled(tmp[i * H]);
			}
			if (!solid)
				code = RC_NOT_SOLID;
			else if (visited)
				code = RC_ALL_KMERS_VISITED;
			else {
				code = RC_GENERATED_CONTIGS;
				as.readID = &ids[r];
				as.collected.clear();
				bool repeat = false;
				if (!walk_read<KW>(c, (const uint8_t*)s.data(), (unsigned)s.size(), as)) {
					if (!c.tile_cycle) {
						fprintf(stderr, "host_walk_spaced: walk failed on read %zu\n", r);
						return 4;
					}
					repeat = true; // tile chain cycled: exact fallback below
					c.fail_ = false;
					c.tile_cycle = false;
				}
				if (!repeat)
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
		fprintf(log, "%s\t%s\n", ids[r].c_str(), names[code]);
	}
	fclose(log);
	fprintf(stderr, "host_walk_spaced: %zu reads, %zu contigs, %llu neighbour probes, %llu tile splices, %zu serial fallbacks\n",
	        seqs.size(), as.contigID, c.probes, c.tile_splices, fallbacks);
	return 0;
}

} // namespace

int main(int argc, char** argv)
{
	if (argc < 9) {
		fprintf(stderr, "usage: host_walk_spaced K KC H COUNTERS TRIM MASK reads.fq readlog [DROP_SEED]\n");
		return 2;
	}
	const unsigned k = atoi(argv[1]), kc = atoi(argv[2]), H = atoi(argv[3]);
	const uint64_t m = strtoull(argv[4], 0, 10);
	const unsigned trim = atoi(argv[5]);
	const char* mask = strcmp(argv[6], "-") ? argv[6] : nullptr;
	const char* drop = argc > 9 ? argv[9] : nullptr;
	switch ((2 * k + 63) / 64) {
	case 1: return run_spaced<1>(k, kc, H, m, trim, mask, argv[7], argv[8], drop);
	case 2: return run_spaced<2>(k, kc, H, m, trim, mask, argv[7], argv[8], drop);
	case 3: return run_spaced<3>(k, kc, H, m, trim, mask, argv[7], argv[8], drop);
	case 4: return run_spaced<4>(k, kc, H, m, trim, mask, argv[7], argv[8], drop);
	default: return run_spaced<6>(k, kc, H, m, trim, mask, argv[7], argv[8], drop);
	}
}
