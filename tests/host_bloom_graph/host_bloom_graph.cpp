// tests/host_bloom_graph/host_bloom_graph.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// CPU emulation of `abyss-bloom graph`: the product's traversal (abyss_b200/host/bloom_graph.h) with the GPU query replaced by a
// loop over the 32 lanes of the SAME device functions (kmer_hash_part, nbr_lane at the probe bound the kernel is launched with,
// nbr_mask of csrc/abb_graph.cuh), on rolling-hash filters rebuilt by the C oracle from the reads they were built from.  Prints the dump (stdout only).
//
//   host_bloom_graph K DEPTH FILTER [-R KMER | -f FASTA | -a ATTR:FASTA | -A ATTR:FILTER]...
//   FILTER = H,LEVELS,BITS_PER_LEVEL,READS[+READS...]   (abyss-bloom build -t rolling-hash; the last level is the filter)
#include "../../abyss_b200/csrc/abb_graph.cuh"
#include "../../abyss_b200/host/bloom_graph.h"
#include "../../abyss_b200/host/reads.h"
#include <iostream>
#include <sstream>
extern "C" {
#include "../../oracle/abyss_oracle.h"
}

using namespace abb;

struct Bits {
	unsigned H = 0;
	uint64_t mbits = 0;
	std::vector<uint8_t> levels; // all levels; the last is the filter
	const uint8_t* last() const { return levels.data() + (levels.size() - mbits / 8); }
};

static Bits build(unsigned k, const std::string& spec)
{
	std::istringstream in(spec);
	std::string f;
	std::vector<std::string> p;
	while (std::getline(in, f, ','))
		p.push_back(f);
	Bits b;
	b.H = atoi(p[0].c_str());
	const unsigned L = atoi(p[1].c_str());
	b.mbits = strtoull(p[2].c_str(), 0, 10);
	b.levels.assign(b.mbits / 8 * L, 0);
	std::istringstream files(p[3]);
	host::ReadOpts ropt;
	while (std::getline(files, f, '+')) {
		host::SeqReader r(f, ropt);
		std::string id, seq;
		while (r.next(id, seq))
			abo_casc_load_seq(b.levels.data(), b.mbits, L, seq.data(), seq.size(), k, b.H, nullptr);
	}
	return b;
}

/** canonical hash and position of every valid window of a sequence */
static std::vector<std::pair<uint64_t, uint32_t>> windows(const std::string& s, unsigned k)
{
	std::vector<uint64_t> h(s.size() + 1);
	std::vector<uint32_t> pos(s.size() + 1);
	const size_t n = abo_hash_seq(s.data(), s.size(), k, 1, nullptr, h.data(), pos.data());
	std::vector<std::pair<uint64_t, uint32_t>> out;
	for (size_t i = 0; i < n; ++i)
		out.emplace_back(h[i], pos[i]);
	return out;
}

int main(int argc, char** argv)
{
	if (argc < 4) {
		fprintf(stderr, "usage: host_bloom_graph K DEPTH FILTER [-R KMER | -f FASTA | -a ATTR:FASTA | -A ATTR:FILTER]...\n");
		return 2;
	}
	const unsigned k = atoi(argv[1]);
	const unsigned depth = (unsigned)strtoull(argv[2], 0, 10); // as abyss-bloom graph stores -d
	const Bits g = build(k, argv[3]);
	NbrQuery q;
	q.cfg.H = g.H;
	q.cfg.k = k;
	q.cfg.mod = make_fastmod(g.mbits);
	for (unsigned i = 0; i < kMaxHashes; ++i)
		q.cfg.mult[i] = (uint64_t)i ^ ((uint64_t)k * kMultiSeed);
	q.rt = make_rolltab(k);
	q.bits = g.last();
	q.n_attr = 0;
	auto contains = [&](uint64_t h0) {
		for (unsigned i = 0; i < g.H; ++i)
			if (!bit_at(q.bits, nth_pos(h0, q.cfg, i)))
				return false;
		return true;
	};
	host::ReadOpts ropt;
	host::GraphRoots roots;
	std::vector<host::FastaAttr> fastaAttrs;
	std::vector<std::string> bloomAttrs;
	std::vector<Bits> attrBits;
	std::vector<std::string> rootFastas;
	for (int i = 4; i + 1 < argc; i += 2) {
		const std::string opt = argv[i], val = argv[i + 1];
		if (opt == "-R") {
			const auto w = windows(val, k);
			if (!w.empty() && contains(w[0].first))
				roots.add(w[0].first, val.data(), k);
		} else if (opt == "-f")
			rootFastas.push_back(val);
		else if (opt == "-a") {
			fastaAttrs.emplace_back(val.substr(0, val.find(':')), std::unordered_set<uint64_t>());
			host::SeqReader r(val.substr(val.find(':') + 1), ropt);
			std::string id, seq;
			while (r.next(id, seq))
				for (const auto& w : windows(seq, k))
					fastaAttrs.back().second.insert(w.first);
		} else if (opt == "-A") {
			bloomAttrs.push_back(val.substr(0, val.find(':')));
			attrBits.push_back(build(k, val.substr(val.find(':') + 1)));
		}
	}
	for (const std::string& path : rootFastas) { // -f after every -R, as the reference inserts them
		host::SeqReader r(path, ropt);
		std::string id, seq;
		while (r.next(id, seq))
			for (const auto& w : windows(seq, k))
				if (contains(w.first))
					roots.add(w.first, seq.data() + w.second, k);
	}
	q.n_attr = (unsigned)attrBits.size();
	for (unsigned a = 0; a < q.n_attr; ++a)
		q.attr[a] = { attrBits[a].last(), make_fastmod(attrBits[a].mbits), attrBits[a].H };
	host::bloom_graph(
	    k, depth, roots, fastaAttrs, bloomAttrs,
	    [&](const char* kmers, uint64_t n, abb_nbr_info* out) {
		    for (uint64_t v = 0; v < n; ++v) {
			    const uint8_t* km = (const uint8_t*)kmers + v * k;
			    HashPair h = { 0, 0 };
			    for (unsigned lane = 0; lane < 32; ++lane) {
				    const HashPair p = kmer_hash_part(km, k, lane, 32);
				    h.fh ^= p.fh;
				    h.rh ^= p.rh;
			    }
			    abb_nbr_info o = {};
			    unsigned gl = 0, al = 0;
			    for (unsigned lane = 0; lane < 32; ++lane) {
				    bool gok, aok;
				    const uint64_t hn = nbr_lane<kMaxLaneProbes>(q, h, base_code(km[0]) & 3u, base_code(km[k - 1]) & 3u, lane, &gok, &aok);
				    gl |= (unsigned)gok << lane;
				    al |= (unsigned)aok << lane;
				    if ((lane & 3) == 0)
					    o.hash[lane >> 2] = hn;
			    }
			    o.self = h.canonical();
			    o.attr = al;
			    o.mask = (uint8_t)nbr_mask(gl);
			    out[v] = o;
		    }
	    },
	    std::cout);
	return 0;
}
