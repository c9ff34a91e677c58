// adjlist_main.h -- the reference's AdjList command line (AdjList/AdjList.cpp:33-425) and its graph writers
// (Graph/AdjIO.h, DotIO.h, GfaIO.h, AsqgIO.h, SAMIO.h) over an edge list.  The overlap computation itself is a
// functor: the AdjList program (adjlist.cc) passes the C ABI (abb_overlap_build, CUDA), the CPU test harness
// (tests/host_overlap) passes a single-thread emulation of the same per-item functions.
#pragma once
#include "../../include/abyss_b200.h"
#include "reads.h"
#include <getopt.h>
#include <algorithm>
#include <iomanip>
#include <iostream>
#include <iterator>
#include <sstream>
#include <unordered_set>

namespace adjlist {

#define ADJ_PROGRAM "AdjList"

/** Graph/Options.h:13 */
enum { ADJ, ASQG, DIST, DOT, DOT_MEANCOV, GFA1, GFA2, SAM, TSV };

struct Contig {
	std::string name;
	unsigned length = 0, coverage = 0;
};

struct Graph {
	std::vector<Contig> contigs;
	const abb_overlap_edge* edges = nullptr; // vertices ascending, out-lists in the reference's order
	uint64_t n_edges = 0;
	unsigned k = 0;
	std::string vname(uint32_t v) const { return contigs[v >> 1].name + ((v & 1) ? '-' : '+'); }
};

/** " [d=-N]" only when the distance is not the default -(k-1) (write_edge_prop, AdjIO.h:19-24; Distance(), ContigProperties.h:135) */
inline void write_edge_prop(std::ostream& out, const Graph& g, const abb_overlap_edge& e)
{
	if (e.distance != -(int)g.k + 1)
		out << " [d=" << e.distance << ']';
}

/** write_adj (Graph/AdjIO.h:31-61) */
inline void write_adj(std::ostream& out, const Graph& g)
{
	uint64_t ei = 0;
	for (uint32_t u = 0; u < 2 * g.contigs.size(); ++u) {
		const bool sense = u & 1;
		const Contig& c = g.contigs[u >> 1];
		if (!sense)
			out << c.name << ' ' << c.length << ' ' << c.coverage;
		out << "\t;";
		for (; ei < g.n_edges && g.edges[ei].u == u; ++ei) {
			out << ' ' << g.vname(g.edges[ei].v ^ (uint32_t)sense);
			write_edge_prop(out, g, g.edges[ei]);
		}
		if (sense)
			out << '\n';
	}
}

/** write_dot (Graph/DotIO.h:82-119) */
inline void write_dot(std::ostream& out, const Graph& g)
{
	out << "digraph adj {\n";
	if (g.k > 0)
		out << "graph [k=" << g.k << "]\nedge [d=" << -int(g.k - 1) << "]\n";
	for (uint32_t u = 0; u < 2 * g.contigs.size(); ++u) {
		const Contig& c = g.contigs[u >> 1];
		out << '"' << g.vname(u) << "\" [l=" << c.length << " C=" << c.coverage << "]\n";
	}
	for (uint64_t i = 0; i < g.n_edges; ++i) {
		out << '"' << g.vname(g.edges[i].u) << "\" -> \"" << g.vname(g.edges[i].v) << '"';
		write_edge_prop(out, g, g.edges[i]);
		out << '\n';
	}
	out << "}\n";
}

/** only the canonical one of an edge and its complement is written (GfaIO.h:52-54) */
inline bool canonical_edge(const abb_overlap_edge& e) { return !(e.u > (e.v ^ 1u)); }

/** write_gfa1 (Graph/GfaIO.h:17-68) */
inline void write_gfa1(std::ostream& out, const Graph& g)
{
	out << "H\tVN:Z:1.0\n";
	for (const Contig& c : g.contigs) {
		out << "S\t" << c.name << "\t*\tLN:i:" << c.length;
		if (c.coverage > 0)
			out << "\tKC:i:" << c.coverage;
		out << '\n';
	}
	for (uint64_t i = 0; i < g.n_edges; ++i) {
		const abb_overlap_edge& e = g.edges[i];
		if (!canonical_edge(e))
			continue;
		out << "L\t" << g.contigs[e.u >> 1].name << '\t' << ((e.u & 1) ? '-' : '+') << '\t' << g.contigs[e.v >> 1].name << '\t'
		    << ((e.v & 1) ? '-' : '+');
		if (e.distance <= 0)
			out << '\t' << -e.distance << "M\n";
		else
			out << "\t*\n";
	}
}

/** write_gfa2 (Graph/GfaIO.h:70-218) */
inline void write_gfa2(std::ostream& out, const Graph& g)
{
	out << "H\tVN:Z:2.0\n";
	for (const Contig& c : g.contigs) {
		out << "S\t" << c.name << '\t' << c.length << "\t*";
		if (c.coverage > 0)
			out << "\tKC:i:" << c.coverage;
		out << '\n';
	}
	for (uint64_t i = 0; i < g.n_edges; ++i) {
		const abb_overlap_edge& e = g.edges[i];
		if (!canonical_edge(e))
			continue;
		const unsigned overlap = (unsigned)-e.distance, ulen = g.contigs[e.u >> 1].length, vlen = g.contigs[e.v >> 1].length;
		const bool usense = e.u & 1, vsense = e.v & 1;
		const unsigned ustart = usense ? 0 : ulen - overlap, uend = usense ? overlap : ulen;
		const unsigned vstart = !vsense ? 0 : vlen - overlap, vend = !vsense ? overlap : vlen;
		out << "E\t*\t" << g.vname(e.u) << '\t' << g.vname(e.v) << '\t' << ustart;
		if (ustart == ulen)
			out << '$';
		out << '\t' << uend;
		if (uend == ulen)
			out << '$';
		out << '\t' << vstart;
		if (vstart == vlen)
			out << '$';
		out << '\t' << vend;
		if (vend == vlen)
			out << '$';
		out << '\t' << overlap << "M\n";
	}
}

/** write_asqg (Graph/AsqgIO.h:15-74) */
inline void write_asqg(std::ostream& out, const Graph& g)
{
	out << "HT\tVN:i:1\n";
	for (const Contig& c : g.contigs) {
		out << "VT\t" << c.name << "\t*\tLN:i:" << c.length;
		if (c.coverage > 0)
			out << "\tKC:i:" << c.coverage;
		out << '\n';
	}
	for (uint64_t i = 0; i < g.n_edges; ++i) {
		const abb_overlap_edge& e = g.edges[i];
		if (!canonical_edge(e))
			continue;
		const unsigned overlap = (unsigned)-e.distance, ulen = g.contigs[e.u >> 1].length, vlen = g.contigs[e.v >> 1].length;
		const bool usense = e.u & 1, vsense = e.v & 1;
		out << "ED\t" << g.contigs[e.u >> 1].name << ' ' << g.contigs[e.v >> 1].name << ' ' << (usense ? 0 : ulen - overlap) << ' '
		    << int((usense ? overlap : ulen) - 1) << ' ' << ulen << ' ' << (!vsense ? 0 : vlen - overlap) << ' '
		    << int((!vsense ? overlap : vlen) - 1) << ' ' << vlen << ' ' << (usense != vsense) << " -1\n";
	}
}

/** write_sam (Graph/SAMIO.h:19-70) */
inline void write_sam(std::ostream& out, const Graph& g, const std::string& program, const std::string& version, const std::string& commandLine)
{
	out << "@HD\tVN:1.0\n@PG\tID:" << program << "\tVN:" << version << "\tCL:" << commandLine << '\n';
	for (const Contig& c : g.contigs) {
		out << "@SQ\tSN:" << c.name << "\tLN:" << c.length;
		if (c.coverage > 0)
			out << "\tXC:" << c.coverage;
		out << '\n';
	}
	for (uint64_t i = 0; i < g.n_edges; ++i) {
		const abb_overlap_edge& e = g.edges[i];
		if (e.distance > 0)
			continue;
		const bool usense = e.u & 1, vsense = e.v & 1;
		const unsigned flag = usense == vsense ? 0 : 0x10;
		const unsigned alen = (unsigned)-e.distance;
		const unsigned pos = 1 + (usense ? 0 : g.contigs[e.u >> 1].length - alen);
		out << g.contigs[e.v >> 1].name << '\t' << flag << '\t' << g.contigs[e.u >> 1].name << '\t' << pos << "\t255\t";
		const unsigned clip = g.contigs[e.v >> 1].length - alen;
		if (usense)
			out << clip << 'H' << alen << "M\t";
		else
			out << alen << 'M' << clip << "H\t";
		out << "*\t0\t0\t*\t*\n";
	}
}

/** write_graph (Graph/GraphIO.h:21-44) */
inline void write_graph(std::ostream& out, const Graph& g, int format, const std::string& commandLine)
{
	switch (format) {
	case ADJ: write_adj(out, g); break;
	case ASQG: write_asqg(out, g); break;
	case DOT: case DOT_MEANCOV: write_dot(out, g); break;
	case GFA1: write_gfa1(out, g); break;
	case GFA2: write_gfa2(out, g); break;
	case SAM: write_sam(out, g, ADJ_PROGRAM, "2.3.10", commandLine); break;
	default:
		std::cerr << ADJ_PROGRAM ": unsupported output format\n";
		exit(EXIT_FAILURE);
	}
}

/** printGraphStats (Graph/GraphUtil.h:43-64) without the bar plot */
inline void print_graph_stats(std::ostream& out, const Graph& g)
{
	const uint64_t v = 2 * g.contigs.size();
	std::vector<unsigned> deg(v, 0);
	for (uint64_t i = 0; i < g.n_edges; ++i)
		++deg[g.edges[i].u];
	uint64_t n0 = 0, n1 = 0, n234 = 0, mx = 0;
	for (unsigned d : deg) {
		n0 += d == 0;
		n1 += d == 1;
		n234 += d >= 2 && d <= 4;
		mx = std::max<uint64_t>(mx, d);
	}
	const uint64_t n5 = v - (n0 + n1 + n234);
	out << "V=" << v << " E=" << g.n_edges << " E/V=" << std::setprecision(3) << (float)g.n_edges / v << std::endl;
	if (v)
		out << "0: " << std::setprecision(2) << (float)100 * n0 / v << "% 1: " << std::setprecision(2) << (float)100 * n1 / v << "% 2-4: "
		    << std::setprecision(2) << (float)100 * n234 / v << "% 5+: " << std::setprecision(2) << (float)100 * n5 / v << "% max: " << mx << std::endl;
}

static const char USAGE_MESSAGE[] =
    "Usage: " ADJ_PROGRAM " -k<kmer> [OPTION]... [FILE]...\n"
    "Find overlaps of [m,k) bases. Contigs may be read from FILE(s)\n"
    "or standard input. Output is written to standard output.\n"
    "Both the overlaps of exactly k-1 bases and the shorter ones are found\n"
    "by hash joins on an NVIDIA H100 GPU.\n"
    "\n"
    " Options:\n"
    "\n"
    "  -k, --kmer=N          the length of a k-mer\n"
    "  -m, --min-overlap=M   require a minimum overlap of M bases [50]\n"
    "                        value of 0 is interpreted as k - 1\n"
    "      --adj             output the graph in ADJ format [default]\n"
    "      --asqg            output the graph in ASQG format\n"
    "      --dot             output the graph in GraphViz format\n"
    "      --gfa             output the graph in GFA1 format\n"
    "      --gfa1            output the graph in GFA1 format\n"
    "      --gfa2            output the graph in GFA2 format\n"
    "      --gv              output the graph in GraphViz format\n"
    "      --sam             output the graph in SAM format\n"
    "      --SS              expect contigs to be oriented correctly\n"
    "      --no-SS           no assumption about contig orientation\n"
    "  -v, --verbose         display verbose output\n"
    "      --help            display this help and exit\n"
    "      --version         output version information and exit\n"
    "      --device=N        CUDA device to use [0]\n"
    "\n"
    "The paired de Bruijn graph mode (-K) and the --db options of the reference are not supported.\n";

/** getCoverage (AdjList.cpp:128-134): the second integer of the FASTA comment */
inline unsigned get_coverage(const std::string& comment)
{
	std::istringstream ss(comment);
	unsigned length, coverage = 0;
	ss >> length >> coverage;
	return coverage;
}

/** build(bases, offsets, n_contigs, k, min_overlap, ss, device, &edges, &n_edges): fills the edge list or exits */
template <typename BuildFn>
int run(int argc, char** argv, BuildFn build)
{
	std::string commandLine;
	{
		std::ostringstream ss;
		char** last = argv + argc - 1;
		std::copy(argv, last, std::ostream_iterator<const char*>(ss, " "));
		ss << *last;
		commandLine = ss.str();
	}
	static int format = ADJ, ss_flag = 0;
	unsigned k = 0, minOverlap = 50, singleKmer = 0;
	int verbose = 0, device = 0;
	enum { OPT_HELP = 1, OPT_VERSION, OPT_DB, OPT_LIBRARY, OPT_STRAIN, OPT_SPECIES, OPT_DEVICE };
	static const struct option longopts[] = {
		{ "kmer", required_argument, NULL, 'k' },
		{ "single-kmer", required_argument, NULL, 'K' },
		{ "min-overlap", required_argument, NULL, 'm' },
		{ "adj", no_argument, &format, ADJ },
		{ "asqg", no_argument, &format, ASQG },
		{ "dot", no_argument, &format, DOT },
		{ "gfa", no_argument, &format, GFA1 },
		{ "gfa1", no_argument, &format, GFA1 },
		{ "gfa2", no_argument, &format, GFA2 },
		{ "gv", no_argument, &format, DOT },
		{ "sam", no_argument, &format, SAM },
		{ "SS", no_argument, &ss_flag, 1 },
		{ "no-SS", no_argument, &ss_flag, 0 },
		{ "verbose", no_argument, NULL, 'v' },
		{ "help", no_argument, NULL, OPT_HELP },
		{ "version", no_argument, NULL, OPT_VERSION },
		{ "db", required_argument, NULL, OPT_DB },
		{ "library", required_argument, NULL, OPT_LIBRARY },
		{ "strain", required_argument, NULL, OPT_STRAIN },
		{ "species", required_argument, NULL, OPT_SPECIES },
		{ "device", required_argument, NULL, OPT_DEVICE },
		{ NULL, 0, NULL, 0 }
	};
	bool die = false;
	for (int c; (c = getopt_long(argc, argv, "k:K:m:v", longopts, NULL)) != -1;) {
		std::istringstream arg(optarg != NULL ? optarg : "");
		switch (c) {
		case '?': die = true; break;
		case 'k': arg >> k; break;
		case 'K': arg >> singleKmer; break;
		case 'm': arg >> minOverlap; break;
		case 'v': verbose++; break;
		case OPT_HELP: std::cout << USAGE_MESSAGE; exit(EXIT_SUCCESS);
		case OPT_VERSION: std::cout << ADJ_PROGRAM " (abyss-b200) 0.1.0, command-line compatible with " ADJ_PROGRAM " (ABySS) 2.3.10\n"; exit(EXIT_SUCCESS);
		case OPT_DB: case OPT_LIBRARY: case OPT_STRAIN: case OPT_SPECIES: {
			std::string ignored;
			arg >> ignored; // the SQLite statistics repository of the reference is not kept
			break;
		}
		case OPT_DEVICE: arg >> device; break;
		}
		if (optarg != NULL && !arg.eof()) {
			std::cerr << ADJ_PROGRAM ": invalid option: `-" << (char)c << optarg << "'\n";
			exit(EXIT_FAILURE);
		}
	}
	if (k <= 0) {
		std::cerr << ADJ_PROGRAM ": missing -k,--kmer option\n";
		die = true;
	}
	if (singleKmer > 0) {
		std::cerr << ADJ_PROGRAM ": the paired de Bruijn graph mode (-K) is not supported by the GPU implementation\n";
		die = true;
	}
	if (die) {
		std::cerr << "Try `" << ADJ_PROGRAM << " --help' for more information.\n";
		exit(EXIT_FAILURE);
	}
	if (minOverlap == 0)
		minOverlap = k - 1;
	minOverlap = std::min(minOverlap, k - 1);

	/* readContigs (AdjList.cpp:203-245): FOLD_CASE, opt::trimMasked = false (:392) */
	host::ReadOpts ropt;
	ropt.trimMasked = 0;
	ropt.chastityFilter = 1;
	Graph g;
	g.k = k;
	std::vector<char> bases;
	std::vector<uint64_t> offsets{ 0 };
	std::unordered_set<std::string> names;
	std::vector<std::string> files(argv + optind, argv + argc);
	if (files.empty())
		files.push_back("-");
	for (const std::string& path : files) {
		if (verbose > 0)
			std::cerr << "Reading `" << path << "'...\n";
		host::SeqReader in(path, ropt);
		std::string id, seq;
		while (in.next(id, seq)) {
			if (seq.size() <= k - 1) {
				std::cerr << ADJ_PROGRAM ": contig `" << id << "' is not longer than k-1 = " << k - 1 << " bases\n";
				exit(EXIT_FAILURE);
			}
			if (!names.insert(id).second) {
				std::cerr << "error: duplicate ID: `" << id << "'\n"; // Dictionary::insert (Common/Dictionary.h)
				exit(EXIT_FAILURE);
			}
			Contig c;
			c.name = id;
			c.length = (unsigned)seq.size();
			c.coverage = get_coverage(in.last_comment());
			g.contigs.push_back(c);
			bases.insert(bases.end(), seq.begin(), seq.end());
			offsets.push_back(bases.size());
		}
	}
	if (verbose > 0)
		std::cerr << "Finding overlaps of exactly k-1 bp...\n";
	build(bases.data(), offsets.data(), (uint64_t)g.contigs.size(), k, minOverlap, ss_flag, device, &g.edges, &g.n_edges);
	if (verbose > 0)
		print_graph_stats(std::cerr, g);
	write_graph(std::cout, g, format, commandLine);
	std::cout.flush();
	if (!std::cout.good()) {
		std::cerr << ADJ_PROGRAM ": error writing the graph\n";
		return EXIT_FAILURE;
	}
	return 0;
}

} // namespace adjlist
