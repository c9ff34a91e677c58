// bloom_graph.h -- `abyss-bloom graph`: the GraphViz dump of the rolling-hash Bloom filter de Bruijn graph around root k-mers, in
// the reference's order, with the Bloom lookups behind one functor.  abyss_bloom.cc passes the C ABI (abb_graph_neighbors: CUDA),
// the CPU test harness (tests/host_bloom_graph) an emulation built on the same device functions.
#pragma once
#include "../../include/abyss_b200.h"
#include <ostream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

namespace host {

/** The roots of the search: -R k-mers in command-line order, then every window of the -f files, each inserted once up to
 *  reverse complement, the first string inserted being the one printed (Bloom/bloom.cc:1112-1137). */
struct GraphRoots {
	// The search starts from the roots in the iteration order of this set, and that order is the order of the output.  The
	// reference keeps its roots in a std::unordered_set<RollingBloomDBGVertex> whose std::hash is the canonical ntHash
	// (BloomDBG/RollingBloomDBG.h:163-172) and whose equality is canonical k-mer equality.  libstdc++ orders such a set by the
	// hash values, the insertion sequence and its rehash policy alone, and this program is built with the same library, so a set
	// of the same hashes inserted in the same order iterates in the reference's order.  It must never be reserve()d: the
	// sequence of rehashes is part of the order.
	std::unordered_set<uint64_t> set;
	std::unordered_map<uint64_t, std::string> text;
	void add(uint64_t hash, const char* kmer, unsigned k)
	{
		if (set.insert(hash).second)
			text.emplace(hash, std::string(kmer, k));
	}
};

/** a -a/--fasta-attr attribute: its text and the canonical hashes of the k-mers of its FASTA file */
using FastaAttr = std::pair<std::string, std::unordered_set<uint64_t>>;

/** breadthFirstSearchMulti(roots, g, undirected = true, RollingBloomDBGVisitor) (Graph/BreadthFirstSearch.h:95-173,
 *  Bloom/RollingBloomDBGVisitor.h):
 *   - every root is discovered, in the set's order, at depth 0;
 *   - FIFO: each dequeued vertex u visits its out-edges u[1:] + b, then its in-edges b + u[:-1], b = A, C, G, T;
 *   - an edge to an undiscovered vertex discovers it at depth(u) + 1, printing "u -> v" first if it is an out-edge, unless
 *     depth(u) >= maxDepth: then nothing happens and the vertex stays undiscovered;
 *   - an edge to a discovered vertex prints "u -> v" if it is an out-edge, and an in-edge w -> u only if w is u up to reverse
 *     complement (isForwardEdge compares the edge's source with u);
 *   - a vertex is printed in the orientation it was reached in, with its depth, the -a attributes whose set holds it and the -A
 *     filters that contain it.
 *  A FIFO search visits the vertices level by level, so one query per level (`neighbors(kmers, n, out)`, abb_graph_neighbors:
 *  neighbour hashes and mask, attribute bits) serves the whole level: it gives the edges of the level's vertices and the
 *  attributes of their lines, which the previous level discovered.  So the text of level d is written when the query of level
 *  d + 1 has returned. */
template <typename NbrFn>
void bloom_graph(unsigned k, unsigned maxDepth, const GraphRoots& roots, const std::vector<FastaAttr>& fastaAttrs,
                 const std::vector<std::string>& bloomAttrs, NbrFn neighbors, std::ostream& out)
{
	static const char BASES[] = "ACGT";
	out << "digraph  {\n";
	std::unordered_set<uint64_t> discovered; // the colour map: white = absent
	std::vector<std::string> level, next;    // the vertices of one depth, in queue order
	for (uint64_t h : roots.set) {
		discovered.insert(h);
		level.push_back(roots.text.at(h));
	}
	// the text of the previous level: runs of edge lines, and the places of the vertex lines of `level` (offset, index)
	std::string text;
	std::vector<std::pair<size_t, size_t>> lines;
	for (size_t i = 0; i < level.size(); ++i)
		lines.emplace_back(0, i);
	std::vector<abb_nbr_info> info;
	std::string kmers;
	for (unsigned depth = 0; !level.empty(); ++depth) {
		kmers.clear();
		for (const std::string& u : level)
			kmers += u;
		info.resize(level.size());
		neighbors(kmers.data(), (uint64_t)level.size(), info.data());
		size_t at = 0;
		for (const auto& l : lines) { // discover_vertex of the vertices of this depth
			out.write(text.data() + at, (std::streamsize)(l.first - at));
			at = l.first;
			const abb_nbr_info& v = info[l.second];
			out << '\t' << level[l.second] << " [depth=" << depth;
			for (const FastaAttr& a : fastaAttrs)
				if (a.second.count(v.self))
					out << ',' << a.first;
			for (size_t a = 0; a < bloomAttrs.size(); ++a)
				if ((v.attr >> a) & 1)
					out << ',' << bloomAttrs[a];
			out << "];\n";
		}
		out.write(text.data() + at, (std::streamsize)(text.size() - at));
		text.clear();
		lines.clear();
		next.clear();
		for (size_t i = 0; i < level.size(); ++i) {
			const std::string& u = level[i];
			const abb_nbr_info& v = info[i];
			for (unsigned j = 0; j < 8; ++j) {
				if (!((v.mask >> j) & 1))
					continue;
				const bool outEdge = j < 4;
				const std::string w = outEdge ? u.substr(1) + BASES[j] : BASES[j - 4] + u.substr(0, k - 1);
				if (!discovered.count(v.hash[j])) { // tree_edge
					if (depth >= maxDepth)
						continue;
					discovered.insert(v.hash[j]);
					if (outEdge)
						text += '\t' + u + " -> " + w + ";\n";
					lines.emplace_back(text.size(), next.size());
					next.push_back(w);
				} else if (outEdge) // non_tree_edge
					text += '\t' + u + " -> " + w + ";\n";
				else if (v.hash[j] == v.self)
					text += '\t' + w + " -> " + u + ";\n";
			}
		}
		level.swap(next);
	}
	out << text << "}\n";
}

} // namespace host
