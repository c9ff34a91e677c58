// AdjList (GPU) -- the reference's AdjList command line (AdjList/AdjList.cpp; run by bin/abyss-pe:577 on the unitig
// FASTA that abyss-bloom-dbg writes) over libabyssb200: contig ends are hashed, joined and verified on the GPU
// (abb_overlap_build, csrc/abb_overlap.cu); options, formats and output bytes are the reference's.
//
//   AdjList -k<kmer> [-m<min_overlap>] [--adj|--dot|--gfa1|--gfa2|--asqg|--sam] [--SS] [FILE]... > graph
#include "adjlist_main.h"

int main(int argc, char** argv)
{
	return adjlist::run(argc, argv,
	                    [](const char* bases, const uint64_t* offsets, uint64_t n, unsigned k, unsigned m, int ss, int device,
	                       const abb_overlap_edge** edges, uint64_t* n_edges) {
		                    abb_overlap* h = nullptr; // lives until exit: the edge array belongs to it
		                    int rc = abb_overlap_create(&h, device);
		                    if (rc == ABB_OK)
			                    rc = abb_overlap_build(h, bases, offsets, n, k, m, ss, edges, n_edges);
		                    if (rc != ABB_OK) {
			                    std::cerr << ADJ_PROGRAM ": " << abb_last_error() << "\n";
			                    exit(EXIT_FAILURE);
		                    }
	                    });
}
