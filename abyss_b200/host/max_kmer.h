// max_kmer.h -- MAX_KMER of the command-line programs.  The reference refuses k above the MAX_KMER it was configured with
// (configure --enable-maxk, 192 by default; Common/Kmer.h:44-56).  These programs accept k up to 192 likewise, or up to
// the value of the environment variable ABYSS_MAX_KMER (at most 256), which plays the part of that configure option.
#pragma once
#include "../../include/abyss_b200.h"
#include <cstdlib>
#include <iostream>

namespace host {

/** sets the library's MAX_KMER from ABYSS_MAX_KMER when it is set (exits with a message when it is not a number in 1..256)
 *  and returns the limit in force */
inline unsigned apply_max_kmer(const char* program)
{
	const char* e = std::getenv("ABYSS_MAX_KMER");
	if (e && *e) {
		char* end = nullptr;
		const unsigned long v = std::strtoul(e, &end, 10);
		if (*end || v > 0xffffffffUL || abb_set_max_kmer((unsigned)v) != ABB_OK) {
			std::cerr << program << ": ABYSS_MAX_KMER=" << e << ": the largest k-mer size must be a number in 1..256\n";
			std::exit(EXIT_FAILURE);
		}
	}
	return abb_max_kmer();
}

} // namespace host
