// trim.h -- the host half of `abyss-bloom trim` (Bloom/bloom.cc:1292-1382): the branch length threshold and the record writer.
// Shared by abyss_bloom.cc and the CPU harness tests/host_trim.
#pragma once
#include <cmath>
#include <cstdint>
#include <string>

namespace host {

/** minBranchLen = (size_t)ceil(log(0.0001) / log(FPR)), FPR = popcount / size (bloom.cc:1324-1327).  An empty filter gives
 *  0.  A full filter (FPR = 1) makes the reference convert -inf to size_t, which is undefined: false, and the caller refuses. */
inline bool trim_min_branch_len(uint64_t popcount, uint64_t size, uint64_t* out)
{
	if (popcount >= size)
		return false;
	const double falseBranchProbability = 0.0001;
	*out = (uint64_t)std::ceil(std::log(falseBranchProbability) / std::log((double)popcount / (double)size));
	return true;
}

/** What trim() prints for one record: the record itself when it is shorter than k, nothing when the two trims meet, else
 *  the bases and qualities [left, len - 1 - right] (operator<<(FastqRecord), DataLayer/FastaReader.h:186-196: the FASTA
 *  form when there is no quality string).  left / right are calcLeftTrim of the read and of its reverse complement, taken
 *  as the reference's `unsigned`.  Returns whether the record counts towards the "Processed N reads" progress line. */
inline bool append_trimmed_record(std::string& out, const char* id, size_t id_len, const char* comment, size_t comment_len, const char* seq,
                                  size_t len, const char* qual, size_t qual_len, unsigned k, uint32_t left, uint32_t right)
{
	size_t start = 0, n = len;
	bool trimmed = false;
	if (len >= k) {
		const unsigned startPos = left, endPos = (unsigned)len - 1 - right;
		if (endPos < startPos)
			return false;
		start = startPos;
		n = endPos - startPos + 1;
		trimmed = true;
	}
	// std::string::substr(pos, n): pos past the end throws in the reference; the trims never exceed len here because
	// start <= endPos <= len - 1.  A quality string is as long as its sequence (the reader checks it).
	out += qual_len ? '@' : '>';
	out.append(id, id_len);
	if (comment_len) {
		out += ' ';
		out.append(comment, comment_len);
	}
	out += '\n';
	out.append(seq + start, n);
	out += '\n';
	if (qual_len) {
		out += "+\n";
		out.append(qual + start, n);
		out += '\n';
	}
	return trimmed;
}

} // namespace host
