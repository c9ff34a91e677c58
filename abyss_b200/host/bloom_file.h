// bloom_file.h -- the on-disk contract of the reference's Bloom filters (SURVEY.md section 8b):
// a TOML-like header ([MAGIC]\n\tKey = value ... [HeaderEnd]\n) followed by the raw array.
//   [BTLCountingBloomFilter_v1]  vendor/btl_bloomfilter/CountingBloomFilter.hpp:262-379
//   [BTLBloomFilter_v1]          vendor/btl_bloomfilter/BloomFilter.hpp:104-163,261-294
// Key order follows what the reference writes (cpptoml unordered_map iteration order under
// libstdc++), so files are byte-identical; loaders parse by key.
#pragma once
#include <cerrno>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

namespace host {

struct BloomHeader {
	uint64_t size = 0, sizeInBytes = 0;
	unsigned hashNum = 0, kmerSize = 0, bitsPerCounter = 8;
};

inline std::map<std::string, std::string> read_header(std::istream& in, const std::string& magic, const std::string& path)
{
	std::string line;
	std::getline(in, line);
	if (line != "[" + magic + "]") {
		std::cerr << "ERROR: magic string does not match (likely version mismatch)\n"
		          << "Your magic string:                " << line << "\n"
		          << "CountingBloomFilter magic string: [" << magic << "]" << std::endl;
		exit(EXIT_FAILURE);
	}
	std::map<std::string, std::string> kv;
	bool end = false;
	while (std::getline(in, line)) {
		if (line == "[HeaderEnd]") {
			end = true;
			break;
		}
		size_t eq = line.find('=');
		if (eq == std::string::npos)
			continue;
		auto trim = [](std::string s) {
			size_t a = s.find_first_not_of(" \t"), b = s.find_last_not_of(" \t");
			return a == std::string::npos ? std::string() : s.substr(a, b - a + 1);
		};
		kv[trim(line.substr(0, eq))] = trim(line.substr(eq + 1));
	}
	if (!end) {
		std::cerr << "ERROR: pre-built bloom filter does not have the correct header end." << std::endl;
		exit(EXIT_FAILURE);
	}
	(void)path;
	return kv;
}

inline void read_counting_bloom(const std::string& path, BloomHeader& h, std::vector<uint8_t>& raw)
{
	std::ifstream in(path, std::ios::binary);
	if (!in) {
		std::cerr << "error: `" << path << "': cannot open\n";
		exit(EXIT_FAILURE);
	}
	auto kv = read_header(in, "BTLCountingBloomFilter_v1", path);
	h.size = strtoull(kv["BloomFilterSize"].c_str(), nullptr, 10);
	h.hashNum = (unsigned)strtoul(kv["HashNum"].c_str(), nullptr, 10);
	h.kmerSize = (unsigned)strtoul(kv["KmerSize"].c_str(), nullptr, 10);
	h.sizeInBytes = strtoull(kv["BloomFilterSizeInBytes"].c_str(), nullptr, 10);
	h.bitsPerCounter = (unsigned)strtoul(kv["BitsPerCounter"].c_str(), nullptr, 10);
	raw.resize(h.sizeInBytes);
	in.read(reinterpret_cast<char*>(raw.data()), (std::streamsize)raw.size());
	if (!in) {
		std::cerr << "error: `" << path << "': truncated filter\n";
		exit(EXIT_FAILURE);
	}
}

/** BloomFilter::loadFilter (BloomFilter.hpp:104-163): header + raw bit array */
inline void read_bit_bloom(const std::string& path, BloomHeader& h, std::vector<uint8_t>& raw)
{
	std::ifstream in(path, std::ios::binary);
	if (!in) {
		std::cerr << "error: `" << path << "': cannot open\n";
		exit(EXIT_FAILURE);
	}
	auto kv = read_header(in, "BTLBloomFilter_v1", path);
	h.size = strtoull(kv["BloomFilterSize"].c_str(), nullptr, 10);
	h.hashNum = (unsigned)strtoul(kv["HashNum"].c_str(), nullptr, 10);
	h.kmerSize = (unsigned)strtoul(kv["KmerSize"].c_str(), nullptr, 10);
	h.sizeInBytes = strtoull(kv["BloomFilterSizeInBytes"].c_str(), nullptr, 10);
	h.bitsPerCounter = 1;
	raw.resize(h.sizeInBytes);
	in.read(reinterpret_cast<char*>(raw.data()), (std::streamsize)raw.size());
	if (!in) {
		std::cerr << "error: `" << path << "': truncated filter\n";
		exit(EXIT_FAILURE);
	}
}

/** CountingBloomFilter::storeHeader + operator<< (CountingBloomFilter.hpp:341-379) */
inline void write_counting_bloom(std::ostream& out, const BloomHeader& h, const std::vector<uint8_t>& raw)
{
	out << "[BTLCountingBloomFilter_v1]\n"
	    << "\tBloomFilterSize = " << h.size << "\n"
	    << "\tHashNum = " << h.hashNum << "\n"
	    << "\tKmerSize = " << h.kmerSize << "\n"
	    << "\tBloomFilterSizeInBytes = " << h.sizeInBytes << "\n"
	    << "\tBitsPerCounter = " << h.bitsPerCounter << "\n"
	    << "[HeaderEnd]\n";
	out.write(reinterpret_cast<const char*>(raw.data()), (std::streamsize)raw.size());
}

/** BloomFilter::writeHeader + operator<< (BloomFilter.hpp:261-294); dFPR/nEntry/Entry are 0 for
 *  filters built by abyss-bloom */
inline void write_bit_bloom(std::ostream& out, uint64_t sizeBits, unsigned hashNum, unsigned kmerSize, const std::vector<uint8_t>& raw)
{
	out << "[BTLBloomFilter_v1]\n"
	    << "\tnEntry = 0\n"
	    << "\tdFPR = 0.0000000000000000\n"
	    << "\tEntry = 0\n"
	    << "\tBloomFilterSizeInBytes = " << raw.size() << "\n"
	    << "\tBloomFilterSize = " << sizeBits << "\n"
	    << "\tHashNum = " << hashNum << "\n"
	    << "\tKmerSize = " << kmerSize << "\n"
	    << "[HeaderEnd]\n";
	out.write(reinterpret_cast<const char*>(raw.data()), (std::streamsize)raw.size());
}

/** The Konnector filter file (Bloom/Bloom.h:136-191): a text header "5\n{k}\n{full}\t{start}\t{end}\n{seed}\n" and the bits
 *  [start, end] of a filter of `full` bits, (end - start + 1 + 7) / 8 bytes, bit i in byte i/8 under mask 0x80 >> i%8. */
struct KonnectorHeader {
	unsigned version = 5, k = 0;
	uint64_t full = 0, start = 0, end = 0, seed = 0;
	uint64_t bits() const { return end - start + 1; }
	uint64_t bytes() const { return (bits() + 7) / 8; }
};

/** true if the first line of the file is a Konnector header ("5"), false for anything else (the BTL formats) */
inline bool is_konnector_bloom(const std::string& path)
{
	std::ifstream in(path, std::ios::binary);
	std::string line;
	return in && std::getline(in, line) && !line.empty() && line.find_first_not_of("0123456789") == std::string::npos;
}

/** Bloom::readHeader with its messages and exits; k = 0 skips the k check */
inline KonnectorHeader read_konnector_header(std::istream& in, unsigned k)
{
	KonnectorHeader h;
	char c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0;
	in >> h.version;
	in.get(c1);
	if (h.version != 5) {
		std::cerr << "error: bloom filter version (`" << h.version << "'), does not match version required by this program (`5').\n";
		exit(EXIT_FAILURE);
	}
	in >> h.k;
	in.get(c2);
	if (k != 0 && h.k != k) {
		std::cerr << "error: this program must be run with the same kmer size as the bloom filter being loaded (k=" << h.k << ").\n";
		exit(EXIT_FAILURE);
	}
	in >> h.full;
	in.get(c3);
	in >> h.start;
	in.get(c4);
	in >> h.end;
	in.get(c5);
	in >> h.seed;
	char c6 = 0;
	in.get(c6);
	if (!in || c1 != '\n' || c2 != '\n' || c3 != '\t' || c4 != '\t' || c5 != '\n' || c6 != '\n' || h.start >= h.full || h.end >= h.full ||
	    h.start > h.end) {
		std::cerr << "error: malformed Konnector Bloom filter header\n";
		exit(EXIT_FAILURE);
	}
	return h;
}

/** the header and the raw bytes of a Konnector filter file */
inline KonnectorHeader read_konnector_bloom(const std::string& path, unsigned k, std::vector<uint8_t>& raw)
{
	std::ifstream in(path, std::ios::binary);
	if (!in) {
		std::cerr << "error: `" << path << "': " << strerror(errno) << "\n";
		exit(EXIT_FAILURE);
	}
	KonnectorHeader h = read_konnector_header(in, k);
	raw.resize(h.bytes());
	in.read(reinterpret_cast<char*>(raw.data()), (std::streamsize)raw.size());
	if (!in) {
		std::cerr << "error: `" << path << "': truncated filter\n";
		exit(EXIT_FAILURE);
	}
	return h;
}

inline void write_konnector_bloom(std::ostream& out, const KonnectorHeader& h, const uint8_t* raw)
{
	out << 5 << '\n' << h.k << '\n' << h.full << '\t' << h.start << '\t' << h.end << '\n' << h.seed << '\n';
	out.write(reinterpret_cast<const char*>(raw), (std::streamsize)h.bytes());
}

} // namespace host
