// reads.h -- host-side FASTA/FASTQ ingestion for the GPU CLIs.
//
// Mirrors the semantics of the reference reader for the formats the Bloom-DBG stage is fed with
// (DataLayer/FastaReader.cpp:130-421, FOLD_CASE flag; Common/Uncompress.cpp for .gz/.bz2/.xz):
//   '>' FASTA (multi-line) and '@' FASTQ records, '#' comment lines, Casava 1.8 headers with the
//   chastity filter (opt::chastityFilter, default on), trimming of masked (lower-case) ends
//   (opt::trimMasked, default on -- FastaReader.cpp:29), quality trimming (-q) and masking (-Q),
//   quality offset 33/64, case folding; SAM records (FastaReader.cpp:270-327: secondary / QC-fail filters, /1 /2 suffixes,
//   reverse-strand records turned back) and qseq / export records (:328-352).  Colour-space input is not handled.
#pragma once
#include <algorithm>
#include <cctype>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <cerrno>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace host {

struct ReadOpts {
	int chastityFilter = 1;
	int trimMasked = 1;
	int qualityThreshold = 0;
	int internalQThreshold = 0;
	int qualityOffset = 0; // opt::qualityOffset: 0 = the format's own (33 for FASTA / FASTQ / SAM, 64 for qseq / export)
};

/** growable byte buffer that does not zero-fill (std::vector<char>::resize would touch every byte twice) */
struct RawBuf {
	std::unique_ptr<char[]> p;
	size_t n = 0, cap = 0;
	char* data() { return p.get(); }
	const char* data() const { return p.get(); }
	size_t size() const { return n; }
	bool empty() const { return n == 0; }
	void reserve(size_t want)
	{
		if (want <= cap)
			return;
		size_t c = cap ? cap : 4096;
		while (c < want)
			c *= 2;
		std::unique_ptr<char[]> q(new char[c]);
		if (n)
			memcpy(q.get(), p.get(), n);
		p = std::move(q);
		cap = c;
	}
};

/** a batch of reads: concatenated bases + offsets; ids concatenated the same way (for the FASTA comments) */
struct ReadBatch {
	std::vector<char> bases;
	std::vector<uint64_t> offsets{ 0 };
	std::vector<char> id_chars;
	std::vector<uint64_t> id_offsets{ 0 };
	void clear()
	{
		bases.clear();
		offsets.assign(1, 0);
		id_chars.clear();
		id_offsets.assign(1, 0);
	}
	size_t size() const { return offsets.size() - 1; }
	void add(const std::string& id, const std::string& seq)
	{
		id_chars.insert(id_chars.end(), id.begin(), id.end());
		id_offsets.push_back(id_chars.size());
		bases.insert(bases.end(), seq.begin(), seq.end());
		offsets.push_back(bases.size());
	}
	std::string id(size_t i) const { return std::string(id_chars.data() + id_offsets[i], id_chars.data() + id_offsets[i + 1]); }
};

/** the shell command that decompresses `path` to stdout ("" = plain file).  The name goes through /bin/sh (popen),
 *  so a single quote inside it is escaped as '\'' (Common/Uncompress.cpp of the reference builds its commands the
 *  same way and has the same exposure). */
inline std::string decompress_command(const std::string& path)
{
	auto ends = [&](const char* suf) {
		size_t n = strlen(suf);
		return path.size() >= n && path.compare(path.size() - n, n, suf) == 0;
	};
	const char* tool = (ends(".gz") || ends(".z") || ends(".Z")) ? "gunzip -c" : ends(".bz2") ? "bunzip2 -c" : ends(".xz") ? "xzdec -c" : nullptr;
	if (!tool)
		return "";
	std::string q = "'";
	for (char c : path) {
		if (c == '\'')
			q += "'\\''";
		else
			q += c;
	}
	q += "'";
	return std::string(tool) + " " + q;
}
/** close an input opened with fopen / popen; a decompressor that failed (missing tool, corrupt file) is an error, not an
 *  empty input */
inline void close_input(FILE* f, bool is_pipe, const std::string& path)
{
	if (!f || f == stdin)
		return;
	if (!is_pipe) {
		fclose(f);
		return;
	}
	const int st = pclose(f);
	if (st != 0) {
		fprintf(stderr, "error: `%s': the decompressor exited with status %d\n", path.c_str(), st);
		exit(EXIT_FAILURE);
	}
}

class SeqReader {
  public:
	SeqReader(const std::string& path, const ReadOpts& o) : m_path(path), m_opt(o)
	{
		const char* p = path.c_str();
		const std::string cmd = decompress_command(path);
		if (!cmd.empty()) {
			m_f = popen(cmd.c_str(), "r");
			m_pipe = true;
		} else if (path == "-")
			m_f = stdin;
		else
			m_f = fopen(p, "r");
		if (!m_f) {
			fprintf(stderr, "error: `%s': %s\n", p, strerror(errno)); // assert_good (Common/IOUtil.h:14-22)
			exit(EXIT_FAILURE);
		}
		setvbuf(m_f, nullptr, _IONBF, 0); // the reader does its own buffering
		m_buf.reserve(1 << 23);
	}
	/** parse an in-memory piece of a file (BatchStream): `data` holds whole records, numbered from `first_line` */
	SeqReader(RawBuf&& data, const std::string& path, const ReadOpts& o, uint64_t first_line)
	    : m_path(path), m_opt(o), m_eof(true), m_buf(std::move(data)), m_end(m_buf.size()), m_line(first_line)
	{
	}
	/** parse a piece of a memory-mapped file in place (BatchStream): `data[0, n)` holds whole records and stays valid for the
	 *  life of the reader.  line_of = byte offset of the piece in the file: line numbers (only needed for an error message) are
	 *  counted from the start of the file when one has to be printed. */
	SeqReader(const char* data, size_t n, const std::string& path, const ReadOpts& o, uint64_t byte_offset, const char* file_base)
	    : m_path(path), m_opt(o), m_eof(true), m_view(data), m_end(n), m_fileBase(file_base), m_byteOffset(byte_offset)
	{
	}
	/** give the buffer back (BatchStream recycles them: fresh 16 MB allocations page-fault on every use) */
	RawBuf release() { return std::move(m_buf); }
	~SeqReader()
	{
		close_input(m_f, m_pipe, m_path);
	}

	/** the comment (rest of the header line after the id) of the record the last next() returned */
	const std::string& last_comment() const { return m_comment; }

	/** next record; false at end of file */
	bool next(std::string& id, std::string& seq)
	{
		const char* l;
		size_t n;
		for (;;) {
			int c = peek();
			while (c == '#') { // discard comments
				line(l, n);
				c = peek();
			}
			if (c == EOF)
				return false;
			if (c != '>' && c != '@') {
				if (!line_record(id, seq))
					continue; // filtered out (secondary alignment, failed the chastity filter)
				finish_record(seq, m_q, m_lineQualityOffset);
				return true;
			}
			line(l, n); // header
			if (n > 3 && l[0] == '@' && isalpha((unsigned char)l[1]) && isalpha((unsigned char)l[2]) && l[3] == '\t')
				continue; // SAM header line
			const char type = l[0];
			size_t i = 1;
			while (i < n && !isspace((unsigned char)l[i]))
				++i;
			id.assign(l + 1, i - 1);
			while (i < n && isspace((unsigned char)l[i]))
				++i;
			const char* comment = l + i;
			const size_t clen = n - i;
			m_comment.assign(comment, clen);
			bool skip = false;
			if (clen > 3 && comment[1] == ':' && comment[3] == ':') { // Casava: read:chastity:flags:index
				if (m_opt.chastityFilter && comment[2] == 'Y')
					skip = true;
				else if (id.size() > 2 && id[id.size() - 2] != '/') {
					id += '/';
					id += comment[0];
				}
			}
			line(l, n);
			seq.assign(l, n);
			const bool needq = m_opt.qualityThreshold > 0 || m_opt.internalQThreshold > 0;
			size_t qlen = 0;
			bool haveq = false;
			if (type == '>') {
				for (int p = peek(); p != '>' && p != '#' && p != EOF; p = peek()) {
					line(l, n);
					seq.append(l, n);
				}
				m_q.clear();
			} else {
				int plus = peek();
				if (plus != '+') {
					die();
					fprintf(stderr, "expected `+' and saw `%c'\n", plus);
					exit(EXIT_FAILURE);
				}
				line(l, n);
				line(l, n); // quality
				qlen = n;
				haveq = n > 0;
				if (needq)
					m_q.assign(l, n);
			}
			if (skip)
				continue;
			if (seq.empty()) {
				die();
				fprintf(stderr, "sequence with ID `%s' is empty\n", id.c_str());
				exit(EXIT_FAILURE);
			}
			if (haveq && qlen != seq.size()) {
				die();
				fprintf(stderr, "sequence and quality must be the same length near\n%s\n%.*s\n", seq.c_str(), (int)n, l);
				exit(EXIT_FAILURE);
			}
			std::string& q = m_q;
			if (!needq)
				q.clear();
			if (m_opt.trimMasked && (islower((unsigned char)seq.front()) || islower((unsigned char)seq.back()))) { // FastaReader.cpp:236-250
				size_t front = 0, back = seq.size();
				while (front < seq.size() && islower((unsigned char)seq[front]))
					++front;
				while (back > 0 && islower((unsigned char)seq[back - 1]))
					--back;
				if (front >= back) {
					seq.clear();
					q.clear();
				} else {
					seq = seq.substr(front, back - front);
					if (!q.empty())
						q = q.substr(front, back - front);
				}
			}
			for (auto& ch : seq) // FOLD_CASE
				if (ch >= 'a' && ch <= 'z')
					ch = (char)(ch - 32);
			finish_record(seq, q, 33);
			return true;
		}
	}

  private:
	/** the part of FastaReader::read every format shares (FastaReader.cpp:361-407): -q trims the ends, -Q masks inside.  The
	 *  quality offset is the format's (33 for FASTA / FASTQ / SAM, 64 for qseq / export) unless --standard-quality or
	 *  --illumina-quality was given (`if (opt::qualityOffset > 0) qualityOffset = opt::qualityOffset`, :361-362). */
	void finish_record(std::string& seq, std::string& q, int formatOffset) const
	{
		const int qoff = m_opt.qualityOffset > 0 ? m_opt.qualityOffset : formatOffset;
		if (m_opt.qualityThreshold > 0 && !q.empty()) { // FastaReader.cpp:376-394
			const int good = qoff + m_opt.qualityThreshold;
			size_t front = 0, back = q.size();
			while (front < q.size() && (unsigned char)q[front] < good)
				++front;
			while (back > 0 && (unsigned char)q[back - 1] < good)
				--back;
			if (front >= back) {
				seq.erase(1);
				q.erase(1);
			} else {
				seq = seq.substr(front, back - front);
				q = q.substr(front, back - front);
			}
		}
		if (m_opt.internalQThreshold > 0 && !q.empty()) { // FastaReader.cpp:396-407
			const int good = qoff + m_opt.internalQThreshold;
			for (size_t j = 0; j < q.size(); ++j)
				if ((unsigned char)q[j] < good)
					seq[j] = 'N';
		}
	}
	/** isChaste (FastaReader.cpp:94-107) */
	bool is_chaste(const std::string& s, const char* l, size_t n)
	{
		if (s == "1" || s == "Y")
			return true;
		if (s == "0" || s == "N")
			return false;
		die();
		fprintf(stderr, "chastity filter should be one of 0, 1, N or Y\nand saw `%s' near\n%.*s\n", s.c_str(), (int)n, l);
		exit(EXIT_FAILURE);
	}
	/** a record that is one tab-separated line: SAM (FastaReader.cpp:283-327) or qseq / export (:328-352).  Neither is case
	 *  folded nor trimmed of masked ends (the reference only does that for '>' / '@' records).  false = record filtered out. */
	bool line_record(std::string& id, std::string& seq)
	{
		const char* l;
		size_t n;
		line(l, n);
		std::vector<std::string>& f = m_fields;
		f.clear();
		{ // std::getline(in, field, '\t') semantics: a trailing tab does not open an empty last field
			size_t b = 0;
			while (b < n) {
				const char* t = (const char*)memchr(l + b, '\t', n - b);
				const size_t e = t ? (size_t)(t - l) : n;
				f.emplace_back(l + b, e - b);
				b = e + 1;
			}
		}
		std::string& q = m_q;
		if (f.size() >= 11 && (f[9].size() == f[10].size() || f[10] == "*")) { // SAM
			const unsigned long flags = strtoul(f[1].c_str(), nullptr, 0);
			if (flags & 0x100) // FSECONDARY
				return false;
			if (m_opt.chastityFilter && (flags & 0x200)) // FQCFAIL
				return false;
			id = f[0];
			char which = '0';
			switch (flags & 0xc1) { // FPAIRED|FREAD1|FREAD2
			case 0: case 1: break;
			case 0x41: id += "/1"; which = '1'; break;
			case 0x81: id += "/2"; which = '2'; break;
			default:
				die();
				fprintf(stderr, "invalid flags: `%s' near%.*s\n", id.c_str(), (int)n, l);
				exit(EXIT_FAILURE);
			}
			m_comment = (flags & 0x200) ? "0:Y:0:" : "0:N:0:";
			m_comment[0] = which;
			seq = f[9];
			q = f[10];
			if (seq == "*")
				seq.clear();
			if (q == "*")
				q.clear();
			if (flags & 0x10) { // FREVERSE: back to the strand that was sequenced (reverseComplement, Common/Sequence.cpp)
				std::string rcs(seq.rbegin(), seq.rend());
				for (char& ch : rcs)
					ch = complement_char(ch);
				seq.swap(rcs);
				std::reverse(q.begin(), q.end());
			}
			m_lineQualityOffset = 33;
			if (!q.empty() && q.size() != seq.size()) {
				die();
				fprintf(stderr, "sequence and quality must be the same length near\n%s\n%s\n", seq.c_str(), q.c_str());
				exit(EXIT_FAILURE);
			}
			return true;
		}
		if (f.size() == 11 || f.size() == 22) { // qseq or export
			const bool chaste = is_chaste(f.back(), l, n);
			if (m_opt.chastityFilter && !chaste)
				return false;
			id = f[0];
			for (int i = 1; i < 6; ++i)
				if (!f[i].empty()) {
					id += ':';
					id += f[i];
				}
			if (!f[6].empty() && f[6] != "0") {
				id += '#';
				id += f[6];
			}
			id += '/'; // the reverse read is the second read, or the third of an indexed run
			id += f[7] == "3" ? "2" : f[7];
			m_comment = f[7] + (chaste ? ":N:0:" : ":Y:0:");
			seq = f[8];
			q = f[9];
			m_lineQualityOffset = 64;
			if (q.size() != seq.size()) {
				die();
				fprintf(stderr, "sequence and quality must be the same length near\n%s\n%s\n", seq.c_str(), q.c_str());
				exit(EXIT_FAILURE);
			}
			return true;
		}
		die();
		fprintf(stderr, "Expected either `>' or `@' or 11 fields\nand saw `%c' and %zu fields near\n%.*s\n", n ? l[0] : ' ', f.size(), (int)n, l);
		exit(EXIT_FAILURE);
	}
	/** complement of a nucleotide or IUPAC code, case kept (complementBaseChar, Common/Sequence.cpp:24-58) */
	static char complement_char(char c)
	{
		static const char* from = "ACGTMRWSYKVHDBNacgtmrwsykvhdbn.";
		static const char* to = "TGCAKYWSRMBDHVNtgcakywsrmbdhvn.";
		const char* p = c ? strchr(from, c) : nullptr;
		if (!p) {
			fprintf(stderr, "error: unexpected character: `%c'\n", c);
			abort();
		}
		return to[p - from];
	}
	FILE* die()
	{
		uint64_t ln = m_line;
		if (m_fileBase) // a piece of a mapped file: count the lines before it now that the number is needed
			for (const char *q = m_fileBase, *e = m_fileBase + m_byteOffset; q < e && (q = (const char*)memchr(q, '\n', (size_t)(e - q))); ++q)
				++ln;
		fprintf(stderr, "%s:%llu: error: ", m_path.c_str(), (unsigned long long)ln);
		return stderr;
	}
	/** make at least one unread byte available; false at end of input */
	bool fill()
	{
		if (m_pos < m_end)
			return true;
		if (m_eof || !m_f)
			return false;
		m_pos = 0;
		m_end = fread(m_buf.data(), 1, m_buf.cap, m_f);
		if (m_end == 0)
			m_eof = true;
		return m_end > 0;
	}
	const char* dataptr() const { return m_view ? m_view : m_buf.data(); }
	int peek() { return fill() ? (unsigned char)dataptr()[m_pos] : EOF; }
	/** next line without its terminator; the pointer stays valid until the next call */
	bool line(const char*& p, size_t& n)
	{
		if (!fill()) {
			p = dataptr();
			n = 0;
			return false;
		}
		for (;;) {
			const char* nl = (const char*)memchr(dataptr() + m_pos, '\n', m_end - m_pos);
			if (nl) {
				p = dataptr() + m_pos;
				n = (size_t)(nl - p);
				m_pos += n + 1;
				break;
			}
			if (m_eof || !m_f) { // last line without '\n'
				p = dataptr() + m_pos;
				n = m_end - m_pos;
				m_pos = m_end;
				break;
			}
			// the line continues past the buffer: move its head to the front and read more
			const size_t have = m_end - m_pos;
			memmove(m_buf.data(), m_buf.data() + m_pos, have);
			if (have == m_buf.cap) {
				m_buf.n = have;
				m_buf.reserve(m_buf.cap * 2);
			}
			const size_t got = fread(m_buf.data() + have, 1, m_buf.cap - have, m_f);
			m_pos = 0;
			m_end = have + got;
			if (got == 0)
				m_eof = true;
		}
		++m_line;
		while (n > 0 && p[n - 1] == '\r')
			--n;
		return true;
	}
	std::string m_path;
	ReadOpts m_opt;
	FILE* m_f = nullptr;
	bool m_pipe = false, m_eof = false;
	RawBuf m_buf;
	const char* m_view = nullptr; // borrowed data (a piece of a mapped file) instead of m_buf
	size_t m_pos = 0, m_end = 0;
	std::string m_q, m_comment;
	std::vector<std::string> m_fields;
	int m_lineQualityOffset = 33;
	uint64_t m_line = 0;
	const char* m_fileBase = nullptr; // start of the mapping a view belongs to
	uint64_t m_byteOffset = 0;        // of the view in the file
};

/**
 * Reads of a list of files as batches of `batch_reads` reads (the last one shorter), in file order, parsed in the
 * background: one thread reads the files sequentially in pieces of ~16 MB cut at record boundaries, `threads` workers
 * parse the pieces (the semantics are SeqReader's), and next() stitches them together in order -- so the host parses
 * the next batch while the GPU works on the current one (SURVEY 8(f).1: the reference parses under `critical(in)`,
 * BloomIO.h:50-94).  A piece boundary is a line that starts a record: in a file whose first byte is '>' a line
 * starting with '>' (sequence lines cannot); in a file whose first byte is '@' a line starting with '@' whose second
 * successor starts with '+' (a quality line that starts with '@' is followed by a header and a sequence line).
 * SAM, qseq and export files hold one record per line and are cut at any line start.  A file that begins with '#' comment
 * lines is handed to one worker as a single piece.
 */
class BatchStream {
  public:
	BatchStream(const std::vector<std::string>& files, const ReadOpts& o, uint64_t batch_reads, unsigned threads = 0,
	            bool verbose = false, size_t piece_bytes = 16u << 20)
	    : m_files(files), m_opt(o), m_batchReads(batch_reads ? batch_reads : 1), m_verbose(verbose), m_piece(piece_bytes)
	{
		if (threads == 0) {
			threads = std::thread::hardware_concurrency();
			threads = threads > 8 ? 8 : threads ? threads : 1;
		}
		m_maxInFlight = 2 * threads + 2;
		for (unsigned i = 0; i < threads; ++i)
			m_workers.emplace_back([this] { work(); });
		m_reader = std::thread([this] { read_files(); });
		m_stitcher = std::thread([this] { stitch(); });
	}
	~BatchStream()
	{
		{
			std::lock_guard<std::mutex> l(m_mu);
			m_stop = true;
		}
		m_cv.notify_all();
		m_reader.join();
		for (auto& w : m_workers)
			w.join();
		m_stitcher.join();
		if (getenv("ABB_STREAM_STATS"))
			fprintf(stderr, "BatchStream: consumer waited %.3f s, stitched %.3f s; reader read %.3f s, blocked %.3f s\n", m_tWait, m_tAppend,
			        m_tRead, m_tThrottle);
	}
	/** next batch (owned by the stream, valid until the following call), nullptr at the end */
	const ReadBatch* next()
	{
		const auto w0 = std::chrono::steady_clock::now();
		std::unique_lock<std::mutex> l(m_mu);
		if (m_given) {
			m_outFree.push_back(std::move(m_given));
			m_cv.notify_all();
		}
		m_cv.wait(l, [&] { return !m_outQ.empty() || m_stitchDone; });
		m_tWait += std::chrono::duration<double>(std::chrono::steady_clock::now() - w0).count();
		if (m_outQ.empty())
			return nullptr;
		m_given = std::move(m_outQ.front());
		m_outQ.pop_front();
		l.unlock();
		m_cv.notify_all();
		return m_given.get();
	}

  private:
	/** a memory-mapped input file, unmapped when its last piece has been parsed */
	struct Mapping {
		const char* base = nullptr;
		size_t len = 0;
		~Mapping()
		{
			if (base)
				munmap((void*)base, len);
		}
	};
	struct Piece {
		uint64_t seq;
		RawBuf data;
		std::string path;
		uint64_t first_line;
		// pieces of a mapped file are parsed in place: [view, view + view_len) at byte view_off of the file
		std::shared_ptr<Mapping> map;
		const char* view = nullptr;
		size_t view_len = 0;
		uint64_t view_off = 0;
	};
	/** background: cut the parsed pieces, in order, into batches of exactly m_batchReads reads (at most two wait) */
	void stitch()
	{
		for (bool more = true; more;) {
			std::unique_ptr<ReadBatch> out;
			{
				std::unique_lock<std::mutex> l(m_mu);
				m_cv.wait(l, [&] { return m_stop || m_outQ.size() < 2; });
				if (m_stop)
					break;
				if (!m_outFree.empty()) {
					out = std::move(m_outFree.back());
					m_outFree.pop_back();
				}
			}
			if (!out)
				out.reset(new ReadBatch());
			out->clear();
			m_outp = out.get();
			while (out->size() < m_batchReads && out->bases.size() < kBatchBaseBudget) {
				if (!m_cur || m_curPos == m_cur->size()) {
					std::unique_lock<std::mutex> l(m_mu);
					m_cv.wait(l, [&] { return m_stop || m_done.count(m_nextOut) || (m_readerDone && m_nextOut == m_nextSeq); });
					auto it = m_done.find(m_nextOut);
					if (m_stop || it == m_done.end()) {
						more = false; // no more pieces
						break;
					}
					if (m_cur)
						m_free.push_back(std::move(m_cur)); // recycled by the workers: its pages are already mapped
					m_cur = std::move(it->second);
					m_done.erase(it);
					++m_nextOut;
					m_curPos = 0;
					l.unlock();
					m_cv.notify_all();
					continue;
				}
				size_t take = (size_t)std::min<uint64_t>(m_batchReads - out->size(), m_cur->size() - m_curPos);
				// long records (contigs, genomes): stop at the base budget, but always take at least one record
				while (take > 1 && out->bases.size() + (m_cur->offsets[m_curPos + take] - m_cur->offsets[m_curPos]) > kBatchBaseBudget)
					take = (take + 1) / 2;
				if (out->bases.capacity() == 0 && m_cur->size()) { // size a new output batch from the piece's average read: a hint, capped
					const double n = (double)m_cur->size();
					const uint64_t want = m_batchReads;
					const size_t cap = (size_t)1 << 30;
					out->bases.reserve(std::min(cap, (size_t)(1.05 * want * (m_cur->bases.size() / n)) + 4096));
					out->id_chars.reserve(std::min(cap, (size_t)(1.25 * want * (m_cur->id_chars.size() / n)) + 4096));
					out->offsets.reserve(std::min<size_t>(want + 1, cap / 8));
					out->id_offsets.reserve(std::min<size_t>(want + 1, cap / 8));
				}
				const auto a0 = std::chrono::steady_clock::now();
				append(*m_cur, m_curPos, take);
				m_tAppend += std::chrono::duration<double>(std::chrono::steady_clock::now() - a0).count();
				m_curPos += take;
			}
			if (out->size()) {
				std::lock_guard<std::mutex> l(m_mu);
				m_outQ.push_back(std::move(out));
			}
			m_cv.notify_all();
		}
		{
			std::lock_guard<std::mutex> l(m_mu);
			m_stitchDone = true;
		}
		m_cv.notify_all();
	}
	void append(const ReadBatch& b, size_t r0, size_t n)
	{
		ReadBatch& m_out = *m_outp;
		const uint64_t b0 = b.offsets[r0], b1 = b.offsets[r0 + n], i0 = b.id_offsets[r0], i1 = b.id_offsets[r0 + n];
		const uint64_t base = m_out.bases.size(), ibase = m_out.id_chars.size();
		m_out.bases.insert(m_out.bases.end(), b.bases.begin() + b0, b.bases.begin() + b1);
		m_out.id_chars.insert(m_out.id_chars.end(), b.id_chars.begin() + i0, b.id_chars.begin() + i1);
		const size_t at = m_out.offsets.size();
		m_out.offsets.resize(at + n);
		m_out.id_offsets.resize(at + n);
		uint64_t* o = m_out.offsets.data() + at;
		uint64_t* io = m_out.id_offsets.data() + at;
		const uint64_t* so = b.offsets.data() + r0 + 1;
		const uint64_t* sio = b.id_offsets.data() + r0 + 1;
		const uint64_t d = base - b0, di = ibase - i0; // modulo 2^64: fine when base < b0
		for (size_t r = 0; r < n; ++r) {
			o[r] = so[r] + d;
			io[r] = sio[r] + di;
		}
	}
	/** hand a parsed piece to next() */
	void publish(uint64_t seq, std::unique_ptr<ReadBatch> b)
	{
		{
			std::lock_guard<std::mutex> l(m_mu);
			m_done[seq] = std::move(b);
		}
		m_cv.notify_all();
	}
	/** wait until fewer than m_maxInFlight pieces are queued or parsed-but-unconsumed; false when stopping */
	bool throttle()
	{
		const auto t0 = std::chrono::steady_clock::now();
		std::unique_lock<std::mutex> l(m_mu);
		m_cv.wait(l, [&] { return m_stop || m_nextSeq - m_nextOut < m_maxInFlight; });
		m_tThrottle += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
		return !m_stop;
	}
	void work()
	{
		for (;;) {
			Piece pc;
			{
				std::unique_lock<std::mutex> l(m_mu);
				m_cv.wait(l, [&] { return m_stop || !m_tasks.empty() || m_readerDone; });
				if (m_tasks.empty()) {
					if (m_stop || m_readerDone)
						return;
					continue;
				}
				pc = std::move(m_tasks.front());
				m_tasks.pop_front();
			}
			std::unique_ptr<ReadBatch> b;
			{
				std::lock_guard<std::mutex> l(m_mu);
				if (!m_free.empty()) {
					b = std::move(m_free.back());
					m_free.pop_back();
				}
			}
			if (b)
				b->clear();
			else {
				b.reset(new ReadBatch());
				b->bases.reserve(pc.data.size() / 2);
			}
			std::string id, seq;
			if (pc.view) {
				SeqReader in(pc.view, pc.view_len, pc.path, m_opt, pc.view_off, pc.map->base);
				while (in.next(id, seq))
					b->add(id, seq);
				pc.map.reset(); // the last piece of a file unmaps it
			} else {
				SeqReader in(std::move(pc.data), pc.path, m_opt, pc.first_line);
				while (in.next(id, seq))
					b->add(id, seq);
				std::lock_guard<std::mutex> l(m_mu);
				m_freeBufs.push_back(in.release());
			}
			publish(pc.seq, std::move(b));
		}
	}
	/** offset of the last record start in [1, n) of buf, or 0 if there is none */
	static size_t last_record_start(const char* buf, size_t n, char mode)
	{
		size_t end = n;
		for (;;) {
			// start of the last line that begins before `end`
			const char* nl = end > 1 ? (const char*)memrchr(buf, '\n', end - 1) : nullptr;
			if (!nl)
				return 0;
			const size_t ls = (size_t)(nl - buf) + 1;
			if (ls < n && buf[ls] == mode) {
				if (mode == '>')
					return ls;
				// FASTQ: the line after next must be present and start with '+'
				const char* l1 = (const char*)memchr(buf + ls, '\n', n - ls);
				const char* l2 = l1 ? (const char*)memchr(l1 + 1, '\n', n - (size_t)(l1 + 1 - buf)) : nullptr;
				if (l2 && (size_t)(l2 + 1 - buf) < n && l2[1] == '+')
					return ls;
			}
			end = ls; // try the previous line
			if (end <= 1)
				return 0;
		}
	}
	void read_files()
	{
		for (const auto& path : m_files) {
			if (m_verbose)
				fprintf(stderr, "Reading `%s'...\n", path.c_str());
			if (!read_file(path))
				break;
		}
		{
			std::lock_guard<std::mutex> l(m_mu);
			m_readerDone = true;
		}
		m_cv.notify_all();
	}
	RawBuf take_buf()
	{
		std::lock_guard<std::mutex> l(m_mu);
		if (m_freeBufs.empty())
			return RawBuf();
		RawBuf b = std::move(m_freeBufs.back());
		m_freeBufs.pop_back();
		b.n = 0;
		return b;
	}
	static FILE* open_input(const std::string& path, bool* is_pipe)
	{
		const std::string cmd = decompress_command(path);
		*is_pipe = !cmd.empty();
		FILE* f = !cmd.empty() ? popen(cmd.c_str(), "r") : path == "-" ? stdin : fopen(path.c_str(), "r");
		if (!f) {
			fprintf(stderr, "error: `%s': %s\n", path.c_str(), strerror(errno)); // assert_good (Common/IOUtil.h:14-22)
			exit(EXIT_FAILURE);
		}
		setvbuf(f, nullptr, _IONBF, 0);
		return f;
	}
	/** Regular uncompressed files are memory-mapped and cut into pieces without being read by this thread: only the bytes
	 *  around each cut are touched (the search for the last record start runs backwards from the end of the piece), the
	 *  workers fault their pieces in while they parse them, in parallel -- the single reading thread (2.9 GB/s of read() and
	 *  newline counting) was what bounded the ingest.  Returns 0 when the file has to go through read_file_stream (pipes,
	 *  stdin, a '#' comment first, mmap refused), 1 when done, -1 when the stream is being shut down. */
	int read_file_mapped(const std::string& path)
	{
		if (getenv("ABB_NO_MMAP") || path == "-" || !decompress_command(path).empty())
			return 0;
		const int fd = open(path.c_str(), O_RDONLY);
		if (fd < 0)
			return 0; // let the stream path report the error
		struct stat st;
		if (fstat(fd, &st) != 0 || !S_ISREG(st.st_mode) || st.st_size == 0) {
			close(fd);
			return 0;
		}
		void* m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
		close(fd);
		if (m == MAP_FAILED)
			return 0;
		auto map = std::make_shared<Mapping>();
		map->base = (const char*)m;
		map->len = (size_t)st.st_size;
		madvise(m, map->len, MADV_SEQUENTIAL);
		const char* d = map->base;
		const size_t n = map->len;
		const bool sam_header = n > 3 && d[0] == '@' && isalpha((unsigned char)d[1]) && isalpha((unsigned char)d[2]) && d[3] == '\t';
		const char mode = sam_header ? 'L' : (d[0] == '>' || d[0] == '@') ? d[0] : d[0] == '#' ? '?' : 'L';
		if (mode == '?')
			return 0;
		size_t pos = 0;
		while (pos < n) {
			size_t end = std::min(n, pos + m_piece);
			while (end < n) { // cut at the last record start of [pos, end); a record longer than a piece: look further
				size_t cut = 0;
				if (mode == 'L') {
					const char* nl = end - pos > 1 ? (const char*)memrchr(d + pos, '\n', end - pos - 1) : nullptr;
					cut = nl ? (size_t)(nl - (d + pos)) + 1 : 0;
				} else
					cut = last_record_start(d + pos, end - pos, mode);
				if (cut) {
					end = pos + cut;
					break;
				}
				end = std::min(n, end + m_piece);
			}
			if (!throttle())
				return -1;
			Piece pc;
			pc.path = path;
			pc.first_line = 0;
			pc.map = map;
			pc.view = d + pos;
			pc.view_len = end - pos;
			pc.view_off = pos;
			{
				std::lock_guard<std::mutex> l(m_mu);
				pc.seq = m_nextSeq++;
				m_tasks.push_back(std::move(pc));
			}
			m_cv.notify_all();
			pos = end;
		}
		return 1;
	}
	bool read_file(const std::string& path)
	{
		const auto m0 = std::chrono::steady_clock::now();
		const int mapped = read_file_mapped(path);
		if (mapped) {
			m_tRead += std::chrono::duration<double>(std::chrono::steady_clock::now() - m0).count();
			return mapped > 0;
		}
		bool is_pipe = false;
		FILE* f = open_input(path, &is_pipe);
		const auto r0 = std::chrono::steady_clock::now();
		RawBuf carry = take_buf(); // bytes read but not yet handed out
		uint64_t line = 0;
		char mode = 0;
		bool eof = false, ok = true;
		while (ok && !(eof && carry.empty())) {
			RawBuf buf(std::move(carry));
			carry = take_buf();
			size_t want = buf.n + m_piece;
			for (;;) { // read until the piece holds a record boundary (or the file ends)
				buf.reserve(want);
				while (!eof && buf.n < want) {
					const size_t got = fread(buf.data() + buf.n, 1, want - buf.n, f);
					if (got == 0)
						eof = true;
					buf.n += got;
				}
				if (!mode && buf.n) {
					const char* d = buf.data();
					const bool sam_header = buf.n > 3 && d[0] == '@' && isalpha((unsigned char)d[1]) && isalpha((unsigned char)d[2]) && d[3] == '\t';
					// SAM / qseq / export: one record per line, a piece may end at any line; '#' comments first: serial
					mode = sam_header ? 'L' : (d[0] == '>' || d[0] == '@') ? d[0] : d[0] == '#' ? '?' : 'L';
				}
				if (eof || mode == '?')
					break;
				size_t cut = 0;
				if (mode == 'L') {
					const char* nl = buf.n > 1 ? (const char*)memrchr(buf.data(), '\n', buf.n - 1) : nullptr;
					cut = nl ? (size_t)(nl - buf.data()) + 1 : 0;
				} else
					cut = last_record_start(buf.data(), buf.n, mode);
				if (cut) {
					carry.reserve(buf.n - cut + m_piece);
					memcpy(carry.data(), buf.data() + cut, buf.n - cut);
					carry.n = buf.n - cut;
					buf.n = cut;
					break;
				}
				want += m_piece; // one record longer than the piece: keep reading
			}
			if (mode == '?') {
				// not a plain FASTA/FASTQ start: one piece holds the rest of the file, i.e. it is parsed serially
				while (!eof) {
					buf.reserve(buf.n + m_piece);
					const size_t got = fread(buf.data() + buf.n, 1, m_piece, f);
					buf.n += got;
					if (got == 0)
						eof = true;
				}
			}
			if (buf.empty())
				break;
			uint64_t nl = 0;
			for (const char *q = buf.data(), *e = q + buf.size(); q < e && (q = (const char*)memchr(q, '\n', (size_t)(e - q))); ++q)
				++nl;
			if (!throttle()) {
				ok = false;
				break;
			}
			Piece pc;
			pc.data = std::move(buf);
			pc.path = path;
			pc.first_line = line;
			line += nl;
			{
				std::lock_guard<std::mutex> l(m_mu);
				pc.seq = m_nextSeq++;
				m_tasks.push_back(std::move(pc));
			}
			m_cv.notify_all();
		}
		close_input(f, is_pipe, path);
		m_tRead += std::chrono::duration<double>(std::chrono::steady_clock::now() - r0).count();
		return ok;
	}

	static constexpr size_t kBatchBaseBudget = (size_t)3 << 29; // 1.5 G bases per batch at most
	std::vector<std::string> m_files;
	ReadOpts m_opt;
	uint64_t m_batchReads;
	bool m_verbose;
	size_t m_piece;
	uint64_t m_maxInFlight = 4;
	std::mutex m_mu;
	std::condition_variable m_cv;
	std::deque<Piece> m_tasks;
	std::map<uint64_t, std::unique_ptr<ReadBatch>> m_done;
	uint64_t m_nextSeq = 0, m_nextOut = 0;
	bool m_readerDone = false, m_stop = false;
	std::vector<std::thread> m_workers;
	std::thread m_reader;
	std::unique_ptr<ReadBatch> m_cur;
	std::vector<std::unique_ptr<ReadBatch>> m_free;
	std::vector<RawBuf> m_freeBufs;
	size_t m_curPos = 0;
	ReadBatch* m_outp = nullptr;                      // batch the stitcher is filling
	std::deque<std::unique_ptr<ReadBatch>> m_outQ;    // finished batches
	std::vector<std::unique_ptr<ReadBatch>> m_outFree;
	std::unique_ptr<ReadBatch> m_given;               // the batch the caller holds
	bool m_stitchDone = false;
	std::thread m_stitcher;
	double m_tWait = 0, m_tAppend = 0, m_tRead = 0, m_tThrottle = 0;
};

/** SIToBytes (Common/StringUtil.h:181-219): number with optional k/M/G suffix (powers of 1024) */
inline bool si_to_bytes(const char* s, uint64_t* out)
{
	char* end = nullptr;
	double v = strtod(s, &end);
	if (end == s)
		return false;
	if (*end) {
		if (end[1])
			return false;
		switch (tolower((unsigned char)*end)) {
		case 'k': v *= (double)(1ULL << 10); break;
		case 'm': v *= (double)(1ULL << 20); break;
		case 'g': v *= (double)(1ULL << 30); break;
		default: return false;
		}
	}
	*out = (uint64_t)std::ceil(v);
	return true;
}

} // namespace host
