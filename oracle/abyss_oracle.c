/*
 * oracle/abyss_oracle.c -- TEST INFRASTRUCTURE ONLY (see abyss_oracle.h).
 *
 * Sequential restatement of the reference's hashing and Bloom-filter arithmetic for the
 * abyss-bloom-dbg path.  Written from the reference's behaviour, citing file:line under
 * the reference source tree; validated against the compiled reference (tests/test_oracle_*.py).
 */
#include "abyss_oracle.h"
#include <ctype.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * ntHash (vendor/nthash/nthash.hpp)
 * ---------------------------------------------------------------------------------------- */

#define SEED_A 0x3c8bfbb395c60474ULL /* nthash.hpp:25 */
#define SEED_C 0x3193c18562a02b4cULL /* :26 */
#define SEED_G 0x20323ed082572324ULL /* :27 */
#define SEED_T 0x295549f54be24456ULL /* :28 */
#define MULTI_SEED 0x90b45d39fb6da1faULL /* :22 */
#define MULTI_SHIFT 27 /* :19 */

/* seedTab (nthash.hpp:31-64): only A/C/G/T/U (either case) and the 3-bit complement codes
 * 1,3,4,5,7 carry a non-zero seed; everything else (N included) hashes as 0. */
uint64_t abo_seed(unsigned char c)
{
	switch (c) {
	case 'A': case 'a': case 4: case 5: return SEED_A;
	case 'C': case 'c': case 7: return SEED_C;
	case 'G': case 'g': case 3: return SEED_G;
	case 'T': case 't': case 'U': case 'u': case 1: return SEED_T;
	default: return 0;
	}
}

/* complement seed: the reference indexes seedTab with (c & cpOff), cpOff = 7 (nthash.hpp:16,235) */
static uint64_t comp_seed(unsigned char c) { return abo_seed(c & 7); }

/* rol1 + swapbits033 (nthash.hpp:196-198,208-211): the low 33 bits and the high 31 bits
 * each rotate left by one inside their own field. */
uint64_t abo_srol(uint64_t v)
{
	uint64_t r = (v << 1) | (v >> 63);
	uint64_t x = (r ^ (r >> 33)) & 1;
	return r ^ (x | (x << 33));
}

/* ror1 + swapbits3263 (nthash.hpp:201-203,214-217): inverse of abo_srol */
uint64_t abo_sror(uint64_t v)
{
	uint64_t r = (v >> 1) | (v << 63);
	uint64_t x = ((r >> 32) ^ (r >> 63)) & 1;
	return r ^ ((x << 32) | (x << 63));
}

/* value of the msTab31l[c][n%31] | msTab33r[c][n%33] tables (nthash.hpp:66-194): the seed
 * split-rotated n times.  Computed, not tabulated. */
uint64_t abo_srol_n(uint64_t x, unsigned n)
{
	uint64_t lo = x & 0x1FFFFFFFFULL, hi = x >> 33;
	unsigned a = n % 33, b = n % 31;
	if (a)
		lo = ((lo << a) | (lo >> (33 - a))) & 0x1FFFFFFFFULL;
	if (b)
		hi = ((hi << b) | (hi >> (31 - b))) & 0x7FFFFFFFULL;
	return (hi << 33) | lo;
}

/* NTF64 + NTR64 of a whole k-mer (nthash.hpp:220-239) */
void abo_base_hash(const char* kmer, unsigned k, uint64_t* fh, uint64_t* rh)
{
	uint64_t f = 0, r = 0;
	for (unsigned i = 0; i < k; ++i) {
		f = abo_srol(f) ^ abo_seed((unsigned char)kmer[i]);
		r = abo_srol(r) ^ comp_seed((unsigned char)kmer[k - 1 - i]);
	}
	*fh = f;
	*rh = r;
}

/* NTF64/NTR64 sliding one base to the right (nthash.hpp:242-257) */
void abo_roll_right(uint64_t* fh, uint64_t* rh, unsigned k, unsigned char out, unsigned char in)
{
	*fh = abo_srol(*fh) ^ abo_seed(in) ^ abo_srol_n(abo_seed(out), k);
	*rh = abo_sror(*rh ^ abo_srol_n(comp_seed(in), k) ^ comp_seed(out));
}

/* NTF64L/NTR64L sliding one base to the left (nthash.hpp:282-297) */
void abo_roll_left(uint64_t* fh, uint64_t* rh, unsigned k, unsigned char out, unsigned char in)
{
	*fh = abo_sror(*fh ^ abo_srol_n(abo_seed(in), k) ^ abo_seed(out));
	*rh = abo_srol(*rh) ^ comp_seed(in) ^ abo_srol_n(comp_seed(out), k);
}

/* maskHash (nthash.hpp:537-547): XOR the contribution of every non-'1' seed position back
 * out of both strands, then take the smaller. */
uint64_t abo_mask_hash(uint64_t fh, uint64_t rh, const char* mask, const char* kmer, unsigned k)
{
	for (unsigned i = 0; i < k; ++i)
		if (mask[i] != '1') {
			fh ^= abo_srol_n(abo_seed((unsigned char)kmer[i]), k - 1 - i);
			rh ^= abo_srol_n(comp_seed((unsigned char)kmer[i]), i);
		}
	return rh < fh ? rh : fh;
}

/* NTE64 (nthash.hpp:337-342); note C precedence: i ^ (k * multiSeed) */
uint64_t abo_extra_hash(uint64_t h0, unsigned k, unsigned i)
{
	uint64_t t = h0 * ((uint64_t)i ^ ((uint64_t)k * MULTI_SEED));
	return t ^ (t >> MULTI_SHIFT);
}

/* ------------------------------------------------------------------------------------------
 * RollingHashIterator (BloomDBG/RollingHashIterator.h) + RollingHash (BloomDBG/RollingHash.h)
 * ---------------------------------------------------------------------------------------- */

static int is_acgt(char c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }

size_t abo_hash_seq(const char* seq_in, size_t len, unsigned k, unsigned H, const char* mask,
                    uint64_t* out_h, uint32_t* out_pos)
{
	if (mask && !mask[0])
		mask = NULL;
	if (len < k || k == 0) /* RollingHashIterator.h:37-40 */
		return 0;
	/* init(): private upper-cased copy (RollingHashIterator.h:131) */
	char* seq = (char*)malloc(len + 1);
	for (size_t i = 0; i < len; ++i)
		seq[i] = (char)toupper((unsigned char)seq_in[i]);
	seq[len] = 0;

	size_t n = 0, pos = 0;
	int roll = 0; /* m_rollNextHash */
	uint64_t fh = 0, rh = 0;
	while (pos + k <= len) {
		/* a window is bad if a non-ACGT char sits on a position the seed cares about
		 * (RollingHashIterator.h:46-73) */
		int bad = 0;
		size_t firstBad = 0;
		for (size_t j = 0; j < k; ++j)
			if (!is_acgt(seq[pos + j]) && (!mask || mask[j] == '1')) {
				bad = 1;
				firstBad = pos + j;
				break;
			}
		if (bad) {
			roll = 0;
			/* without a seed the iterator jumps past the first bad char; with one it
			 * advances by one (:52-56 vs :69-72) -- same set of k-mers either way */
			pos = mask ? pos + 1 : firstBad + 1;
			continue;
		}
		uint64_t h0;
		if (!roll) { /* RollingHash::reset (RollingHash.h:69-80) */
			abo_base_hash(seq + pos, k, &fh, &rh);
			roll = 1;
		} else /* RollingHash::rollRight (RollingHash.h:88-102) */
			abo_roll_right(&fh, &rh, k, (unsigned char)seq[pos - 1], (unsigned char)seq[pos + k - 1]);
		h0 = rh < fh ? rh : fh; /* canonicalHash (RollingHash.h:28-31) */
		if (mask)
			h0 = abo_mask_hash(fh, rh, mask, seq + pos, k);
		if (out_h) { /* getHashes (RollingHash.h:143-148) */
			out_h[n * H] = h0;
			for (unsigned i = 1; i < H; ++i)
				out_h[n * H + i] = abo_extra_hash(h0, k, i);
		}
		if (out_pos)
			out_pos[n] = (uint32_t)pos;
		++n;
		++pos;
	}
	free(seq);
	return n;
}

/* ------------------------------------------------------------------------------------------
 * CountingBloomFilter<uint8_t> (vendor/btl_bloomfilter/CountingBloomFilter.hpp)
 * ---------------------------------------------------------------------------------------- */

uint8_t abo_cbf_min(const uint8_t* c, uint64_t m, const uint64_t* h, unsigned H)
{
	uint8_t mn = c[h[0] % m];
	for (unsigned i = 1; i < H; ++i) {
		uint8_t v = c[h[i] % m];
		if (v < mn)
			mn = v;
	}
	return mn;
}

/* incrementMin, single-threaded: every counter equal to the minimum gets +1, a saturated
 * minimum (255) is left alone, and a position that occurs twice in h[] is bumped once
 * because the second compare-and-swap sees the new value (CountingBloomFilter.hpp:138-162). */
void abo_cbf_insert(uint8_t* c, uint64_t m, const uint64_t* h, unsigned H)
{
	uint8_t mn = abo_cbf_min(c, m, h, H);
	uint8_t nv = (uint8_t)(mn + 1);
	if (mn > nv)
		return;
	for (unsigned i = 0; i < H; ++i) {
		uint64_t p = h[i] % m;
		if (c[p] == mn)
			c[p] = nv;
	}
}

#define ABO_MAX_HASHES 32 /* configure.ac:151-159 MAX_HASHES */

size_t abo_cbf_load_seq(uint8_t* c, uint64_t m, const char* seq, size_t len, unsigned k, unsigned H,
                        const char* mask)
{
	if (len < k)
		return 0;
	size_t cap = len - k + 1;
	uint64_t* h = (uint64_t*)malloc(cap * H * sizeof(uint64_t));
	size_t n = abo_hash_seq(seq, len, k, H, mask, h, NULL);
	for (size_t i = 0; i < n; ++i)
		abo_cbf_insert(c, m, h + i * H, H);
	free(h);
	return n;
}

uint64_t abo_cbf_popcount(const uint8_t* c, uint64_t m, unsigned threshold)
{
	uint64_t n = 0;
	for (uint64_t i = 0; i < m; ++i)
		n += threshold == 0 ? (c[i] != 0) : (c[i] >= threshold);
	return n;
}

/* ------------------------------------------------------------------------------------------
 * BloomFilter (vendor/btl_bloomfilter/BloomFilter.hpp): bit n lives in byte n/8, mask 1<<(n%8)
 * ---------------------------------------------------------------------------------------- */

void abo_bf_insert(uint8_t* bits, uint64_t mbits, const uint64_t* h, unsigned H)
{
	for (unsigned i = 0; i < H; ++i) {
		uint64_t n = h[i] % mbits;
		bits[n >> 3] |= (uint8_t)(1u << (n & 7));
	}
}

int abo_bf_contains(const uint8_t* bits, uint64_t mbits, const uint64_t* h, unsigned H)
{
	for (unsigned i = 0; i < H; ++i) {
		uint64_t n = h[i] % mbits;
		if (!(bits[n >> 3] & (1u << (n & 7))))
			return 0;
	}
	return 1;
}

size_t abo_bf_load_seq(uint8_t* bits, uint64_t mbits, const char* seq, size_t len, unsigned k,
                       unsigned H, const char* mask)
{
	if (len < k)
		return 0;
	size_t cap = len - k + 1;
	uint64_t* h = (uint64_t*)malloc(cap * H * sizeof(uint64_t));
	size_t n = abo_hash_seq(seq, len, k, H, mask, h, NULL);
	for (size_t i = 0; i < n; ++i)
		abo_bf_insert(bits, mbits, h + i * H, H);
	free(h);
	return n;
}

/* ------------------------------------------------------------------------------------------
 * HashAgnosticCascadingBloom (Bloom/HashAgnosticCascadingBloom.h:112-133): insert into the
 * first level that does not already contain the element; stop there.
 * ---------------------------------------------------------------------------------------- */

void abo_casc_insert(uint8_t* levels, uint64_t mbits, unsigned L, const uint64_t* h, unsigned H)
{
	for (unsigned l = 0; l < L; ++l) {
		uint8_t* bits = levels + (size_t)l * (mbits / 8);
		if (!abo_bf_contains(bits, mbits, h, H)) {
			abo_bf_insert(bits, mbits, h, H);
			break;
		}
	}
}

size_t abo_casc_load_seq(uint8_t* levels, uint64_t mbits, unsigned L, const char* seq, size_t len,
                         unsigned k, unsigned H, const char* mask)
{
	if (len < k)
		return 0;
	size_t cap = len - k + 1;
	uint64_t* h = (uint64_t*)malloc(cap * H * sizeof(uint64_t));
	size_t n = abo_hash_seq(seq, len, k, H, mask, h, NULL);
	for (size_t i = 0; i < n; ++i)
		abo_casc_insert(levels, mbits, L, h + i * H, H);
	free(h);
	return n;
}

/* ------------------------------------------------------------------------------------------
 * counters = roundUpToMultiple(round(B / 1.125), 64)   (BloomDBG/bloom-dbg.cc:359-367)
 * ---------------------------------------------------------------------------------------- */
uint64_t abo_counters_for_budget(uint64_t bloom_size_bytes)
{
	double x = (double)bloom_size_bytes / 1.125;
	uint64_t r = (uint64_t)(x + 0.5); /* round() of a positive double */
	uint64_t rem = r % 64;
	return rem ? r + 64 - rem : r;
}
