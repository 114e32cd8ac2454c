// ingest.cpp -- see ingest.h. BGZF blocks (or pieces of a plain SAM file) are copied into chunks in parallel on the host and the header (BAM, or SAM's @ lines) is read here; everything the reference's record loop does
// runs on the device (csrc/records.cu), and so does the fragment table (csrc/fragtable.cu). An input that is not a regular file (a pipe: STAR ... | arriba
// -x /dev/stdin) is read in sequence into the chunks; its BGZF blocks go to the device as they were read, and the device assembles the inflated chunk.
#include "ingest.h"
#include "../../../include/arriba_b200.h"
#include <set>
#include "../records_hd.h"
#include <zlib.h>
#include <fcntl.h>
#include <errno.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <stdexcept>
#include <thread>
#include <mutex>

namespace arb { namespace host {

// ------------------------------------------------------------------------------------------- recycled host blocks (ingest.h)
namespace {
struct host_block_pool {
	std::mutex lock; std::vector<std::pair<size_t, void*> > free_blocks; size_t held;
	std::set<void*> from_backend; // blocks obtained from the backend (page-locked memory in the CUDA library): they go back through it
	host_block_pool(): held(0) {}
};
void* (*g_backend_alloc)(size_t) = NULL; void (*g_backend_free)(void*) = NULL;
host_block_pool& block_pool() { static host_block_pool* p = new host_block_pool(); return *p; } // never destroyed: blocks may be returned during static destruction
}
void* host_block_get(size_t bytes, size_t& granted) {
	granted = bytes;
	host_block_pool& pool = block_pool();
	{
		std::lock_guard<std::mutex> g(pool.lock);
		for (size_t k = pool.free_blocks.size(); k-- > 0; ) if (pool.free_blocks[k].first == bytes) {
			void* p = pool.free_blocks[k].second; pool.free_blocks[k] = pool.free_blocks.back(); pool.free_blocks.pop_back(); pool.held -= bytes; return p;
		}
	}
	if (g_backend_alloc) { // page-locked: the columns built in such blocks are copied to the device asynchronously at full PCIe speed, and the blocks are recycled
		void* p = g_backend_alloc(bytes);
		if (p) { std::lock_guard<std::mutex> g(pool.lock); pool.from_backend.insert(p); return p; }
	}
	return malloc(bytes);
}
static void release_block(host_block_pool& pool, void* p) { // pool.lock held
	std::set<void*>::iterator it = pool.from_backend.find(p);
	if (it != pool.from_backend.end()) { pool.from_backend.erase(it); g_backend_free(p); } else free(p);
}
void host_block_put(void* p, size_t granted) {
	host_block_pool& pool = block_pool();
	std::lock_guard<std::mutex> g(pool.lock);
	if (pool.held + granted <= ((size_t) 64 << 30)) { pool.free_blocks.push_back(std::make_pair(granted, p)); pool.held += granted; return; }
	release_block(pool, p);
}
void host_block_trim() {
	host_block_pool& pool = block_pool();
	std::lock_guard<std::mutex> g(pool.lock);
	for (size_t k = 0; k < pool.free_blocks.size(); ++k) release_block(pool, pool.free_blocks[k].second);
	pool.free_blocks.clear(); pool.held = 0;
}
void set_host_block_backend(void* (*alloc)(size_t), void (*release)(void*)) { g_backend_alloc = alloc; g_backend_free = release; }

static void fail(const std::string& m) { throw std::runtime_error(m); }
// Tables of hundreds of megabytes that are visited all over (the coverage windows): on 4 KiB pages nearly every visit also misses
// the TLB. Where the kernel offers transparent huge pages on request (THP "madvise"), ask for them; elsewhere the call does nothing.
static void advise_huge(const void* p, size_t bytes) {
#ifdef MADV_HUGEPAGE
	const size_t huge = (size_t) 2 << 20;
	if (p == NULL || bytes < 4 * huge) return;
	const uintptr_t lo = ((uintptr_t) p + huge - 1) & ~(uintptr_t) (huge - 1), hi = ((uintptr_t) p + bytes) & ~(uintptr_t) (huge - 1);
	if (hi > lo) madvise((void*) lo, hi - lo, MADV_HUGEPAGE);
#else
	(void) p; (void) bytes;
#endif
}
static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static inline u32 rd32(const u8* p) { u32 v; memcpy(&v, p, 4); return v; }
static inline u16 rd16(const u8* p) { u16 v; memcpy(&v, p, 2); return v; }

// ------------------------------------------------------------------------------------------- coverage
void coverage_windows::resize(const refdata& ref) {
	const size_t nc = ref.contig_ids.size();
	coverage.resize(nc); starts.resize(nc); ends.resize(nc);
	for (size_t c = 0; c < nc; ++c) if (ref.has_sequence((u32) c)) {
		const size_t w = ref.seq_len[c] / 20 + 2;
		if (coverage[c].size() < w) { coverage[c].reserve(w); advise_huge(coverage[c].data(), w * sizeof(coverage[c][0])); coverage[c].resize(w, 0); starts[c].resize(w, 0); ends[c].resize(w, 0); }
	}
}
bool coverage_windows::fragment_starts_here(u32 contig, i32 start, i32 end) const {
	if (contig >= starts.size()) return false;
	for (int w = start / 20 + 1; w <= end / 20; ++w) { if ((u32) w >= starts[contig].size()) return false; if (starts[contig][w]) return true; }
	return false;
}
bool coverage_windows::fragment_ends_here(u32 contig, i32 start, i32 end) const {
	if (contig >= ends.size()) return false;
	for (int w = start / 20; w < end / 20; ++w) { if ((u32) w >= ends[contig].size()) return false; if (ends[contig][w]) return true; }
	return false;
}
int coverage_windows::get_coverage(u32 contig, i32 position, u32 direction) const {
	if (contig >= coverage.size() || coverage[contig].empty()) return -1;
	if (direction == UPSTREAM) return position < 20 ? 0 : coverage[contig][position / 20 - 1];
	return coverage[contig][position / 20 + 1];
}

// ------------------------------------------------------------------------------------------- BGZF container
// STAR is run with --outBAMcompression 0 (run_arriba.sh:34): every BGZF block then holds ONE stored deflate block -- header byte 0x01 (final, type 00),
// LEN, ~LEN, the bytes (RFC 1951 3.2.4). Is the payload `in` (in_len bytes, out_len inflated) such a block?
static bool stored_block(const u8* in, u32 in_len, u32 out_len) {
	return in_len == 5ull + out_len && in[0] == 0x01 && rd16(in + 1) == (u16) out_len && (u16) (rd16(in + 1) ^ rd16(in + 3)) == 0xFFFF;
}
static void inflate_payload(const u8* in, u32 in_len, u32 out_len, u8* dst) {
	if (out_len == 0) return;
	if (stored_block(in, in_len, out_len)) { memcpy(dst, in + 5, out_len); return; } // copied; anything else goes through zlib
	z_stream zs; memset(&zs, 0, sizeof(zs));
	if (inflateInit2(&zs, -15) != Z_OK) fail("failed to load alignments");
	zs.next_in = (Bytef*) in; zs.avail_in = in_len; zs.next_out = dst; zs.avail_out = out_len;
	const int rc = inflate(&zs, Z_FINISH);
	inflateEnd(&zs);
	if (rc != Z_STREAM_END || zs.avail_out != 0) fail("failed to load alignments");
}

struct bgzf_file {
	const u8* data; size_t size; int fd;
	struct block { u64 in_off; u32 in_len; u32 out_len; u64 out_off; };
	std::vector<block> blocks; u64 total_out;
	bgzf_file(): data(NULL), size(0), fd(-1), total_out(0), raw(false) {}
	~bgzf_file() { if (data) munmap((void*) data, size); if (fd >= 0) close(fd); }
	bool raw; // plain SAM text: the "blocks" are pieces of the file, copied as they are
	// A regular file is mapped (true). Anything else that can be read in sequence (a pipe, a FIFO, a character device) is left open in fd for the
	// stream reader (false).
	bool map(const std::string& path) {
		fd = ::open(path.c_str(), O_RDONLY);
		if (fd < 0) fail("failed to open SAM file");
		struct stat st; if (fstat(fd, &st) != 0 || S_ISDIR(st.st_mode)) fail("failed to open SAM file");
		size = st.st_size;
		if (!S_ISREG(st.st_mode)) { size = 0; return false; }
		if (size == 0) fail("failed to read SAM header");
		data = (const u8*) mmap(NULL, size, PROT_READ, MAP_PRIVATE, fd, 0);
		if (data == MAP_FAILED) { data = NULL; fail("failed to open SAM file"); }
		madvise((void*) data, size, MADV_SEQUENTIAL);
		return true;
	}
	void raw_pieces(u64 piece) {
		raw = true;
		for (u64 off = 0; off < size; off += piece) { block b; b.in_off = b.out_off = off; b.in_len = b.out_len = (u32) std::min<u64>(piece, size - off); blocks.push_back(b); }
		total_out = size;
	}
	void block_table(int threads) {
		// Block table. A block is found from the one before it (its size sits in its header), and every header read faults a page of the mapping in: a
		// 7 GB file of stored blocks costs a quarter of a second on one thread. So every piece of the file guesses its first block (two well-formed
		// headers in a row), walks from there, and the guesses are VERIFIED: the chain of piece s must arrive exactly at the guess of piece s+1; where it
		// does not, that stretch is walked serially. Errors are raised by the serial walk only, at the same offsets as before.
		auto header = [&](u64 off, u32& bsize, u32& xlen) { // well-formed BGZF header at off (SAMv1 4.1)?
			if (off + 18 > size) return false;
			const u8* h = data + off;
			if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return false;
			xlen = rd16(h + 10);
			if (off + 12 + xlen > size) return false;
			bool found = false;
			for (u32 x = 0; x + 4 <= xlen;) { const u8* e = h + 12 + x; const u32 slen = rd16(e + 2); if (e[0] == 'B' && e[1] == 'C' && slen == 2) { bsize = rd16(e + 4) + 1u; found = true; } x += 4 + slen; }
			return found && bsize >= 12 + xlen + 8 && off + bsize <= size;
		};
		auto walk = [&](u64 off, u64 limit, std::vector<block>& out, bool strict) { // blocks starting before `limit`; returns where the chain stands
			while (off < limit && off + 18 <= size) {
				u32 bsize = 0, xlen = 0;
				if (!header(off, bsize, xlen)) {
					if (!strict) break;
					const u8* h = data + off;
					const bool magic = h[0] == 0x1f && h[1] == 0x8b && h[2] == 8 && (h[3] & 4);
					fail(!magic && off == 0 ? "failed to read SAM header" : "failed to load alignments"); // not BGZF (SAM text / CRAM are not supported); at the start of the file no header can be read (arriba.cpp:122)
				}
				block b; b.in_off = off + 12 + xlen; b.in_len = bsize - 12 - xlen - 8; b.out_len = rd32(data + off + bsize - 4); b.out_off = 0;
				out.push_back(b);
				off += bsize;
			}
			return off;
		};
		const size_t min_bytes = getenv("ARB_SCAN_MIN_BYTES") ? (size_t) atol(getenv("ARB_SCAN_MIN_BYTES")) : (size_t) 64 << 20; // test hook
		const int pieces = threads > 1 && size > min_bytes ? threads : 1;
		if (pieces > 1) {
			std::vector<u64> guess(pieces + 1, size), stop_at(pieces, 0);
			std::vector<std::vector<block> > found(pieces);
			guess[0] = 0;
			std::vector<std::thread> pool;
			for (int s = 1; s < pieces; ++s) pool.emplace_back([&, s]() {
				u64 q = (u64) size * s / pieces; const u64 give_up = std::min<u64>(size, q + (256u << 10));
				for (; q < give_up; ++q) { u32 b1 = 0, x1 = 0, b2 = 0, x2 = 0; if (header(q, b1, x1) && (q + b1 + 18 > size || header(q + b1, b2, x2))) break; }
				guess[s] = q < give_up ? q : size;
			});
			for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
			pool.clear();
			for (int s = 1; s < pieces; ++s) pool.emplace_back([&, s]() { stop_at[s] = guess[s] < size ? walk(guess[s], guess[s + 1], found[s], false) : size; });
			stop_at[0] = walk(0, guess[1], found[0], false);
			for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
			u64 q = 0;
			for (int s = 0; s < pieces; ++s) {
				if (q == guess[s] && guess[s] < size) { blocks.insert(blocks.end(), found[s].begin(), found[s].end()); q = stop_at[s]; }
				if (q < guess[s + 1]) q = walk(q, guess[s + 1], blocks, true); // wrong or missing guess, or a chain that broke off: walk (and diagnose) this stretch
			}
			walk(q, size, blocks, true);
		} else walk(0, size, blocks, true);
		u64 out = 0;
		for (size_t b = 0; b < blocks.size(); ++b) { blocks[b].out_off = out; out += blocks[b].out_len; }
		total_out = out;
	}
	void inflate_block(const block& b, u8* dst) const {
		if (b.out_len == 0) return;
		if (raw) { memcpy(dst, data + b.in_off, b.out_len); return; }
		inflate_payload(data + b.in_off, b.in_len, b.out_len, dst);
	}
};

template <class F> static void parallel_for(int threads, size_t n, F f) { // f(thread, begin, end)
	if (threads <= 1 || n < 2) { f(0, (size_t) 0, n); return; }
	std::vector<std::thread> pool; std::vector<std::string> errors(threads);
	for (int t = 0; t < threads; ++t) pool.emplace_back([&, t]() {
		try { f(t, n * t / threads, n * (t + 1) / threads); } catch (const std::exception& e) { errors[t] = e.what(); }
	});
	for (size_t t = 0; t < pool.size(); ++t) pool[t].join();
	for (int t = 0; t < threads; ++t) if (!errors[t].empty()) fail(errors[t]);
}

// ------------------------------------------------------------------------------------------- driver
frag_view fragment_table::view() {
	frag_view v;
	v.n = n; v.n_aln = n_aln.data(); v.fflags = fflags.data(); v.filter = filter.data(); v.contig = contig.data(); v.start = start.data(); v.end = end.data();
	v.aflags = aflags.data(); v.cigar_off = cigar_off.data(); v.cigar_cnt = cigar_cnt.data(); v.seq_off = seq_off.data(); v.seq_len = seq_len.data();
	v.genes_off = genes_off.data(); v.genes_cnt = genes_cnt.data(); v.cigar = cigar.data(); v.seq = seq.data(); v.genes = genes.data();
	return v;
}


// the text of a fatal record error (records_hd.h: kinds and order); tid_to_contig: the map of the file the record came from
static std::string record_error_text(u64 error, arb_ctx* ctx, const std::vector<u16>& tid_to_contig, const refdata& ref) {
	const u32 kind = (u32) (error & 7);
	if (kind == REC_ERR_ANNOTATION) return "too many overlapping annotation records at one locus";
	if (kind == REC_ERR_CIGAR || kind == REC_ERR_BEYOND || kind == REC_ERR_UNMAPPED) {
		const uint8_t* body = NULL; uint64_t n = 0;
		rec_t r;
		if (arb_records_error_record(ctx, &body, &n) == 0 && body && rec_parse(body, (u32) n, r)) {
			const std::string name(r.qname(), r.name_len());
			if (kind == REC_ERR_UNMAPPED) return "alignment of read '" + name + "' in the chimeric alignment file has no reference sequence (the file must hold mapped records only, as STAR writes Chimeric.out.sam)";
			if (r.tid >= 0 && (size_t) r.tid < tid_to_contig.size()) {
				const u32 contig = tid_to_contig[r.tid];
				i64 query_span = 0;
				rec_validate(r, ref.has_sequence(contig) ? (u32) ref.seq_len[contig] : 0, query_span);
				if (kind == REC_ERR_CIGAR) return "CIGAR string of read '" + name + "' does not fit its sequence (" + std::to_string(query_span) + " bases in " + std::to_string(r.n_cigar) + " operations, sequence of " + std::to_string(r.l_seq) + ")";
				return "alignment of read '" + name + "' extends beyond the end of contig '" + ref.original_names[contig] + "' (was the file aligned to another assembly?)";
			}
		}
	}
	return "failed to load alignments";
}

// The format is decided by the input's content, as htslib's sam_open does: BGZF whose stream starts with "BAM\1" is BAM, any other BGZF stream is SAM
// text, and an input that is not gzip is plain SAM if its first line starts with '@' or has at least 10 tabs. detect_prefix_bgzf is that rule over the first
// bytes: all of a shorter input, for a gzip input its first header, else at least its first line. Files and streams both call it.
enum input_format { INPUT_BAM, INPUT_SAM_BGZF, INPUT_SAM };
static bool detect_prefix_bgzf(const u8* d, size_t n) { // true: BGZF (BAM or SAM); false: plain SAM
	if (n >= 3 && d[0] == 0x1f && d[1] == 0x8b && d[2] == 8) {
		const u32 xlen = n >= 12 ? rd16(d + 10) : 0;
		bool bgzf = false;
		if (n >= 4 && (d[3] & 4) && n >= 12ull + xlen)
			for (u32 x = 0; x + 4 <= xlen;) { const u8* e = d + 12 + x; if (e[0] == 'B' && e[1] == 'C') bgzf = true; x += 4 + rd16(e + 2); }
		if (!bgzf) fail("failed to read SAM header (gzip-compressed SAM must be BGZF (bgzip) or uncompressed)");
		return true;
	}
	if (n >= 4 && memcmp(d, "CRAM", 4) == 0) fail("failed to read SAM header (CRAM input is not supported: convert it to BAM or SAM)");
	u32 tabs = 0;
	for (size_t x = 0; x < n && d[x] != '\n'; ++x) tabs += d[x] == '\t';
	if (n == 0 || (d[0] != '@' && tabs < 10)) fail("failed to read SAM header");
	return false;
}
// BAM or SAM, from the first inflated bytes of a BGZF input
template <class S> static input_format bgzf_format(S& src) {
	std::vector<u8> head;
	while (head.size() < 4 && src.more(head)) {}
	src.rewind();
	return head.size() >= 4 && memcmp(head.data(), "BAM\1", 4) == 0 ? INPUT_BAM : INPUT_SAM_BGZF;
}

// The inflated bytes of an input from its start, one block (or piece of plain text) at a time, for format detection and the header: more() appends the
// next one (false at the end), available(n): the input holds at least n inflated bytes, rewind(): more() starts again at the first block.
struct file_source {
	const bgzf_file& f; size_t next;
	explicit file_source(const bgzf_file& file): f(file), next(0) {}
	template <class B> bool more(B& out) {
		if (next >= f.blocks.size()) return false;
		const size_t at = out.size(); out.resize(at + f.blocks[next].out_len); f.inflate_block(f.blocks[next], (u8*) &out[at]); ++next;
		return true;
	}
	bool available(u64 n) const { return n <= f.total_out; }
	void rewind() { next = 0; }
};

// A block header as the file path's block table judges it, at d[0, n) of an input read in sequence (at_eof: no more bytes will come): 1 = a whole block
// (bsize, xlen), 0 = more bytes are needed to tell, -1 = the end of the blocks (fewer than 18 bytes left: the block table ignores them). A malformed
// header stops the run with a framing_error, which no other error of the input outranks (the file path checks the framing of the whole file first).
struct framing_error: std::runtime_error { explicit framing_error(const std::string& m): std::runtime_error(m) {} };
static int stream_block_at(const u8* d, size_t n, bool at_eof, u32& bsize, u32& xlen) {
	if (n < 18) return at_eof ? -1 : 0;
	if (!(d[0] == 0x1f && d[1] == 0x8b && d[2] == 8 && (d[3] & 4))) throw framing_error("failed to load alignments");
	xlen = rd16(d + 10);
	if (n < 12ull + xlen + 2 && !at_eof) return 0;
	bool found = false;
	for (u32 x = 0; x + 4 <= xlen && 12ull + x + 6 <= n;) { const u8* e = d + 12 + x; const u32 slen = rd16(e + 2); if (e[0] == 'B' && e[1] == 'C' && slen == 2) { bsize = rd16(e + 4) + 1u; found = true; } x += 4 + slen; }
	if (!found || bsize < 12 + xlen + 8) throw framing_error("failed to load alignments");
	if (bsize > n) { if (!at_eof) return 0; throw framing_error("failed to load alignments"); }
	return 1;
}

// ------------------------------------------------------------------------------------------- stream input
// An input that is not a regular file: read in sequence. Format detection and the header read into `head`, and what they read beyond the header stays
// there for the first chunk; the chunks are read into the page-locked chunk buffers. `left` / `n_left`: the bytes read but not yet put into a chunk (in
// `head`, or behind the blocks of the last chunk in its buffer).
struct stream_input {
	int fd; bool eof, started, bgzf;
	std::vector<u8> head; size_t head_walk; // BGZF: head[head_walk, ...) is not walked yet (header phase)
	bool in_head;
	const u8* left; size_t n_left;
	u64 out_pos; // inflated (plain: stream) position of the first byte behind the last chunk
	struct block { size_t start; u32 in_off, in_len, out_len; u64 out_off; };
	std::vector<block> walked; u64 walked_out; size_t inflated; // the header phase's blocks
	stream_input(int f): fd(f), eof(false), started(false), bgzf(false), head_walk(0), in_head(true), left(NULL), n_left(0), out_pos(0), walked_out(0), inflated(0) {}
	~stream_input() { if (fd >= 0) close(fd); } // a producer still writing gets EPIPE
	size_t read_some(u8* dst, size_t n) { // 0: end of the input
		for (;;) {
			const ssize_t r = ::read(fd, dst, n);
			if (r > 0) { started = true; return (size_t) r; }
			if (r == 0) { eof = true; return 0; }
			if (errno == EINTR) continue;
			fail(started ? "failed to load alignments" : "failed to open SAM file");
		}
	}
	bool read_head() { const size_t at = head.size(); head.resize(at + (64u << 10)); const size_t got = eof ? 0 : read_some(head.data() + at, 64u << 10); head.resize(at + got); return got > 0; }
	// format detection: the bytes detect_prefix_bgzf looks at
	bool detect() {
		auto fill = [&](size_t n) { while (head.size() < n && read_head()) {} };
		fill(4);
		if (head.size() >= 3 && head[0] == 0x1f && head[1] == 0x8b && head[2] == 8) { fill(12); if (head.size() >= 12) fill(12 + (size_t) rd16(head.data() + 10)); }
		else for (size_t scanned = 0; !memchr(head.data() + scanned, '\n', head.size() - scanned);) { scanned = head.size(); if (!read_head()) break; }
		bgzf = detect_prefix_bgzf(head.data(), head.size());
		return bgzf;
	}
	// header phase, BGZF: walk the next block of head (reading as needed); false at the end of the blocks
	bool walk_one() {
		u32 bsize = 0, xlen = 0; int r;
		while ((r = stream_block_at(head.data() + head_walk, head.size() - head_walk, eof, bsize, xlen)) == 0) read_head();
		if (r < 0) return false;
		block b; b.start = head_walk; b.in_off = (u32) (12 + xlen); b.in_len = bsize - 20 - xlen; b.out_len = rd32(head.data() + head_walk + bsize - 4); b.out_off = walked_out;
		walked.push_back(b); walked_out += b.out_len; head_walk += bsize;
		return true;
	}
	// the source of format detection and the header (file_source's interface)
	template <class B> bool more(B& out) {
		if (!bgzf) { // plain text: whatever is read next
			if (head_walk >= head.size() && !read_head()) return false;
			const size_t at = out.size(); out.resize(at + head.size() - head_walk); memcpy(&out[at], head.data() + head_walk, head.size() - head_walk); head_walk = head.size();
			return true;
		}
		if (inflated >= walked.size() && !walk_one()) return false;
		const block& b = walked[inflated++];
		const size_t at = out.size(); out.resize(at + b.out_len); inflate_payload(head.data() + b.start + b.in_off, b.in_len, b.out_len, (u8*) &out[at]);
		return true;
	}
	bool available(u64 n) { while (walked_out < n && walk_one()) {} return walked_out >= n; }
	void rewind() { inflated = 0; if (!bgzf) head_walk = 0; }
	// the header ends at header_end: the first chunk starts at the block of the first record (plain text: at the piece of the file path that holds it)
	void header_done(u64 header_end, u64 piece) {
		size_t start = head_walk; out_pos = walked_out;
		if (bgzf) { for (size_t k = 0; k < walked.size(); ++k) if (walked[k].out_off + walked[k].out_len > header_end) { start = walked[k].start; out_pos = walked[k].out_off; break; } }
		else { out_pos = header_end / piece * piece; start = (size_t) out_pos; }
		in_head = false; left = head.data() + start; n_left = head.size() - start;
	}
	// where the records stop (after an error, or at the end): the framing of the rest of the input is checked (not inflated), as the file path checks it
	// before anything else. Called while `left` still points into a live chunk buffer; afterwards nothing of the input is read any more.
	bool drained = false;
	void drain() {
		if (!bgzf || drained) return;
		drained = true;
		std::vector<u8> w;
		if (in_head) w.assign(head.begin() + head_walk, head.end()); else w.assign(left, left + n_left);
		in_head = false; left = NULL; n_left = 0;
		size_t at = 0;
		for (;;) {
			u32 bsize = 0, xlen = 0;
			const int r = stream_block_at(w.data() + at, w.size() - at, eof, bsize, xlen);
			if (r < 0) return;
			if (r > 0) { at += bsize; continue; }
			w.erase(w.begin(), w.begin() + at); at = 0;
			const size_t have = w.size(); w.resize(have + (256u << 10)); w.resize(have + read_some(w.data() + have, 256u << 10));
		}
	}
};

// The @ lines at the start of a SAM stream, however many blocks they span; every @SQ line gives the next reference (its SN) to `reference`. Returns the
// offset of the first record in the stream. src: file_source or stream_input.
template <class S, class F> static u64 read_sam_header(S& src, F reference) {
	std::string text;
	auto more = [&]() { return src.more(text); };
	size_t p = 0;
	for (;;) {
		while (p >= text.size() && more()) {}
		if (p >= text.size() || text[p] != '@') return p;
		size_t lf;
		while ((lf = text.find('\n', p)) == std::string::npos && more()) {}
		std::string line = text.substr(p, lf == std::string::npos ? std::string::npos : lf - p);
		if (lf != std::string::npos && !line.empty() && line.back() == '\r') line.pop_back();
		if (line.compare(0, 4, "@SQ\t") == 0) {
			std::string name; bool has_name = false, has_length = false;
			for (size_t a = 4; a <= line.size();) {
				size_t b = line.find('\t', a); if (b == std::string::npos) b = line.size();
				const std::string field = line.substr(a, b - a);
				if (field.compare(0, 3, "SN:") == 0 && !has_name) { name = field.substr(3); has_name = !name.empty(); }
				else if (field.compare(0, 3, "LN:") == 0 && !has_length) {
					u64 v = 0; bool ok = field.size() > 3 && field.size() <= 3 + 18;
					for (size_t x = 3; ok && x < field.size(); ++x) { ok = field[x] >= '0' && field[x] <= '9'; v = v * 10 + (u64) (field[x] - '0'); }
					has_length = ok && v > 0;
				}
				a = b + 1;
			}
			if (!has_name || !has_length) fail("failed to read SAM header");
			reference(name);
		}
		if (lf == std::string::npos) return text.size();
		p = lf + 1;
	}
}

// The BAM header (magic, text, references), however many blocks it spans; every reference's name goes to `reference`. Returns the offset of the first
// record in the inflated stream.
template <class S, class F> static u64 read_bam_header(S& src, F reference) {
	std::vector<u8> h;
	auto have = [&](u64 n) { // the first n bytes of the stream are in h
		if (!src.available(n)) return false;
		while (h.size() < n && src.more(h)) {}
		return h.size() >= n;
	};
	if (!have(12) || memcmp(h.data(), "BAM\1", 4) != 0) fail("failed to read SAM header");
	u64 p = 8ull + rd32(h.data() + 4);
	if (!have(p + 4)) fail("failed to read SAM header");
	const u32 n_ref = rd32(h.data() + p); p += 4;
	for (u32 k = 0; k < n_ref; ++k) {
		if (!have(p + 4)) fail("failed to read SAM header");
		const u32 l_name = rd32(h.data() + p); p += 4;
		if (!have(p + l_name + 4)) fail("failed to read SAM header");
		reference(std::string((const char*) h.data() + p, strnlen((const char*) h.data() + p, l_name))); p += l_name + 4;
	}
	return p;
}

// one input: its blocks (a file) or its reader (a stream), format and header (the contig id of every reference; SAM: the @SQ names, for the RNAME lookup
// on the device)
struct input_file {
	bgzf_file f; std::unique_ptr<stream_input> stream; input_format format; u64 header_end; std::vector<u16> tid_to_contig; std::string sq_names; std::vector<u64> sq_off;
	input_file(): format(INPUT_BAM), header_end(0), sq_off(1, 0) {}
	// opened and its format detected: a file's block table is built here (the framing of the whole file is checked), or it is cut into pieces of at most
	// 4 MiB, and no larger than a chunk (but at least 256 bytes), that are copied as they are (plain SAM); a stream is read as far as the rule needs
	void open(const std::string& path, int threads, u64 chunk_target) {
		if (!f.map(path)) {
			stream.reset(new stream_input(f.fd)); f.fd = -1;
			if (!stream->detect()) { format = INPUT_SAM; return; }
			try { format = bgzf_format(*stream); } catch (const framing_error&) { throw; } catch (const std::exception&) { stream->drain(); throw; }
			return;
		}
		if (!detect_prefix_bgzf(f.data, f.size)) { f.raw_pieces(piece(chunk_target)); format = INPUT_SAM; return; }
		f.block_table(threads);
		file_source src(f);
		format = bgzf_format(src);
	}
	static u64 piece(u64 chunk_target) { return std::max<u64>(256, std::min<u64>(chunk_target, 4ull << 20)); }
	bool has_blocks() const { return stream ? !stream->bgzf || !stream->walked.empty() : !f.blocks.empty(); }
	template <class F> u64 read_header(F reference) {
		if (stream) return format == INPUT_BAM ? read_bam_header(*stream, reference) : read_sam_header(*stream, reference);
		file_source src(f);
		return format == INPUT_BAM ? read_bam_header(src, reference) : read_sam_header(src, reference);
	}
	void drain() { if (stream) stream->drain(); }
};

static void read_inputs(input_file& chim, input_file& main_file, refdata& ref, const ingest_options& opt, fragment_table& out, coverage_windows& coverage, ingest_stats& stats);

void read_chimeric_alignments(const std::string& bam_path, refdata& ref, const ingest_options& opt, fragment_table& out, coverage_windows& coverage, ingest_stats& stats) {
	const int T = std::min(255, std::max(1, opt.threads));
	const u64 chunk_target = getenv("ARB_CHUNK_BYTES") ? (u64) atoll(getenv("ARB_CHUNK_BYTES")) : 128ull << 20; // env: test hook (many small chunks)
	// A separate chimeric file (-c) is read first, in a call of its own in the reference (arriba.cpp:123-130): its header, then the main file's, name the
	// contigs (ids in that order; a contig's printed name is the last header's spelling), its records go into the store ahead of the main file's.
	// A file's framing is checked as it is opened; a stream's as it is read, and after any other error the rest of each stream the file path would have
	// checked by then is walked, so that a framing error wins as it does for a file.
	input_file chim, main_file;
	if (!opt.chimeric_path.empty()) chim.open(opt.chimeric_path, T, chunk_target);
	try { main_file.open(bam_path, T, chunk_target); } catch (const framing_error&) { throw; } catch (const std::exception&) { chim.drain(); throw; }
	try { read_inputs(chim, main_file, ref, opt, out, coverage, stats); }
	catch (const framing_error&) { throw; }
	catch (const std::exception&) { chim.drain(); main_file.drain(); throw; }
}

static void read_inputs(input_file& chim, input_file& main_file, refdata& ref, const ingest_options& opt, fragment_table& out, coverage_windows& coverage, ingest_stats& stats) {
	const int T = std::min(255, std::max(1, opt.threads));
	const bool trace = getenv("ARB_TRACE") != NULL;
	double tr_last = now_s();
	auto lap = [&](const char* what) { if (trace) { const double t = now_s(); fprintf(stderr, "[ingest] %-28s %.3f s\n", what, t - tr_last); tr_last = t; } };
	const u64 chunk_target = getenv("ARB_CHUNK_BYTES") ? (u64) atoll(getenv("ARB_CHUNK_BYTES")) : 128ull << 20;
	const bool has_chimeric = !opt.chimeric_path.empty();
	lap("open + block table");
	stats.t_inflate = stats.t_parse = stats.t_finalize = 0;
	stats.chimeric_records = stats.chimeric_malformed = stats.chimeric_total = 0;
	arb_ctx* const ctx = opt.scan_ctx;
	auto check = [&](int rc, const char* what) { if (rc != 0) fail(std::string(what) + ": " + arb_last_error(ctx)); };

	std::vector<u8> interesting_contig, viral_contig;
	for (input_file* in : {&chim, &main_file}) {
		if (in == &chim && !has_chimeric) continue;
		if (!in->has_blocks()) fail("failed to read SAM header");
		auto add_reference = [&](const std::string& target) { // the next reference of the header (BAM or @SQ)
			const u16 id = ref.contig_id(remove_chr(target));
			ref.original_names[id] = target;
			in->tid_to_contig.push_back(id);
		};
		if (in->format != INPUT_BAM) in->header_end = in->read_header([&](const std::string& name) { add_reference(name); in->sq_names += name; in->sq_off.push_back(in->sq_names.size()); });
		else in->header_end = in->read_header(add_reference);
	}
	{ // the contig flags of the grown contig table, and the coverage windows
		const size_t nc = ref.contig_ids.size();
		interesting_contig.assign(nc, 0); viral_contig.assign(nc, 0);
		for (std::map<std::string, u16>::iterator c = ref.contig_ids.begin(); c != ref.contig_ids.end(); ++c) {
			interesting_contig[c->second] = contig_matches(c->first, opt.interesting_contigs);
			viral_contig[c->second] = contig_matches(c->first, opt.viral_contigs);
			if (!ref.has_sequence(c->second) && interesting_contig[c->second]) fail("could not find sequence of contig '" + c->first + "'");
		}
		ref.flatten(); // contig table may have grown
		coverage.resize(ref);
	}
	if (opt.after_header) opt.after_header(); // the grown contig table and the gene index go to the device
	const u32 nc = (u32) ref.contig_ids.size();
	{
		std::vector<u64> n_windows(nc);
		for (u32 c = 0; c < nc; ++c) n_windows[c] = coverage.coverage[c].size();
		check(arb_records_begin(ctx, main_file.tid_to_contig.data(), (u32) main_file.tid_to_contig.size(), interesting_contig.data(), viral_contig.data(), n_windows.data(), nc,
		                        opt.max_itd_length, opt.external_duplicate_marking ? 1 : 0,
		                        main_file.stream || chim.stream ? 0 : main_file.f.total_out + (has_chimeric ? chim.f.total_out : 0) /* a stream's size is not known */), "arb_records_begin");
	}
	lap("header");

	// chunks of ~128 MiB of decompressed data, each a whole number of BGZF blocks (pieces of a plain SAM file); a record (or line) that straddles a chunk
	// boundary stays on the device for the next one
	// A chunk is inflated by the host while the device copies and scans the previous one. A stream's chunk is read while the device scans the previous one:
	// the producer keeps writing, and waits only when both buffers are full.
	struct chunk_t {
		column<u8> buf /* page-locked: copied to the device asynchronously */; u64 pos /* in the inflated stream */; u64 first; bool last;
		u64 bytes /* stream: the inflated bytes of the chunk */, raw_bytes /* BGZF stream: the bytes of buf that go up */; std::vector<arb_bgzf_block> blocks /* BGZF stream */;
		chunk_t(): pos(0), first(0), last(false), bytes(0), raw_bytes(0) {}
	};
	chunk_t chunks[2];
	double t_inflate = 0; // written by the inflating thread only
	const u64 NO_ERROR = ~(u64) 0;
	u64 record_error = NO_ERROR, main_first = 0;
	// the records of one file; returns their number (record_error set: stopped at the chunk that has the error)
	auto read_records = [&](input_file& in) {
		const bgzf_file& bam = in.f;
		size_t b0 = 0;
		auto prepare = [&](chunk_t& c) {
			const double ti = now_s();
			size_t b1 = b0; u64 bytes = 0;
			while (b1 < bam.blocks.size() && (bytes == 0 || bytes + bam.blocks[b1].out_len <= chunk_target)) bytes += bam.blocks[b1++].out_len;
			column<u8>& buf = c.buf;
			if (buf.capacity() < bytes) buf.reserve(bytes + (16u << 20)); // one page-locked block per buffer for the whole file (chunks differ a little in size)
			buf.resize(bytes);
			c.pos = b0 < bam.blocks.size() ? bam.blocks[b0].out_off : bam.total_out;
			const size_t first = b0;
			parallel_for(T, b1 - first, [&](int, size_t lo, size_t hi) { for (size_t b = first + lo; b < first + hi; ++b) bam.inflate_block(bam.blocks[b], buf.data() + (bam.blocks[b].out_off - c.pos)); });
			b0 = b1;
			c.last = b0 >= bam.blocks.size(); c.first = 0;
			t_inflate += now_s() - ti;
		};
		// A stream's chunk: the bytes left behind the previous chunk, then read(). BGZF: the same whole blocks the file path's chunk would hold (the block
		// that does not fit stays for the next chunk); stored blocks stay where they were read, the others are inflated behind the read bytes, and the
		// block table says where each payload is. Plain SAM: the bytes of the file path's chunk (a whole number of its pieces).
		auto prepare_stream = [&](chunk_t& c) {
			const double ti = now_s();
			stream_input& s = *in.stream;
			column<u8>& buf = c.buf;
			const u64 piece = input_file::piece(chunk_target), text_bytes = std::max<u64>(1, chunk_target / piece) * piece;
			const size_t base = (size_t) std::min<u64>(s.bgzf ? chunk_target : text_bytes, 1ull << 30) + (1u << 20);
			if (buf.capacity() < base) buf.reserve(base);
			buf.resize(std::max(buf.capacity(), std::max(base, s.n_left)));
			size_t have = s.n_left;
			memcpy(buf.data(), s.left, have);
			auto read_more = [&](size_t want) { // false at the end of the stream
				if (buf.size() - have < want) buf.resize(have + want);
				if (want == 0) return true;
				const size_t got = s.read_some(buf.data() + have, want);
				have += got; return got > 0;
			};
			c.pos = s.out_pos; c.first = 0; c.last = false; c.blocks.clear();
			if (!s.bgzf) {
				while (have < text_bytes + 1 && read_more(std::min<size_t>(buf.size() - have, (size_t) text_bytes + (64u << 10) - have))) {} // one byte beyond tells whether this is the last chunk
				c.bytes = std::min<u64>(have, text_bytes); c.last = have <= text_bytes;
				s.left = buf.data() + c.bytes; s.n_left = have - c.bytes; s.out_pos += c.bytes;
				t_inflate += now_s() - ti;
				return;
			}
			size_t at = 0; u64 bytes = 0;
			std::vector<u32> in_len;
			for (;;) {
				u32 bsize = 0, xlen = 0;
				const int r = stream_block_at(buf.data() + at, have - at, s.eof, bsize, xlen);
				if (r < 0) { c.last = true; break; }
				if (r == 0) { // the rest of the chunk is estimated from its ratio of read to inflated bytes so far
					const double ratio = bytes ? std::min(1.0, (double) at / (double) bytes) : 1.0;
					const size_t want = (size_t) std::min<double>((double) (chunk_target > bytes ? chunk_target - bytes : 0) * ratio, (double) (1u << 30)) + (64u << 10) + 64;
					read_more(want);
					continue;
				}
				const u32 out_len = rd32(buf.data() + at + bsize - 4);
				if (bytes != 0 && bytes + out_len > chunk_target) break;
				const arb_bgzf_block b = {at + 12 + xlen, out_len, bytes};
				c.blocks.push_back(b); in_len.push_back(bsize - 20 - xlen);
				bytes += out_len; at += bsize;
			}
			// the payloads: stored ones in place, the others inflated behind the bytes read
			std::vector<size_t> packed; std::vector<u64> deflate_at; u64 inflated = 0;
			for (size_t k = 0; k < c.blocks.size(); ++k) {
				arb_bgzf_block& b = c.blocks[k];
				if (b.bytes == 0) continue;
				if (stored_block(buf.data() + b.src, in_len[k], (u32) b.bytes)) { b.src += 5; continue; }
				packed.push_back(k); deflate_at.push_back(b.src); b.src = have + inflated; inflated += b.bytes;
			}
			if (buf.size() < have + inflated) buf.resize(have + inflated);
			s.left = buf.data() + at; s.n_left = have - at; s.out_pos += bytes;
			c.bytes = bytes; c.raw_bytes = packed.empty() ? at : have + inflated;
			parallel_for(T, packed.size(), [&](int, size_t lo, size_t hi) {
				for (size_t j = lo; j < hi; ++j) { const arb_bgzf_block& b = c.blocks[packed[j]]; inflate_payload(buf.data() + deflate_at[j], in_len[packed[j]], (u32) b.bytes, buf.data() + b.src); }
			});
			t_inflate += now_s() - ti;
		};
		if (in.stream) { in.stream->header_done(in.header_end, input_file::piece(chunk_target)); prepare_stream(chunks[0]); }
		else {
			while (b0 < bam.blocks.size() && bam.blocks[b0].out_off + bam.blocks[b0].out_len <= in.header_end) ++b0; // the first chunk starts at the block of the first record
			prepare(chunks[0]);
		}
		chunks[0].first = in.header_end - chunks[0].pos;
		if (in.format != INPUT_BAM) check(arb_records_text_names(ctx, in.sq_names.data(), in.sq_off.data(), (u32) in.tid_to_contig.size()), "arb_records_text_names");
		u64 total_records = 0;
		for (int cur = 0;; cur ^= 1) {
			chunk_t& c = chunks[cur];
			std::string prepare_error; bool prepare_framing = false; std::thread next;
			if (!c.last) next = std::thread([&]() {
				try { if (in.stream) prepare_stream(chunks[cur ^ 1]); else prepare(chunks[cur ^ 1]); }
				catch (const framing_error& x) { prepare_error = x.what(); prepare_framing = true; }
				catch (const std::exception& x) { prepare_error = x.what(); if (prepare_error.empty()) prepare_error = "failed to load alignments"; }
			});
			const double tp = now_s();
			uint64_t n_records = 0, carry = 0, error = NO_ERROR; uint32_t malformed = 0;
			const u8* data = c.buf.data(); u64 bytes = c.buf.size();
			int rc = 0;
			if (in.stream) bytes = c.bytes;
			if (in.stream && in.stream->bgzf) { rc = arb_records_bgzf_stage(ctx, c.buf.data(), c.raw_bytes, c.blocks.data(), (u32) c.blocks.size()); data = NULL; }
			if (rc == 0) rc = in.format == INPUT_BAM ? arb_records_chunk(ctx, data, bytes, c.first, c.pos, &n_records, &carry, &malformed, &error)
			                                         : arb_records_text_chunk(ctx, data, bytes, c.first, c.pos, c.last ? 1 : 0, &n_records, &carry, &error);
			stats.t_parse += now_s() - tp;
			if (next.joinable()) next.join();
			if (prepare_framing) throw framing_error(prepare_error); // a file's framing is checked before any record
			check(rc, in.format == INPUT_BAM ? "arb_records_chunk" : "arb_records_text_chunk");
			if (malformed) fail("failed to load alignments");
			total_records += n_records;
			if (error != NO_ERROR) { record_error = error; break; } // the replay may still find an earlier one (read-through fragments)
			if (!prepare_error.empty()) fail(prepare_error);
			if (c.last) { if (carry) fail("failed to load alignments"); break; } // truncated file
		}
		return total_records;
	};
	try {
		if (has_chimeric) {
			u64 first = 0;
			check(arb_records_source(ctx, 1, chim.tid_to_contig.data(), (u32) chim.tid_to_contig.size(), &first), "arb_records_source");
			stats.chimeric_records = read_records(chim);
			if (record_error == NO_ERROR) check(arb_records_source(ctx, 0, main_file.tid_to_contig.data(), (u32) main_file.tid_to_contig.size(), &main_first), "arb_records_source");
			else main_first = NO_ERROR; // the main file is not read
		}
		stats.records = record_error == NO_ERROR ? read_records(main_file) : 0;
	} catch (const framing_error&) { throw; } catch (const std::exception&) { chim.drain(); main_file.drain(); throw; }
	// The records stop here (a record error, or the end of the input). A stream's framing error further on outranks whatever follows -- the replay's
	// errors, the -c file's warning and progress line -- as it does for a file, whose framing is checked when it is opened; and the chunk buffers the
	// streams' unread bytes lie in are still alive.
	chim.drain(); main_file.drain();
	if (trace) fprintf(stderr, "[ingest]   of which inflate %.3f s (overlaps with) chunk copies + record extraction %.3f s\n", t_inflate, stats.t_parse);
	stats.t_inflate = t_inflate;
	{ chunk_t a, b; std::swap(chunks[0], a); std::swap(chunks[1], b); }
	lap("inflate + copy + extract");

	// ---- the replay by key: fragment pools, coverage windows, counters (csrc/records.cu) ----
	const double tf = now_s();
	std::vector<u64> counters((size_t) REC_CTR_VIRAL + nc, 0);
	{
		std::vector<u16*> cov(nc); std::vector<u8*> starts(nc), ends(nc);
		for (u32 c = 0; c < nc; ++c) { cov[c] = coverage.coverage[c].data(); starts[c] = coverage.starts[c].data(); ends[c] = coverage.ends[c].data(); }
		uint64_t error = NO_ERROR;
		check(arb_records_finish(ctx, cov.data(), starts.data(), ends.data(), (uint64_t*) counters.data(), &error), "arb_records_finish");
		if (error != NO_ERROR) record_error = std::min<u64>(record_error, error);
	}
	const char* no_chimeric_reads = "no split reads or discordant mates found (STAR must either be run with '--chimOutType WithinBAM' or the file 'Chimeric.out.sam' must be passed to Arriba via the argument -c)";
	// The end of the -c file's call: its first malformed pass (the replay's counting pass has its verdicts, also when the main file has a record error), its
	// warning, its lack of chimeric reads, its progress line. All of it comes before any error of the main file.
	auto chimeric_file_done = [&]() {
		uint64_t c[2];
		check(arb_fragment_table_chimeric_file(ctx, c), "arb_fragment_table_chimeric_file");
		stats.chimeric_malformed = c[0]; stats.chimeric_total = c[1];
		if (c[0] > 0) std::cerr << "WARNING: " << c[0] << " SAM records were malformed and ignored" << std::endl;
		if (counters[REC_CTR_CHIMERIC] == 0) fail(no_chimeric_reads);
		if (opt.chimeric_done) opt.chimeric_done(c[1]);
	};
	if (record_error != NO_ERROR) {
		const bool in_chimeric_file = has_chimeric && (record_error >> 3) < main_first;
		if (has_chimeric && !in_chimeric_file) chimeric_file_done();
		fail(record_error_text(record_error, ctx, in_chimeric_file ? chim.tid_to_contig : main_file.tid_to_contig, ref));
	}
	if (trace) {
		arb_timings tm;
		if (arb_get_timings(ctx, &tm) == 0)
			fprintf(stderr, "[ingest]   record store: allocated %u times, %.1f MB at most; %.1f MB copied to the device, %.1f ms assembling stream chunks\n", tm.rec_store_grows, tm.rec_store_bytes / 1e6, tm.rec_h2d_bytes / 1e6, tm.rec_unwrap_ms);
	}
	lap("replay (device)");
	stats.mapped_reads = counters[REC_CTR_MAPPED]; stats.malformed = counters[REC_CTR_MALFORMED]; stats.missing_hi_tag = counters[REC_CTR_MISSING_HI];
	stats.no_chimeric_reads = counters[REC_CTR_CHIMERIC] == 0;
	stats.mapped_viral_reads_by_contig.assign(counters.begin() + REC_CTR_VIRAL, counters.end());
	if (!has_chimeric && stats.mapped_reads == 0) fail("no normal reads found");

	// ---- the fragment table, built on the device from the pools (csrc/fragtable.cu): slot normalisation and rejection of
	// malformed fragments (read_chimeric_alignments.cpp:340-506), name order, SoA columns, multimapper flags (:792-802) ----
	uint64_t sizes[6];
	check(arb_fragment_table_build(ctx, sizes), "arb_fragment_table_build");
	lap("normalise + name order + columns (device)");
	stats.multimapper_pairs = sizes[5];
	if (has_chimeric) { // the -c file's call ends, then the main file's
		chimeric_file_done();
		if (stats.mapped_reads == 0) fail("no normal reads found");
		stats.malformed += sizes[1] - stats.chimeric_malformed;
		if (stats.malformed > 0) std::cerr << "WARNING: " << stats.malformed << " SAM records were malformed and ignored" << std::endl;
	} else {
		stats.malformed += sizes[1];
		if (stats.malformed > 0) std::cerr << "WARNING: " << stats.malformed << " SAM records were malformed and ignored" << std::endl;
		if (stats.no_chimeric_reads) fail(no_chimeric_reads);
	}
	if (stats.missing_hi_tag > 0) std::cerr << "WARNING: " << stats.missing_hi_tag << " secondary alignments lack the 'HI' tag and were ignored (STAR must be run with '--outSAMattributes HI' for Arriba to make use of multi-mapping reads for fusion detection)" << std::endl;

	// ---- the host's copy of the table (fragment length, strandedness, the mate swaps, the writer, the broadcast of a sharded run read it) ----
	const u32 n = (u32) sizes[0];
	out.n = n;
	out.n_aln.resize(n); out.fflags.resize(n); out.filter.resize(n);
	out.contig.resize(3 * (size_t) n); out.start.resize(3 * (size_t) n); out.end.resize(3 * (size_t) n); out.aflags.resize(3 * (size_t) n);
	out.cigar_off.resize(3 * (size_t) n); out.cigar_cnt.resize(3 * (size_t) n); out.seq_off.resize(2 * (size_t) n); out.seq_len.resize(2 * (size_t) n);
	out.genes_off.resize(3 * (size_t) n); out.genes_cnt.resize(3 * (size_t) n);
	out.cigar.resize(sizes[2] + 1); out.seq.resize(sizes[3]); out.names.resize(sizes[4]); out.name_off.resize((size_t) n + 1);
	{
		arb_soa_chunk c;
		c.n_fragments = n; c.n_aln = out.n_aln.data(); c.fflags = out.fflags.data(); c.filter = out.filter.data();
		c.contig = out.contig.data(); c.start = out.start.data(); c.end = out.end.data(); c.aflags = out.aflags.data();
		c.cigar_off = out.cigar_off.data(); c.cigar_cnt = out.cigar_cnt.data(); c.seq_off = out.seq_off.data(); c.seq_len = out.seq_len.data();
		c.genes_off = out.genes_off.data(); c.genes_cnt = out.genes_cnt.data();
		c.cigar = out.cigar.data(); c.n_cigar = out.cigar.size(); c.seq = out.seq.data(); c.n_seq_bytes = out.seq.size(); c.genes = NULL; c.n_genes = 0;
		check(arb_fragment_table_download(ctx, &c, out.names.data(), out.name_off.data()), "arb_fragment_table_download");
	}
	stats.t_finalize = now_s() - tf;
	lap("table -> host");
}

}} // namespace
