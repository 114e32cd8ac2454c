// ingest.h -- chimeric BAM ingest: BGZF inflate on host threads, the record loop on the device, into structure-of-arrays fragment columns
// (arb_soa_chunk layout, fragments in name order), plus the by-products the later stages need (mapped read count,
// coverage windows). Behavioural contract: read_chimeric_alignments (read_chimeric_alignments.cpp:560-773) and helpers
// (:19-558), mark_multimappers (:792-802), coverage_t (read_stats.cpp:148-306). Input: BAM or SAM text (-x), STAR "WithinBAM" or, with
// STAR's Chimeric.out.sam (-c) read first, "SeparateSAMold"; CRAM is not read.
#pragma once
#include <string>
#include <vector>
#include <cstdlib>
#include <memory>
#include <utility>
#include <new>
#include <functional>
#include "refdata.h"
struct arb_ctx;

namespace arb { namespace host {

struct coverage_windows { // 20 bp windows (read_stats.hpp:14)
	std::vector<std::vector<u16> > coverage;
	std::vector<std::vector<u8> > starts, ends;
	void resize(const refdata& ref);
	bool fragment_starts_here(u32 contig, i32 start, i32 end) const;
	bool fragment_ends_here(u32 contig, i32 start, i32 end) const;
	int get_coverage(u32 contig, i32 position, u32 direction) const;
};

// Large host blocks are recycled inside the process: the first touch of fresh pages costs ~2 us per 4 KiB page on the measured hosts (more than filling
// them), and a process that runs sample after sample would pay it for gigabytes of columns every time. Blocks of 1 MiB and more go back to a free list per
// size class (steps of 25 %) instead of the C library; host_block_trim() (arb_release_host_memory) hands them to the system.
void* host_block_get(size_t bytes, size_t& granted);
void host_block_put(void* p, size_t granted);
void host_block_trim();
// where fresh blocks come from (default: malloc). The CUDA library installs page-locked blocks on 2 MiB pages (capi.cu); a NULL result falls back to malloc.
void set_host_block_backend(void* (*alloc)(size_t), void (*release)(void*));

// vector whose resize() leaves new elements uninitialised: the large columns are first touched (and zeroed where needed) by the threads that fill them
template <class T> struct default_init_allocator {
	typedef T value_type;
	template <class U> struct rebind { typedef default_init_allocator<U> other; };
	default_init_allocator() {}
	template <class U> default_init_allocator(const default_init_allocator<U>&) {}
	static size_t class_of(size_t bytes) { size_t c = (size_t) 1 << 20; while (c < bytes) c += c / 4; return c; }
	T* allocate(size_t n) {
		const size_t bytes = n * sizeof(T);
		void* p;
		if (bytes >= ((size_t) 1 << 20)) { size_t granted; p = host_block_get(class_of(bytes), granted); }
		else p = malloc(bytes ? bytes : 1);
		if (!p) throw std::bad_alloc();
		return (T*) p;
	}
	void deallocate(T* p, size_t n) { const size_t bytes = n * sizeof(T); if (bytes >= ((size_t) 1 << 20)) host_block_put(p, class_of(bytes)); else free(p); }
	template <class U> void construct(U* p) { ::new ((void*) p) U; }
	template <class U, class A0, class... A> void construct(U* p, A0&& a0, A&&... a) { ::new ((void*) p) U(std::forward<A0>(a0), std::forward<A>(a)...); }
	template <class U> bool operator==(const default_init_allocator<U>&) const { return true; }
	template <class U> bool operator!=(const default_init_allocator<U>&) const { return false; }
};
template <class T> using column = std::vector<T, default_init_allocator<T> >;

struct fragment_table { // host image of arb_soa_chunk + names
	u32 n;
	column<u8> n_aln, fflags, filter, aflags;
	column<u16> contig, cigar_cnt, seq_len, genes_cnt;
	column<i32> start, end;
	column<u32> cigar_off, seq_off, genes_off, cigar, genes;
	column<u8> seq;
	column<char> names; column<u64> name_off; // "<qname>,<HI>[ITD]" per fragment, name order
	fragment_table(): n(0) {}
	frag_view view();
	std::string name(u32 i) const { return std::string(names.data() + name_off[i], names.data() + name_off[i + 1]); }
};

struct ingest_stats {
	u64 mapped_reads; std::vector<u64> mapped_viral_reads_by_contig; u64 malformed, missing_hi_tag, records, multimapper_pairs /* neighbours with the same read name */; bool no_chimeric_reads;
	u64 chimeric_records, chimeric_malformed, chimeric_total; // the -c file: records, fragments the first malformed pass rejected / kept (0 without one)
	double t_inflate, t_parse, t_finalize;
};

struct ingest_options {
	bool external_duplicate_marking; u32 max_itd_length; std::string interesting_contigs, viral_contigs; int threads /* inflate */;
	struct ::arb_ctx* scan_ctx; // device context that runs the record loop and builds the fragment table
	std::function<void()> after_header; // once the BAM header has grown the contig table: the contigs and the gene index must reach scan_ctx before the records
	std::string chimeric_path; // -c file, read before the main file (empty: none)
	std::function<void(u64)> chimeric_done; // with a -c file: its part is complete (no error of it is left); the argument is its progress line's total
};

// reads the BAM, fills `out` (name order, slots normalised, multimappers marked); throws std::runtime_error on fatal input errors
void read_chimeric_alignments(const std::string& bam_path, refdata& ref, const ingest_options& opt, fragment_table& out, coverage_windows& coverage, ingest_stats& stats);

}} // namespace
