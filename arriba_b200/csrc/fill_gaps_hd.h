// fill_gaps_hd.h -- gap filling of the fusion transcript sequence (-I): one job fills one side of one row's sequence with the exons of one transcript.
//
// Behavioural contract: fill_gaps_in_fusion_transcript_sequence (output_fusions.cpp:820-1041). The 5' part rewrites only the characters before the first '|',
// the 3' part only those after the last '|', and neither writes a '|' (the assembly's bases are upper-cased letters). So a row's filled sequence for the pair
// (t5, t3) is P5(t5) + seq[b5 .. b3] + S3(t3): a job returns P5, the replacement of seq[0, b5), or S3, the replacement of seq(b3, end), with the positions of
// its characters. A job is planned by one thread (fill_plan_fn: the case, the gap, the overlapping exon, the output length), the lengths are scanned, and one
// team of threads writes each job (fill_emit): the exons' bases in strided, coalesced stores.
//
// The cases of one side, as the reference tells them apart:
//   COPY  the side is left as it is (no overlapping exon, an imprecise breakpoint that may not be snapped, a contig without sequence), or trimmed to the
//         transcript when the transcribed bases cover its end ("^" before a 5' side that reaches the start, "$" after a 3' side that reaches the end);
//   FILL  5': [^] "(" walk [fake] ")" seq[c0, c1)     -- walk: the transcript's exons from its start up to (not including) the target position;
//         3': seq[c0, c1) "(" [fake] walk ")" [$]     -- walk: from the overlapping exon to the transcript's end, after the target position.
//         Exons are separated by "___"; fake is the base of the exon boundary that stands in for an imprecise breakpoint ("...|" / "|...").
#pragma once
#include "model.h"
#include "prims.h"

namespace arb {

enum { FJ_THREE = 1, FJ_FORWARD = 2, FJ_ITD = 4 }; // job flags: the 3' side (else 5'), the side's predicted strand is forward, the row is an ITD
enum { FK_COPY = 0, FK_FILL = 1 };

struct fill_transcripts { // the transcript table of the resident annotation
	const i32* first_exon; const i32* last_exon; const u32* contig; u32 n;
	const i32* exon_next; const i32* exon_prev; // -1: none
};
struct fill_jobs {
	// the rows' unfilled sequences and the positions of their characters: the positions of a row may run longer than its text (the consensus keeps a
	// position for the bases of an insertion that went to the clipped part, output_fusions.cpp:187-190); they are indexed like the text all the same
	const char* text; const u32* row_off; const i32* pos; const u32* pos_off;
	const u32* row; const u32* transcript; const u8* flags; u32 n;
};
struct fill_plan {
	u32 kind, len; u32 c0, c1;   // kind, output length, copied range of the row's text
	i32 target, walk_exon;       // FILL: the walk's target position and first exon
	i32 fake_pos; char fake;     // FILL of an imprecise breakpoint: the fake base (fake != 0)
	u8 mark;                     // '^' / '$' or 0
};

ARB_HD char fill_complement(char c) { // assembly.hpp:9-22
	switch (c) {
		case 'a': return 't'; case 't': return 'a'; case 'c': return 'g'; case 'g': return 'c';
		case 'A': return 'T'; case 'T': return 'A'; case 'C': return 'G'; case 'G': return 'C';
		case '[': return ']'; case ']': return '['; default: return c;
	}
}

// The walk over the exons of a FILL: seg(first position, count, step) for a run of bases, sep() for "___". Returns false when a base lies outside the contig.
template <class SEG, class SEP> ARB_HD bool fill_walk(const annot_view& an, const fill_transcripts& tr, bool three, bool fwd, i32 exon, i32 target, i64 contig_len, SEG seg, SEP sep) {
	auto inside = [&](i32 lo, i32 hi) { return lo > hi || (lo >= 0 && (i64) hi < contig_len); };
	if (!three) { // output_fusions.cpp:895-905: from the transcript's start up to the target
		for (i32 ex = exon; ex >= 0; ex = fwd ? tr.exon_next[ex] : tr.exon_prev[ex]) {
			const i32 s = an.exon_start[ex], e = an.exon_end[ex];
			if (s <= target && target <= e) {
				const u32 n = (u32) (fwd ? target - s : e - target);
				if (n && !inside(fwd ? s : target + 1, fwd ? target - 1 : e)) return false;
				if (n) seg(fwd ? s : e, n, fwd ? 1 : -1);
				return true;
			}
			const u32 n = s <= e ? (u32) (e - s + 1) : 0u;
			if (n && !inside(s, e)) return false;
			if (n) seg(fwd ? s : e, n, fwd ? 1 : -1);
			const i32 after = s <= e ? (fwd ? e + 1 : s - 1) : (fwd ? s : e); // where the reference's loop variable stops
			if (after == target) return true;
			sep();
		}
		return true;
	}
	for (i32 ex = exon; ex >= 0; ex = fwd ? tr.exon_next[ex] : tr.exon_prev[ex]) { // output_fusions.cpp:1005-1014: from the overlapping exon to the end
		const i32 s = an.exon_start[ex], e = an.exon_end[ex];
		if (fwd) { const i32 p0 = hd_max(s, target + 1); if (p0 <= e) { if (!inside(p0, e)) return false; seg(p0, (u32) (e - p0 + 1), 1); } }
		else { const i32 p0 = hd_min(e, target - 1); if (p0 >= s) { if (!inside(s, p0)) return false; seg(p0, (u32) (p0 - s + 1), -1); } }
		if ((fwd ? tr.exon_next[ex] : tr.exon_prev[ex]) >= 0) sep();
	}
	return true;
}

// one thread per job: the case and the output length; bad[0] = the lowest job whose walk leaves its contig (the reference would index out of range)
struct fill_plan_fn {
	annot_view an; fill_transcripts tr; fill_jobs jobs; fill_plan* plan; u32* len; u32* bad;
	ARB_HD void operator()(u32 j) const {
		const u32 r = jobs.row[j], off = jobs.row_off[r], size = jobs.row_off[r + 1] - off, n_pos = jobs.pos_off[r + 1] - jobs.pos_off[r];
		const char* seq = jobs.text + off; const i32* pos = jobs.pos + jobs.pos_off[r];
		const u32 t = jobs.transcript[j]; const bool three = jobs.flags[j] & FJ_THREE, fwd = jobs.flags[j] & FJ_FORWARD, itd = jobs.flags[j] & FJ_ITD;
		const i32 first = tr.first_exon[t], last = tr.last_exon[t];
		const i32 t_start = an.exon_start[first], t_end = an.exon_end[last];
		fill_plan p; p.kind = FK_COPY; p.target = -1; p.walk_exon = -1; p.fake_pos = -1; p.fake = 0; p.mark = 0;
		// the sides: seq[0, b5) and seq(b3, size); a row without '|' has no jobs
		u32 b5 = 0; while (b5 < size && seq[b5] != '|') ++b5;
		u32 b3 = size; while (b3 > 0 && seq[b3 - 1] != '|') --b3; b3 = b3 > 0 ? b3 - 1 : size;
		if (three) { p.c0 = b3 + 1; p.c1 = size; } else { p.c0 = 0; p.c1 = b5; }
		const u32 c = tr.contig[t];
		const u64 seq_off = an.contig_seq_off[c];
		const i64 contig_len = (i64) an.contig_len[c]; // 0: the contig has no sequence (arb_set_contigs)
		auto exon_at = [&](i32 x) { for (i32 ex = first; ex >= 0; ex = tr.exon_next[ex]) if (x >= an.exon_start[ex] && x <= an.exon_end[ex]) return ex; return (i32) -1; };
		bool imprecise = false; u32 gap = 0; bool trim = false;
		if (contig_len == 0) { /* contig without sequence: left as it is (output_fusions.cpp:825-826, 935-936) */ }
		else if (!three) { // output_fusions.cpp:829-861
			const u32 bp = b5;
			u32 g = bp < size ? bp : size - 1; bool found = false; // find_last_of('.', bp)
			for (;; --g) { if (seq[g] == '.') { found = true; break; } if (g == 0) break; }
			if (found && g + 1 == bp && g >= 3) { imprecise = true; gap = g - 3; }
			else if (found && pos[g + 1] > t_start && pos[g + 1] < t_end) gap = g + 1;
			else if (!found && pos[0] > t_start && pos[0] < t_end) gap = 0;
			else trim = true;
			if (trim) {
				u32 i0 = 0;
				for (u32 i = 0; i < bp; ++i) if (pos[i] >= t_start && pos[i] <= t_end) { i0 = i; break; }
				p.c0 = i0;
				if ((fwd && pos[i0] == t_start) || (!fwd && pos[i0] == t_end)) p.mark = '^';
			} else {
				i32 ov = -1;
				for (; gap != bp; ++gap) { ov = exon_at(pos[gap]); if (ov >= 0) break; }
				bool ok = ov >= 0;
				if (imprecise && ((fwd && ov == last) || (!fwd && ov == first) || itd)) ok = false;
				if (ok) {
					p.kind = FK_FILL; p.walk_exon = fwd ? first : last;
					if (imprecise) {
						p.fake_pos = fwd ? an.exon_end[ov] : an.exon_start[ov];
						if (p.fake_pos < 0 || (i64) p.fake_pos >= contig_len) { atomic_min_u32(bad, j); p.kind = FK_COPY; }
						else { const char b = an.assembly[seq_off + (u64) p.fake_pos]; p.fake = fwd ? b : fill_complement(b); }
						p.target = p.fake_pos; gap = bp;
					} else p.target = pos[gap];
					p.c0 = gap;
				}
			}
		} else { // output_fusions.cpp:939-971
			const u32 bp = b3;
			u32 g = size; for (u32 i = bp; i + 2 < size; ++i) if (seq[i] == '.' && seq[i + 1] == '.' && seq[i + 2] == '.') { g = i; break; } // find("...", bp)
			const bool found = g < size;
			if (found && g - 1 == bp && g + 3 < size) { imprecise = true; gap = g + 3; }
			else if (found && pos[g - 1] > t_start && pos[g - 1] < t_end) gap = g - 1;
			else if (!found && pos[size - 1] > t_start && pos[size - 1] < t_end) gap = size - 1;
			else trim = true;
			if (trim) {
				u32 i1 = size - 1;
				for (u32 i = size - 1; i > bp; --i) if (pos[i] >= t_start && pos[i] <= t_end) { i1 = i; break; }
				p.c1 = i1 + 1;
				const i32 back = i1 + 1 < size ? pos[i1] : pos[n_pos - 1]; // the last position of the vector: without a cut, the positions beyond the text stay
				if ((fwd && back == t_end) || (!fwd && back == t_start)) p.mark = '$';
			} else {
				i32 ov = -1;
				for (; gap != bp; --gap) { ov = exon_at(pos[gap]); if (ov >= 0) break; }
				bool ok = ov >= 0;
				if (imprecise && ((fwd && ov == last) || (!fwd && ov == first) || itd)) ok = false;
				if (ok) {
					p.kind = FK_FILL; p.walk_exon = ov;
					if (imprecise) {
						p.fake_pos = fwd ? an.exon_start[ov] : an.exon_end[ov];
						if (p.fake_pos < 0 || (i64) p.fake_pos >= contig_len) { atomic_min_u32(bad, j); p.kind = FK_COPY; }
						else { const char b = an.assembly[seq_off + (u64) p.fake_pos]; p.fake = fwd ? b : fill_complement(b); }
						p.target = p.fake_pos; p.c1 = p.c0; // the fake base moves inside the parentheses (the swap at :1027-1030)
					} else { p.target = pos[gap]; p.c1 = gap + 1; }
				}
			}
		}
		u32 n = p.c1 - p.c0 + (p.mark ? 1u : 0u);
		if (p.kind == FK_FILL) {
			u32 walked = 0; i32 last_pos = -2; bool any_sep = false;
			const bool ok = fill_walk(an, tr, three, fwd, p.walk_exon, p.target, contig_len,
			                          [&](i32 from, u32 k, i32 step) { if (!walked && !three) last_pos = from; walked += k; last_pos = three ? from + step * (i32) (k - 1) : last_pos; any_sep = false; },
			                          [&]() { walked += 3; if (three) any_sep = true; });
			if (!ok) { atomic_min_u32(bad, j); p.kind = FK_COPY; p.mark = 0; n = p.c1 - p.c0; }
			else {
				n += 2 + walked + (p.fake ? 1u : 0u);
				// '^': the character after "(" is the transcript's first base (output_fusions.cpp:923-927); '$': the one before ")" its last (:1033-1037)
				if (!three) {
					const i32 second = walked ? (last_pos == -2 ? -1 : last_pos) : (p.fake ? p.fake_pos : -1);
					if ((fwd && second == t_start) || (!fwd && second == t_end)) { p.mark = '^'; ++n; }
				} else {
					const i32 before = walked ? (any_sep || last_pos == -2 ? -1 : last_pos) : (p.fake ? p.fake_pos : -1);
					if ((fwd && before == t_end) || (!fwd && before == t_start)) { p.mark = '$'; ++n; }
				}
			}
		}
		p.len = n; plan[j] = p; len[j] = n;
	}
};

// one team per job: the output of a plan at out[off[j] ..)
struct fill_emit_fn {
	annot_view an; fill_transcripts tr; fill_jobs jobs; const fill_plan* plan; const u32* off; char* chars; i32* pos;
	ARB_HD void run(u32 j, u32 rank, u32 size) const {
		const fill_plan p = plan[j];
		const u32 r = jobs.row[j], roff = jobs.row_off[r], poff = jobs.pos_off[r];
		const bool three = jobs.flags[j] & FJ_THREE, fwd = jobs.flags[j] & FJ_FORWARD;
		u32 o = off[j];
		auto put = [&](char c, i32 x) { if (rank == 0) { chars[o] = c; pos[o] = x; } ++o; };
		auto copy = [&]() { const u32 n = p.c1 - p.c0; for (u32 k = rank; k < n; k += size) { chars[o + k] = jobs.text[roff + p.c0 + k]; pos[o + k] = jobs.pos[poff + p.c0 + k]; } o += n; };
		if (p.kind == FK_COPY) { if (p.mark && !three) put('^', -1); copy(); if (p.mark && three) put('$', -1); return; }
		const u64 base = an.contig_seq_off[tr.contig[jobs.transcript[j]]];
		if (three) { copy(); put('(', -1); if (p.fake) put(p.fake, p.fake_pos); }
		else { if (p.mark) put('^', -1); put('(', -1); }
		fill_walk(an, tr, three, fwd, p.walk_exon, p.target, (i64) 1 << 62,
		          [&](i32 from, u32 k, i32 step) {
		              for (u32 x = rank; x < k; x += size) { const i32 q = from + step * (i32) x; const char b = an.assembly[base + (u64) q]; chars[o + x] = fwd ? b : fill_complement(b); pos[o + x] = q; }
		              o += k;
		          },
		          [&]() { put('_', -1); put('_', -1); put('_', -1); });
		if (three) { put(')', -1); if (p.mark) put('$', -1); }
		else { if (p.fake) put(p.fake, p.fake_pos); put(')', -1); copy(); }
	}
};

} // namespace arb
