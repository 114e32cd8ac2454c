"""Plain reference of the re-alignment stage (`filter_mismappers`) and of the gene homology test (`is_homolog`), written from the
reference's semantics (filter_mismappers.cpp:33-359, filter_homologs.cpp:13-63) and independent of the product: nothing here imports
arriba_b200, and the search is the reference's recursion, not the product's passes.

Contigs are Python strings of upper-case characters, reads strings over the nt16 alphabet "=ACMGRSVTWYHKDBN". Float arithmetic is done in
float32 (np.float32) exactly where the reference computes in float, and in double (Python float) where it promotes."""
import bisect
import functools
import sys
import numpy as np
from seqrules import reverse_complement

KMER = 8
F32 = np.float32
MIN_ALIGN_FRACTION = F32(0.8)            # filter_mismappers.cpp:274
MIN_EXTENDED_ALIGN_FRACTION = F32(0.7)   # filter_mismappers.cpp:275
F_NONE, F_MISMAPPERS = 0, 11

sys.setrecursionlimit(max(sys.getrecursionlimit(), 20000))   # a continuation per splice site / first mismatch nests one level


# ------------------------------------------------------------------------------------------------ the k-mer index
_BASE2 = np.full(256, 3, np.int64)
for _c, _v in (("T", 0), ("G", 1), ("C", 2)):
    _BASE2[ord(_c)] = _v


def kmer_to_int(s, pos):
    """filter_mismappers.cpp:33-45: T=0 G=1 C=2, every other character (A, N, IUPAC codes, anything else) 3."""
    r = 0
    for c in s[pos:pos + KMER]:
        r = r << 2 | (0 if c == "T" else 1 if c == "G" else 2 if c == "C" else 3)
    return r


def index_intervals(genes, padding, contig_len):
    """Intervals [start, end) of indexed positions the way the host derives them from the genes of the candidates (events.cpp:616-636,
    after filter_mismappers.cpp:61-74): a position p of the padded gene [gs, ge] is a candidate while p + 8 < ge. `genes`: (contig, start,
    end) triples. Overlapping intervals of one contig are merged."""
    padding = max(padding, 0)
    ivs = []
    for c, s, e in genes:
        gs, ge = max(s - padding, 0), min(e + padding, contig_len[c] - 1)
        if gs + KMER < ge:
            ivs.append((c, gs, ge - KMER))
    ivs.sort()
    out = []
    for c, s, e in ivs:
        if out and out[-1][0] == c and s <= out[-1][2]:
            out[-1][2] = max(out[-1][2], e)
        else:
            out.append([c, s, e])
    return [tuple(x) for x in out]


class KmerIndex:
    """make_kmer_index (filter_mismappers.cpp:47-84) over given intervals: a position is indexed when its first base is not 'N'; the hits of
    one (contig, 8-mer) are sorted and unique. Kept as one array sorted by (contig << 16 | 8-mer, position), so that bucket bounds and lower
    bounds are np.searchsorted calls, and as per-contig dicts {8-mer: list of positions} for the search."""

    def __init__(self, contigs, intervals, n_index_contigs):
        self.n_index_contigs = n_index_contigs
        keys, poss = [], []
        for c, s, e in intervals:
            if e <= s:
                continue
            a = np.frombuffer(contigs[c].encode(), np.uint8)
            p = np.arange(s, e, dtype=np.int64)
            code = _BASE2[a]
            k = np.zeros(len(p), np.int64)
            for b in range(KMER):
                k = k << 2 | code[p + b]
            keep = a[p] != ord("N")
            keys.append((c << 16) | k[keep]); poss.append(p[keep])
        key = np.concatenate(keys) if keys else np.zeros(0, np.int64)
        pos = np.concatenate(poss) if poss else np.zeros(0, np.int64)
        order = np.lexsort((pos, key))
        key, pos = key[order], pos[order]
        if len(key):
            uniq = np.ones(len(key), bool); uniq[1:] = (key[1:] != key[:-1]) | (pos[1:] != pos[:-1])
            key, pos = key[uniq], pos[uniq]
        self.key, self.pos = key, pos
        self.by_contig = [dict() for _ in range(n_index_contigs)]
        if len(key):
            cut = np.nonzero(np.diff(key))[0] + 1
            for ks, ps in zip(np.split(key, cut), np.split(pos, cut)):
                c = int(ks[0]) >> 16
                if c < n_index_contigs:
                    self.by_contig[c][int(ks[0]) & 0xFFFF] = ps.tolist()

    def lookup(self, contig, kmer, bound):
        """(lo, hi) of the bucket in the sorted array and the index of the first hit >= bound (hi if none)."""
        k = contig << 16 | kmer
        lo = int(np.searchsorted(self.key, k, "left")); hi = int(np.searchsorted(self.key, k, "right"))
        return lo, hi, lo + int(np.searchsorted(self.pos[lo:hi], bound, "left"))


# ------------------------------------------------------------------------------------------------ align (filter_mismappers.cpp:86-187)
def make_align(read, contig, gene_start, gene_end, kmer_index, splice_sites, min_score, memo=True):
    """align(score, read_pos, gene_pos, max_deletions) of one read against one window [gene_start, gene_end] of `contig`. Everything but
    those four arguments is fixed, so the recursion is a pure function of them and memoizing it is exact."""
    n = len(read)
    kmers = [kmer_to_int(read, p) for p in range(max(n - KMER, 0))]
    splice = list(splice_sites)

    def align(score, read_pos, gene_pos, max_deletions):
        skipped_bases = 0
        while read_pos + KMER < n and read_pos + min_score <= n + score + 2 * KMER:   # :90-94
            hits = kmer_index.get(kmers[read_pos])
            if hits is not None:
                for i in range(bisect.bisect_left(hits, gene_pos), len(hits)):        # :100, lower_bound(gene_pos) and *kmer_hit < gene_end
                    hit = hits[i]
                    if hit >= gene_end:
                        break
                    extended_score = score + KMER
                    if read_pos == skipped_bases:          # every base before the seed was skipped: no penalty for them (:103-104)
                        extended_score += skipped_bases
                    if extended_score >= min_score:
                        return True
                    # left: over the skipped bases, one mismatch allowed, +1 (leading) or +2 per match (:109-137)
                    r, g, mismatch_count = read_pos - 1, hit - 1, 0
                    while r >= read_pos - skipped_bases and g >= gene_start:
                        if read[r] == contig[g]:
                            extended_score += 1 if read_pos == skipped_bases else 2
                            if extended_score >= min_score:
                                return True
                        else:
                            mismatch_count += 1
                            if mismatch_count > 1:
                                break
                        r -= 1; g -= 1
                    # right: spliced continuation at a splice site, one deletion at the first mismatch, 4 consecutive mismatches stop (:140-181)
                    r, g = read_pos + KMER, hit + KMER
                    mismatch_count = consecutive = 0
                    ns = bisect.bisect_left(splice, g - 1)
                    while r < n and g <= gene_end:
                        if ns < len(splice):
                            if g - 1 > splice[ns]:
                                ns += 1
                            if ns < len(splice) and g - 1 == splice[ns]:
                                if align(extended_score, r, g, max_deletions):
                                    return True
                        if read[r] == contig[g]:
                            extended_score += 1
                            if extended_score >= min_score:
                                return True
                            consecutive = 0
                        else:
                            mismatch_count += 1
                            if mismatch_count == 1 and max_deletions > 0 and n >= 30 and align(extended_score, r, g, max_deletions - 1):
                                return True
                            extended_score -= 1
                            consecutive += 1
                            if consecutive >= 4:
                                break
                        r += 1; g += 1
            read_pos += 1; score -= 1; skipped_bases += 1
        return False

    if memo:
        align = functools.lru_cache(maxsize=None)(align)
    return align


def min_score_of(fraction, length):
    """int min_score = min_align_fraction * read_sequence.size() + 0.5 (:195): float product, double sum, truncation toward zero."""
    return int(float(F32(fraction) * F32(length)) + 0.5)


def discordant_fraction(pre, post, size):
    """min(min_align_fraction, min_align_fraction * (1 - clipped_fraction)), clipped_fraction = ((float) pre + post) / size (:326-330)."""
    clipped = (F32(pre) + F32(post)) / F32(size)
    return min(MIN_ALIGN_FRACTION, MIN_ALIGN_FRACTION * (F32(1) - clipped))


class Stage:
    """The genome, genes, splice sites and k-mer index one filter_mismappers / filter_homologs run sees."""

    def __init__(self, contigs, genes, splice_sites, kmer_index, max_mate_gap):
        self.contigs = contigs               # list of str
        self.genes = genes                   # list of (contig, start, end, strand) with strand True = forward
        self.splice = splice_sites           # per gene: sorted list of downstream splice sites
        self.index = kmer_index
        self.max_mate_gap = max_mate_gap

    def window(self, g, read_length):
        c, s, e, _ = self.genes[g]
        return max(s - self.max_mate_gap - read_length, 0), min(e + self.max_mate_gap + read_length, len(self.contigs[c]) - 1)

    def align_both_strands(self, read, read_length, same_contig, aln_start, aln_end, genes, fraction, memo=True):
        """filter_mismappers.cpp:189-230."""
        if len(read) >= 300:
            return False
        min_score = min_score_of(fraction, len(read))
        for g in genes:
            c = self.genes[g][0]
            ws, we = self.window(g, read_length)
            if same_contig and (ws <= aln_start <= we or ws <= aln_end <= we):
                continue
            if c >= self.index.n_index_contigs:
                continue
            for seq in (read, reverse_complement(read)):
                if make_align(seq, self.contigs[c], ws, we, self.index.by_contig[c], self.splice[g], min_score, memo)(0, 0, ws, 1):
                    return True
        return False

    def extend_split_read(self, sr, read):
        """filter_mismappers.cpp:247-270. `sr`: the split read's alignment (contig, start, end, forward, cigar). A reverse split read that
        ends on the contig's last base makes clipped_count negative: substr then takes the whole clipped segment and nothing of the contig.
        The reference then compares the segment with an empty string: base 0 meets its terminating '\\0', which no base matches, and the
        bases after it read past the string, which is undefined. This model counts them as mismatches too: a choice, the same one the product
        makes, under which a clip of two bases or more is then never extended."""
        contig = self.contigs[sr["contig"]]
        pre, post = clips(sr["cigar"])
        if sr["forward"]:
            n = min(pre, sr["start"])
            clipped, ref = read[pre - n:pre], contig[sr["start"] - n:sr["start"]]
        else:
            n = min(post, len(contig) - sr["end"] - 2)
            start = len(read) - post
            clipped = read[start:] if n < 0 else read[start:start + n]
            ref = contig[sr["end"] + 1:] if n < 0 else contig[sr["end"] + 1:sr["end"] + 1 + n]
        matching = sum(1 for i, c in enumerate(clipped) if i < len(ref) and c == ref[i])
        return matching >= float(np.floor(F32(len(clipped)) * MIN_EXTENDED_ALIGN_FRACTION))

    def fragment_is_mismapper(self, frag, kind, same_contig, memo=True):
        """The verdict on one listed fragment of a candidate (:289-333); kind 0 = split read, 1 = discordant mates."""
        a, s = frag["alignments"], frag["sequences"]
        if kind == 0:
            mate1, sr, sup = a[0], a[1], a[2]
            r0, r1 = s[0], s[1]
            pre, post = clips(sr["cigar"])
            mpre, mpost = clips(mate1["cigar"])
            if self.extend_split_read(sr, r1):
                return True
            if sr["forward"]:
                seg0, seg1 = r1[:pre], r0[mpre:]
            else:
                seg0, seg1 = r1[len(r1) - post:], r0[:len(r0) - mpost]
            return (self.align_both_strands(seg0, len(r1), same_contig, sup["start"], sup["end"], sr["genes"], MIN_ALIGN_FRACTION, memo) or
                    self.align_both_strands(seg1, len(r0), same_contig, mate1["start"], mate1["end"], sup["genes"], MIN_ALIGN_FRACTION, memo))
        m1, m2 = a[0], a[1]
        f1 = discordant_fraction(*clips(m1["cigar"]), len(s[0]))
        f2 = discordant_fraction(*clips(m2["cigar"]), len(s[1]))
        return (self.align_both_strands(s[0], len(s[0]), same_contig, m1["start"], m1["end"], m2["genes"], f1, memo) or
                self.align_both_strands(s[1], len(s[1]), same_contig, m2["start"], m2["end"], m1["genes"], f2, memo))


def clips(cigar):
    """(preclipping, postclipping): the length of a leading / trailing S or H operation (common.hpp:205-206)."""
    pre = cigar[0][1] if cigar[0][0] in "SH" else 0
    post = cigar[-1][1] if cigar[-1][0] in "SH" else 0
    return pre, post


def count_mismappers(lst, labels, mismappers, total_reads, supporting_reads):
    """filter_mismappers.cpp:232-244, counters in unsigned short."""
    for i in lst:
        if labels[i] == F_NONE:
            total_reads = (total_reads + 1) & 0xFFFF
        elif labels[i] == F_MISMAPPERS:
            total_reads = (total_reads + 1) & 0xFFFF
            mismappers = (mismappers + 1) & 0xFFFF
            if supporting_reads > 0:
                supporting_reads -= 1
    return supporting_reads, mismappers, total_reads


def filter_mismappers(stage, frags, cands, labels, max_mismapper_fraction, verdict=None):
    """filter_mismappers.cpp:272-359 over candidates `cands` (dict of columns with lists list1 / list2 / listd per candidate) and fragment
    labels `labels`; returns (labels, filter, split_reads1, split_reads2, discordant_mates). Read counts are 15-bit fields
    (common.hpp:240-242) and must be given below 2^15. `verdict(i, kind, same_contig)` may replace fragment_is_mismapper (a cache)."""
    labels = np.array(labels, np.uint8)
    flt = np.array(cands["filter"], np.uint8)
    sr1, sr2, dm = (np.array(cands[k], np.int64) for k in ("split_reads1", "split_reads2", "discordant_mates"))
    verdict = verdict or (lambda i, kind, same: stage.fragment_is_mismapper(frags[i], kind, same))
    for c in range(len(flt)):
        if flt[c] != F_NONE:
            continue
        same = cands["contig1"][c] == cands["contig2"][c]
        for lst, kind in ((cands["list1"][c], 0), (cands["list2"][c], 0), (cands["listd"][c], 1)):
            for i in lst:
                if labels[i] == F_NONE and verdict(i, kind, same):
                    labels[i] = F_MISMAPPERS
    for c in range(len(flt)):
        if flt[c] != F_NONE:
            continue
        mism = total = 0
        sr1[c], mism, total = count_mismappers(cands["list1"][c], labels, mism, total, int(sr1[c]))
        sr2[c], mism, total = count_mismappers(cands["list2"][c], labels, mism, total, int(sr2[c]))
        dm[c], mism, total = count_mismappers(cands["listd"][c], labels, mism, total, int(dm[c]))
        if mism > 0 and mism >= float(np.floor(F32(max_mismapper_fraction) * F32(total))):
            flt[c] = F_MISMAPPERS
    return labels, flt, sr1, sr2, dm


# ------------------------------------------------------------------------------------------------ is_homolog (filter_homologs.cpp:13-63)
def is_homolog(stage, g1, g2, max_identity):
    if g1 == g2:
        return False
    small, big = stage.genes[g1], stage.genes[g2]
    if small[2] - small[1] > big[2] - big[1]:     # length() = end - start; on equal lengths gene1 is the small gene
        small, big = big, small
    sc, ss, se, sstrand = small
    bc, bs, be, bstrand = big
    if sc == bc and (bs <= ss <= be or bs <= se <= be):
        return False
    length = se - ss
    seq = stage.contigs[sc][ss:ss + length]
    if sstrand != bstrand:
        seq = reverse_complement(seq)
    threshold = F32(length) * F32(max_identity)
    index = stage.index.by_contig[bc]
    bref = stage.contigs[bc]
    matching = 0
    pos = 0
    while pos + 2 * KMER < len(seq):
        if F32(matching * KMER + (len(seq) - pos)) < threshold:
            return False
        hits = index.get(kmer_to_int(seq, pos))
        if hits is not None:
            for i in range(bisect.bisect_left(hits, bs), len(hits)):
                hit = hits[i]
                if hit > be:
                    break
                if sc != bc or hit < ss or hit > se:
                    # strncmp over 8 characters: past the big contig's end its '\0' matches no base of the small gene
                    if bref[hit + KMER:hit + 2 * KMER] == seq[pos + KMER:pos + 2 * KMER]:
                        matching += 1
                        if F32(matching * KMER) >= threshold:
                            return True
                        break
        pos += KMER
    return False
