"""A world for the re-alignment stage and the gene homology test, built directly as arb_soa_chunk / arb_annotation / arb_contigs dicts
(no synthetic BAM, no oracle run).

Genome: a contig of more than two 2^17-base blocks of the k-mer block table with gene windows across both block boundaries, a short contig
whose gene window is clamped at 0 and at the last base, a contig of tandem repeats (periods 1-6 and 20-50), and a contig with genes beyond
the indexed contigs; N runs and IUPAC codes; no length a multiple of 8. A second variant adds one 'X', which turns the packed reference off.

Fragments come mostly as twins: a one-parameter family of shapes (mutations applied one by one, a placement shifted base by base across a
window edge, a segment or clip length grown by one) is bisected with the reference until two neighbouring members get different verdicts.
The families are placed in every segment the stage re-aligns (the clipped part of a split read, the mate of a split read, either discordant
mate), on both strands, across splice sites and one-base deletions, in windows at block boundaries, contig ends and tandem repeats."""
import numpy as np
import seqworld as W
from seqrules import reverse_complement

BLOCK = 1 << 17
LENGTHS = (2 * BLOCK + 9_517, 3_001, 24_013, 5_003)   # none a multiple of 8 or 64
N_INDEX = 3                                            # contig 3 has genes but no index
MAX_MATE_GAP = 300
IUPAC_N = W.IUPAC + "N"
SEG_LENGTHS = [0, 1, 7, 8, 9, 15, 16, 17, 29, 30, 31, 32, 33, 63, 64, 65, 100, 101, 299, 300]
MAX_READ = 320
F_NONE, F_DUPLICATES, F_MISMAPPERS, F_OTHER_CANDIDATE_FILTER = 0, 1, 11, 5


# ------------------------------------------------------------------------------------------------ genome
def _random(rng, n, alphabet="ACGT"):
    return "".join(np.array(list(alphabet))[rng.integers(0, len(alphabet), n)])


def _sprinkle(rng, s, rate):
    a = np.array(list(s))
    hit = rng.random(len(a)) < rate
    a[hit] = np.array(list(IUPAC_N))[rng.integers(0, len(IUPAC_N), int(hit.sum()))]
    return "".join(a)


def make_genome(rng):
    c0 = list(_sprinkle(rng, _random(rng, LENGTHS[0]), 0.003))
    for at in rng.integers(0, LENGTHS[0] - 100, 12):   # N runs
        c0[at:at + int(rng.integers(5, 60))] = "N" * len(c0[at:at + 60])
    c0 = "".join(c0)[:LENGTHS[0]]
    c1 = _sprinkle(rng, _random(rng, LENGTHS[1]), 0.003)
    parts = []
    while sum(map(len, parts)) < LENGTHS[2]:
        period = int(rng.choice([1, 2, 3, 4, 5, 6] + list(range(20, 51, 6))))
        motif = _random(rng, period)
        parts.append((motif * (400 // period + 2))[:int(rng.integers(120, 400))])
        parts.append(_random(rng, int(rng.integers(40, 200))))
    c2 = "".join(parts)[:LENGTHS[2]]
    c3 = _sprinkle(rng, _random(rng, LENGTHS[3]), 0.003)
    return [c0, c1, c2, c3]


def with_exotic(contigs):
    """The same genome with one character outside the nt16 alphabet, at a base no test alignment, clip or window reaches (alignments on
    contig 3 start at 600 or later, and it has no index), so that the reference's verdicts stay those of the plain genome."""
    c3 = contigs[3]
    return contigs[:3] + [c3[:5] + "X" + c3[6:]]


def plant_homologs(rng, contigs, genes):
    """Copies of gene sequences (some reverse-complemented, with 0-20 % mutations) into other genes, so that the homology test sits at
    various identities. Returns (small gene, big gene) index pairs."""
    contigs = [list(c) for c in contigs]
    pairs = []
    for k in range(len(genes)):
        c, s, e, strand = genes[k]
        if genes[k][0] >= N_INDEX or e - s > 4000:
            continue
        for j in range(len(genes)):
            if j == k or genes[j][0] >= N_INDEX or genes[j][2] - genes[j][1] < e - s:
                continue
            pairs.append((k, j))
    rng.shuffle(pairs)
    planted = []
    used = set()
    for k, j in pairs:
        if k in used or j in used or len(planted) >= 12:
            continue
        c, s, e, strand = genes[k]
        cj, sj, ej, strandj = genes[j]
        if cj == c and not (e < sj or s > ej):
            continue
        seq = "".join(contigs[c][s:e])
        if strand != strandj:
            seq = reverse_complement(seq)
        rate = float(rng.choice([0.0, 0.02, 0.05, 0.1, 0.2]))
        seq = list(seq)
        for p in np.nonzero(rng.random(len(seq)) < rate)[0]:
            seq[p] = str(rng.choice(list("ACGT" + IUPAC_N)))
        at = sj + int(rng.integers(0, max(1, (ej - sj) - len(seq))))
        at = min(at, len(contigs[cj]) - len(seq))
        contigs[cj][at:at + len(seq)] = seq
        used.update((k, j)); planted.append((k, j))
    return ["".join(c) for c in contigs], planted


# ------------------------------------------------------------------------------------------------ genes
def make_genes(rng):
    """(contig, start, end, forward) per gene, and the genes of the 34-gene alignment."""
    L0 = LENGTHS[0]
    genes = [(0, BLOCK - 1500, BLOCK + 1200, True), (0, 2 * BLOCK - 800, 2 * BLOCK + 2100, False),   # windows across both block boundaries
             (0, 20_000, 23_000, True), (0, 60_000, 61_900, False), (0, 90_001, 92_500, True), (0, 200_000, 201_500, False),
             (0, L0 - 2_500, L0 - 700, True),
             (1, 100, 2_900, True),                         # window clamped at 0 and at the last base
             (2, 1_000, 6_000, True), (2, 12_000, 15_500, False),   # tandem repeats
             (3, 500, 4_500, True), (0, 30_000, 31_500, True), (0, 30_500, 31_000, False)]   # beyond the index; overlapping pair
    many = []
    for k in range(34):   # 34 small genes on one alignment: pass 1 cannot queue their searches
        s = 150_000 + 160 * k
        many.append(len(genes)); genes.append((0, s, s + 120 + int(rng.integers(0, 60)), bool(k & 1)))
    genes.append((0, 240_000, 240_000 + 1_500, True)); genes.append((2, 18_000, 19_500, False))
    return genes, many


def splice_sites_for(rng, genes):
    """Downstream splice sites per gene, given directly: random sites inside the gene, a pair of adjacent sites, and for one gene a site on
    its window end for every read length up to MAX_READ (a run of adjacent sites behind the gene)."""
    out = []
    for g, (c, s, e, _) in enumerate(genes):
        sites = set(int(x) for x in rng.integers(s, e + 1, int(rng.integers(0, 8))))
        if e - s > 1000:
            a = int(rng.integers(s, e - 1)); sites.update((a, a + 1))
        if g == 2:
            sites.update(e + MAX_MATE_GAP + read_length - 1 for read_length in range(1, MAX_READ + 1))
        out.append(sorted(sites))
    return out


def annotation(genes, n_contigs):
    a = W.one_gene_annotation(n_contigs)
    n = len(genes)
    a["n_genes"] = n
    a["gene_contig"] = np.array([g[0] for g in genes], np.uint16); a["gene_start"] = np.array([g[1] for g in genes], np.int32)
    a["gene_end"] = np.array([g[2] for g in genes], np.int32); a["gene_strand"] = np.array([1 if g[3] else 0 for g in genes], np.uint8)
    a["gene_exonic_length"] = np.array([g[2] - g[1] + 1 for g in genes], np.int32); a["gene_flags"] = np.full(n, 2, np.uint8)
    return a


# ------------------------------------------------------------------------------------------------ fragments
def aln(contig, start, forward, cigar, genes):
    span = sum(l for op, l in cigar if op in "MDN=X")
    return {"contig": contig, "start": int(start), "end": int(start) + span - 1, "forward": forward, "cigar": cigar, "genes": sorted(genes)}


class Builder:
    """Wraps a probe sequence into a fragment; every other re-aligned segment is random, so that the probe decides the verdict."""

    def __init__(self, rng, contigs, genes):
        self.rng, self.contigs, self.genes = rng, contigs, genes

    def dead(self, n):
        return _random(self.rng, n)

    def anchor_pos(self, contig, span, lo=1_000):
        return int(self.rng.integers(lo, len(self.contigs[contig]) - span - 1_000))

    def split(self, seg0, seg1, genes0, genes1, forward=True, lead="S", sr=None, sup_start=None, m=None, mclip=None):
        """Split read: slot 0 mate1 (its non-clipped part is seg1), slot 1 the split read (its clip is seg0), slot 2 the supplementary.
        m: bases of the split read's anchor; mclip: clipped bases of mate1."""
        rng = self.rng
        m = m or int(rng.integers(1, max(2, min(40, MAX_READ - len(seg0)))))
        anchor = self.dead(m)
        if forward:
            r1 = seg0 + anchor; cig = ([(lead, len(seg0))] if seg0 else []) + [("M", m)]
        else:
            r1 = anchor + seg0; cig = [("M", m)] + ([(lead, len(seg0))] if seg0 else [])
        csr, psr = sr if sr else (3, self.anchor_pos(3, m, 600))
        mclip = self.dead(mclip or int(rng.integers(1, 30)))
        if forward:
            r0 = mclip + seg1; mcig = [("S", len(mclip))] + ([("M", len(seg1))] if seg1 else [])
        else:
            r0 = seg1 + mclip; mcig = ([("M", len(seg1))] if seg1 else []) + [("S", len(mclip))]
        sup_span = max(len(seg0), 1)
        cs = 3
        ps = sup_start if sup_start is not None else self.anchor_pos(cs, sup_span, 600)
        a0 = aln(3, self.anchor_pos(3, len(seg1) + 1, 600), not forward, mcig, [10])
        a1 = aln(csr, psr, forward, cig, genes0)
        a2 = aln(cs, ps, forward, [("M", sup_span), ("S", m)], genes1)
        return {"alignments": [a0, a1, a2], "sequences": [r0, r1], "multimapper": False, "kind": 0}

    def discordant(self, s0, s1, genes0, genes1, clips0=(0, 0), clips1=(0, 0), c0=3, c1=3):
        """Mates s0 (genes0) and s1 (genes1); mate k is re-aligned against the genes of the other one."""
        def cig(n, clip):
            pre, post = clip
            return ([("S", pre)] if pre else []) + [("M", n - pre - post)] + ([("S", post)] if post else [])
        a0 = aln(c0, self.anchor_pos(c0, len(s0), 600), True, cig(len(s0), clips0), genes0)
        a1 = aln(c1, self.anchor_pos(c1, len(s1), 600), False, cig(len(s1), clips1), genes1)
        return {"alignments": [a0, a1], "sequences": [s0, s1], "multimapper": False, "kind": 1}


def mutate(rng, seq, order, t, chars):
    s = list(seq)
    for k in range(t):
        p = order[k]
        s[p] = chars[k] if chars[k] != s[p] else ("A" if s[p] != "A" else "C")
    return "".join(s)


def bisect_family(make, lo, hi, judge):
    """Neighbouring members (make(t), make(t + 1)) with different verdicts, or None when the ends agree."""
    vlo, vhi = judge(make(lo)), judge(make(hi))
    if vlo == vhi:
        return None
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if judge(make(mid)) == vlo:
            lo = mid
        else:
            hi = mid
    return make(lo), make(hi)


# ------------------------------------------------------------------------------------------------ families of shapes
FAMILIES = ("mutations", "run", "shift_end", "shift_start", "length", "clip", "extend", "same_contig", "splice", "deletion", "many_genes",
            "iupac_reverse", "short")


def probe_length(frag):
    """Bases of the probe segment (mismap_items::segment)."""
    a, slot, seqs = frag["alignments"], frag.get("slot"), frag["sequences"]
    clip = lambda c, end: c[end][1] if c[end][0] in "SH" else 0
    if slot == "seg0":
        return min(clip(a[1]["cigar"], 0 if a[1]["forward"] else -1), len(seqs[1]))
    if slot == "seg1":
        return len(seqs[0]) - clip(a[0]["cigar"], 0 if a[1]["forward"] else -1)
    return len(seqs[0])


def slice_offset(frag):
    """Offset, in bases from the start of its stored read, of the slice the probe segment is re-aligned from (mismap_items::segment): a
    read starts on a 32-base boundary of the sequence pool, so this is the slice's offset in the pool modulo 32."""
    a, slot = frag["alignments"], frag.get("slot")
    if slot == "seg0" and not a[1]["forward"]:
        last = a[1]["cigar"][-1]
        return len(frag["sequences"][1]) - (last[1] if last[0] in "SH" else 0)
    if slot == "seg1" and a[1]["forward"]:
        first = a[0]["cigar"][0]
        return first[1] if first[0] in "SH" else 0
    return 0


class Families:
    """Generates twins. Every family member is built from its own fresh random stream, so that two members differ in the family's
    parameter only."""

    def __init__(self, rng, stage, many, dead_gene):
        self.rng, self.stage, self.many, self.dead_gene = rng, stage, many, dead_gene
        self.search_genes = [g for g, x in enumerate(stage.genes) if x[0] < N_INDEX and g not in many]
        self.attempt = self.iupac_turn = 0
        self.offsets_done = set()
        self.iupac = {}   # gene -> positions of IUPAC codes (not N) in its padded gene
        for g in self.search_genes:
            c, s, e, _ = stage.genes[g]
            self.iupac[g] = [q for q in range(max(s - MAX_MATE_GAP, 20), min(e + MAX_MATE_GAP, len(stage.contigs[c]) - 200)) if stage.contigs[c][q] in W.IUPAC]

    def builder(self, seed):
        return Builder(np.random.default_rng(seed), self.stage.contigs, self.stage.genes)

    def wrap(self, seed, probe, slot, genes, forward, clips=(0, 0), m=None, mclip=None):
        b = self.builder(seed)
        if slot == "seg0":
            f = b.split(probe, b.dead(40), genes, [self.dead_gene], forward=forward, m=m, mclip=mclip)
        elif slot == "seg1":
            f = b.split(b.dead(40), probe, [self.dead_gene], genes, forward=forward, m=m, mclip=mclip)
        else:
            f = b.discordant(probe, b.dead(60), [self.dead_gene], genes, clips0=clips, c0=3, c1=1)
        f["slot"] = slot
        return f

    def copy(self, g, L, rc, lo=None, hi=None):
        c, s, e, _ = self.stage.genes[g]
        contig = self.stage.contigs[c]
        lo = max(0, s - MAX_MATE_GAP) if lo is None else lo
        hi = min(len(contig) - L, e + MAX_MATE_GAP - L) if hi is None else hi
        if hi < lo:
            return None, None
        p = int(self.rng.integers(lo, hi + 1))
        seq = contig[p:p + L]
        return p, (reverse_complement(seq) if rc else seq)

    def judge(self, same):
        return lambda frag: self.stage.fragment_is_mismapper(frag, frag["kind"], same)

    def one(self, family):
        """(family, same_contig listing, twins or None, a plain member)."""
        rng = self.rng
        seed = int(rng.integers(0, 2**31))
        slot = str(rng.choice(["seg0", "seg1", "disc"]))
        g = int(rng.choice(self.search_genes))
        genes = [g]
        rc = bool(rng.random() < 0.5); forward = bool(rng.random() < 0.5)
        same = False
        L = int(rng.choice([x for x in SEG_LENGTHS if x >= 9] + [40, 80, 120, 150, 200, 250]))
        chars = [str(x) for x in rng.choice(list("ACGT" * 3 + IUPAC_N), 400)]
        m = int(rng.integers(1, max(2, min(40, MAX_READ - 300))))
        mclip = None
        self.attempt += 1
        missing = sorted(set(range(32)) - self.offsets_done)   # offsets no twin has yet, in turn
        offset = missing[(self.attempt // 2) % len(missing)] if missing else (self.attempt // 2) % 32
        if self.attempt % 2 and slot != "disc":   # every other shape: the probe's slice at a chosen offset in the pool, all 32 in turn
            if slot == "seg0":
                forward = offset == 0
                m = offset or m
            else:
                forward = offset != 0
                mclip = offset or None
        wrap = lambda seed, probe, slot, genes, forward, **kw: self.wrap(seed, probe, slot, genes, forward, mclip=mclip, **{"m": m, **kw})
        if family == "short":   # 0-8 bases: shorter than one seed, never placed
            L = self.attempt % 9
            slot = "disc" if slot == "disc" and L > 0 else ("seg1" if slot == "disc" else slot)
            p, base = self.copy(g, L, rc)
            return family, same, None, (wrap(seed, base, slot, genes, forward) if base is not None else None)
        if family == "iupac_reverse":   # the word positions in turn, a few tries for one where the code decides
            j = 8 + self.iupac_turn % 8; self.iupac_turn += 1
            for _ in range(8):
                out = self.iupac_reverse(int(rng.integers(0, 2**31)), slot, wrap, j + 8 * int(rng.integers(0, 3)))
                if out[2] is not None and "iupac_word_position" in out[2][0]:
                    break
            return out
        if family == "many_genes":
            slot, genes, g = "seg0", list(self.many), int(rng.choice(self.many))
        if family in ("mutations", "run", "many_genes", "splice", "deletion"):
            if family == "splice":
                sites = [x for x in self.stage.splice[g] if self.stage.genes[g][1] <= x <= self.stage.genes[g][2]]
                if not sites:
                    return family, same, None, None
                s = int(rng.choice(sites)); contig = self.stage.contigs[self.stage.genes[g][0]]
                a = int(rng.integers(10, max(11, L - 10))); b = max(L - a, 9)
                y = s + 2 + int(rng.integers(0, 400))
                if s - a + 1 < 0 or y + b > len(contig):
                    return family, same, None, None
                base = contig[s - a + 1:s + 1] + contig[y:y + b]
                later = [x for x in self.stage.splice[g] if y + 9 <= x < y + 200]
                if later and rng.random() < 0.5:   # a second intron: the second exon ends on a splice site of the gene
                    s2 = int(rng.choice(later)); z = s2 + 2 + int(rng.integers(0, 200))
                    base = contig[s - a + 1:s + 1] + contig[y:s2 + 1] + contig[z:z + 20]
                base = reverse_complement(base) if rc else base
            elif family == "deletion":
                L = int(rng.choice([28, 29, 30, 31, 40]))
                p, base = self.copy(g, L + 1, False)
                if base is None:
                    return family, same, None, None
                a = int(rng.integers(9, L - 8)); base = base[:a] + base[a + 1:]
                base = reverse_complement(base) if rc else base
            else:
                p, base = self.copy(g, L, rc)
                if base is None:
                    return family, same, None, None
            L = len(base)
            if family == "run":
                start = int(rng.integers(0, L)); order = [(start + k) % L for k in range(L)]
            else:
                order = list(rng.permutation(L))
            make = lambda t: wrap(seed, mutate(rng, base, order, t, chars), slot, genes, forward, m=m)
            lo, hi = 0, L
        elif family in ("shift_end", "shift_start"):
            c = self.stage.genes[g][0]; contig = self.stage.contigs[c]
            probe0 = wrap(seed, "A" * L, slot, genes, forward, m=m)
            rl = len(probe0["sequences"][1 if slot == "seg0" else 0])
            ws, we = self.stage.window(g, rl)
            if family == "shift_end":
                lo, hi = we - L - 2, min(we + 2, len(contig) - L)
            else:
                lo, hi = max(ws - L, 0), ws + 3
            if lo < 0 or hi <= lo:
                return family, same, None, None
            seqs = {t: contig[t:t + L] for t in range(lo, hi + 1)}
            make = lambda t: wrap(seed, reverse_complement(seqs[t]) if rc else seqs[t], slot, genes, forward, m=m)
        elif family == "length":
            p, base = self.copy(g, 305, rc)
            if base is None:
                return family, same, None, None
            base = mutate(rng, base, list(rng.permutation(len(base))), int(rng.integers(0, 12)), chars)
            lo, hi = (24, 36) if rng.random() < 0.5 else (292, 300)
            make = lambda t: wrap(seed, base[:t], slot, genes, forward, m=min(m, MAX_READ - t) if slot == "seg0" else m)
        elif family == "clip":
            slot = "disc"
            L = int(rng.integers(30, 200))
            p, base = self.copy(g, L, rc)
            if base is None:
                return family, same, None, None
            base = mutate(rng, base, list(rng.permutation(L)), int(L * rng.uniform(0.1, 0.35)), chars)
            make = lambda t: wrap(seed, base, slot, genes, forward, clips=(t // 2, t - t // 2))
            lo, hi = 0, L - 1
        elif family == "extend":
            c = int(rng.choice([0, 1])); contig = self.stage.contigs[c]
            pre = int(rng.integers(2, 60))
            b0 = self.builder(seed)
            anchor_m = int(rng.integers(1, 30))
            where = rng.random()
            if forward:
                P = int(rng.integers(0, pre)) if where < 0.3 else int(rng.integers(pre, len(contig) - 100))
                seg = (_random(rng, pre - min(pre, P)) + contig[P - min(pre, P):P])
            else:
                E = len(contig) - 1 - int(rng.integers(0, 4)) if where < 0.3 else int(rng.integers(100, len(contig) - pre - 3))
                P = E - anchor_m + 1
                seg = contig[E + 1:E + 1 + pre]; seg += _random(rng, pre - len(seg))
            lead = "H" if rng.random() < 0.3 else "S"
            order = list(rng.permutation(pre))
            def make(t):
                b = self.builder(seed)
                return b.split(mutate(rng, seg, order, t, chars), b.dead(40), [self.dead_gene], [self.dead_gene], forward=forward, lead=lead, sr=(c, P), m=anchor_m)
            lo, hi = 0, pre
        elif family == "same_contig":
            slot, same = "seg0", True
            L = int(rng.integers(20, 120))
            probe0 = wrap(seed, "A" * L, slot, genes, forward, m=m)
            ws, we = self.stage.window(g, len(probe0["sequences"][1]))
            p, base = self.copy(g, L, rc)
            if base is None:
                return family, same, None, None
            span = max(L, 1)
            if rng.random() < 0.5 and ws - span - 2 >= 0:
                lo, hi = ws - 2, ws + 1
                make = lambda t: self.builder(seed).split(base, self.builder(seed + 1).dead(40), genes, [self.dead_gene], forward=forward, m=m, sup_start=t - span + 1)
            else:
                lo, hi = we - 1, we + 2
                make = lambda t: self.builder(seed).split(base, self.builder(seed + 1).dead(40), genes, [self.dead_gene], forward=forward, m=m, sup_start=t)
        else:
            raise ValueError(family)
        judge = self.judge(same)
        twins = bisect_family(make, lo, hi, judge)
        if twins and twins[0].get("slot") in ("seg0", "seg1"):
            self.offsets_done.add(slice_offset(twins[0]) % 32)
        return family, same, twins, make(lo)

    def iupac_reverse(self, seed, slot, wrap, j):
        """A probe copied over an IUPAC code of the genome and stored reverse-complemented, so that the reverse-strand search compares the
        code with itself (the reference complements A/C/G/T only). Mutations elsewhere are bisected to the edge; at the edge, the twin has
        a plain base instead of the code. The code sits at read position 8..31, at position j % 8 of the 8-base words after the seed."""
        rng = self.rng
        genes = [g for g in self.search_genes if self.iupac[g]]
        g = int(rng.choice(genes))
        c = self.stage.genes[g][0]; contig = self.stage.contigs[c]
        L = int(rng.choice([40, 64, 101, 150]))
        q = int(rng.choice(self.iupac[g]))
        if q - j < 0 or q - j + L > len(contig):
            return "iupac_reverse", False, None, None
        base = contig[q - j:q - j + L]
        order = [p for p in rng.permutation(L) if p != j]
        chars = [str(x) for x in rng.choice(list("ACGT"), L)]
        make = lambda t: wrap(seed, reverse_complement(mutate(rng, base, order, t, chars)), slot, [g], False)
        found = bisect_family(make, 0, len(order), self.judge(False))
        if found is None:
            return "iupac_reverse", False, None, make(0)
        kept = found[0]
        t = next(t for t in range(len(order) + 1) if make(t)["sequences"] == kept["sequences"])
        plain = list(mutate(rng, base, order, t, chars)); plain[j] = "A" if base[j] != "A" else "C"
        twin = wrap(seed, reverse_complement("".join(plain)), slot, [g], False)
        if self.judge(False)(twin) == self.judge(False)(kept):
            return "iupac_reverse", False, found, None
        kept["iupac_word_position"] = twin["iupac_word_position"] = j % 8
        return "iupac_reverse", False, (kept, twin), None
