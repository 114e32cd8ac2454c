"""ctypes binding of the C ABI in include/arriba_b200.h.

`load()` opens the CUDA product library (arriba_b200/libarriba_b200.so) and nothing else; it raises if the
library is missing. The CPU test-suite passes the path of tests/hostsim explicitly (`load(path)`)."""
import ctypes as C
import os
import numpy as np

from . import _build

N_FILTERS = 38
FILTER_NAMES = ["", "duplicates", "inconsistently_clipped", "homopolymer", "read_through", "same_gene", "small_insert_size", "long_gap",
                "hairpin", "multimappers", "mismatches", "mismappers", "relative_support", "intronic", "non_coding_neighbors",
                "intragenic_exonic", "internal_tandem_duplication", "min_support", "known_fusions", "spliced", "blacklist", "end_to_end",
                "in_vitro", "merge_adjacent", "select_best", "marginal_read_through", "short_anchor", "no_coverage", "many_spliced",
                "no_genomic_support", "uninteresting_contigs", "viral_contigs", "top_expressed_viral_contigs", "low_coverage_viral_contigs",
                "genomic_support", "isoforms", "low_entropy", "homologs"]

_p = C.POINTER


class Contigs(C.Structure):
    _fields_ = [("n_contigs", C.c_uint32), ("flags", _p(C.c_uint8)), ("length", _p(C.c_uint32)), ("sequence", _p(C.c_char_p))]


class Annotation(C.Structure):
    _fields_ = [("n_genes", C.c_uint32), ("gene_contig", _p(C.c_uint16)), ("gene_start", _p(C.c_int32)), ("gene_end", _p(C.c_int32)),
                ("gene_strand", _p(C.c_uint8)), ("gene_exonic_length", _p(C.c_int32)), ("gene_flags", _p(C.c_uint8)),
                ("n_exons", C.c_uint32), ("exon_gene", _p(C.c_uint32)), ("exon_start", _p(C.c_int32)), ("exon_end", _p(C.c_int32)),
                ("exon_cds_start", _p(C.c_int32)), ("exon_cds_end", _p(C.c_int32)), ("exon_next_start", _p(C.c_int32)), ("exon_flags", _p(C.c_uint8)),
                ("n_contigs", C.c_uint32),
                ("exon_region_begin", _p(C.c_uint32)), ("exon_region_end", _p(C.c_int32)), ("exon_region_off", _p(C.c_uint32)), ("exon_region_items", _p(C.c_uint32)),
                ("gene_region_begin", _p(C.c_uint32)), ("gene_region_end", _p(C.c_int32)), ("gene_region_off", _p(C.c_uint32)), ("gene_region_items", _p(C.c_uint32))]


class Params(C.Structure):
    _fields_ = [("filter_mask", C.c_uint64), ("homopolymer_length", C.c_uint32), ("min_read_through_distance", C.c_int32),
                ("max_kmer_content", C.c_float), ("max_itd_length", C.c_uint32), ("external_duplicate_marking", C.c_uint32),
                ("mismatch_pvalue_cutoff", C.c_float), ("subsampling_threshold", C.c_uint32), ("evalue_cutoff", C.c_float),
                ("max_mismapper_fraction", C.c_float), ("max_homolog_identity", C.c_float)]


class SoaChunk(C.Structure):
    _fields_ = [("n_fragments", C.c_uint32), ("n_aln", _p(C.c_uint8)), ("fflags", _p(C.c_uint8)), ("filter", _p(C.c_uint8)),
                ("contig", _p(C.c_uint16)), ("start", _p(C.c_int32)), ("end", _p(C.c_int32)), ("aflags", _p(C.c_uint8)),
                ("cigar_off", _p(C.c_uint32)), ("cigar_cnt", _p(C.c_uint16)), ("seq_off", _p(C.c_uint32)), ("seq_len", _p(C.c_uint16)),
                ("genes_off", _p(C.c_uint32)), ("genes_cnt", _p(C.c_uint16)),
                ("cigar", _p(C.c_uint32)), ("n_cigar", C.c_uint64), ("seq", _p(C.c_uint8)), ("n_seq_bytes", C.c_uint64),
                ("genes", _p(C.c_uint32)), ("n_genes", C.c_uint64)]


class Candidates(C.Structure):
    _fields_ = [("n", C.c_uint32), ("gene1", _p(C.c_uint32)), ("gene2", _p(C.c_uint32)), ("contig1", _p(C.c_uint16)), ("contig2", _p(C.c_uint16)),
                ("breakpoint1", _p(C.c_int32)), ("breakpoint2", _p(C.c_int32)), ("direction1", _p(C.c_uint8)), ("direction2", _p(C.c_uint8)),
                ("split_reads1", _p(C.c_uint32)), ("split_reads2", _p(C.c_uint32)), ("discordant_mates", _p(C.c_uint32)),
                ("filter", _p(C.c_uint8)), ("bits", _p(C.c_uint8)), ("bits2", _p(C.c_uint8)),
                ("anchor_start1", _p(C.c_int32)), ("anchor_start2", _p(C.c_int32)), ("evalue", _p(C.c_float)),
                ("list1_off", _p(C.c_uint32)), ("list2_off", _p(C.c_uint32)), ("listd_off", _p(C.c_uint32)),
                ("list1", _p(C.c_uint32)), ("list2", _p(C.c_uint32)), ("listd", _p(C.c_uint32))]


class Timings(C.Structure):
    _fields_ = [("duplicates_ms", C.c_float), ("classify_ms", C.c_float), ("read_filters_ms", C.c_float), ("find_fusions_ms", C.c_float),
                ("classify_algorithmic_bytes", C.c_uint64), ("h2d_bytes", C.c_uint64), ("h2d_ms", C.c_float),
                ("merge_adjacent_ms", C.c_float), ("evalue_ms", C.c_float), ("kmer_index_ms", C.c_float), ("homologs_ms", C.c_float), ("mismappers_ms", C.c_float),
                ("mismapper_items", C.c_uint64), ("kmer_positions", C.c_uint64), ("mismapper_heavy_items", C.c_uint64),
                ("mismappers_pass1_ms", C.c_float), ("mismappers_pass2_ms", C.c_float), ("mismapper_tasks", C.c_uint64), ("mismapper_rounds", C.c_uint32), ("mismapper_overflow", C.c_uint32), ("mismapper_table_slots", C.c_uint32),
                ("cascade_head_ms", C.c_float), ("cascade_sequences_ms", C.c_float), ("cascade_queued", C.c_uint64), ("cascade_algorithmic_bytes", C.c_uint64 * 2), ("annotate_ms", C.c_float), ("in_vitro_ms", C.c_float), ("multimappers_ms", C.c_float), ("order_ms", C.c_float), ("partners_ms", C.c_float), ("rows_ms", C.c_float), ("bam_scan_ms", C.c_float), ("consensus_ms", C.c_float), ("mismapper_algorithmic_bytes", C.c_uint64), ("mismapper_sequences", C.c_uint64), ("mismapper_hits", C.c_uint64),
                ("genomic_support_ms", C.c_float), ("blacklist_ms", C.c_float), ("known_fusions_ms", C.c_float), ("tags_ms", C.c_float),
                ("tags_match_ms", C.c_float), ("tags_sort_ms", C.c_float), ("tags_pairs", C.c_uint64), ("protein_domains_ms", C.c_float),
                ("rec_chunk_copy_ms", C.c_float), ("rec_chunk_kernels_ms", C.c_float), ("rec_sort_ms", C.c_float), ("rec_count_ms", C.c_float),
                ("rec_scan_ms", C.c_float), ("rec_write_ms", C.c_float), ("rec_download_ms", C.c_float),
                ("rec_text_parse_ms", C.c_float), ("fill_gaps_ms", C.c_float),
                ("fill_gaps_jobs", C.c_uint64), ("fill_gaps_chars", C.c_uint64),
                ("rec_unwrap_ms", C.c_float), ("rec_store_grows", C.c_uint32), ("rec_store_bytes", C.c_uint64), ("rec_h2d_bytes", C.c_uint64)]


_CTYPE = {np.dtype(np.uint8): C.c_uint8, np.dtype(np.uint16): C.c_uint16, np.dtype(np.uint32): C.c_uint32, np.dtype(np.int32): C.c_int32,
          np.dtype(np.float32): C.c_float, np.dtype(np.uint64): C.c_uint64}


def ptr(a):
    """numpy array -> typed ctypes pointer (array must be C-contiguous and stay alive)."""
    assert a.flags["C_CONTIGUOUS"], "array must be contiguous"
    return a.ctypes.data_as(_p(_CTYPE[a.dtype]))


class EvalueInputs(C.Structure):
    _fields_ = [("partner_count", _p(C.c_int32)), ("n_genes", C.c_uint32), ("spliced_breakpoints", C.c_uint32), ("exonic_breakpoints", C.c_uint32),
                ("intronic_breakpoints", C.c_uint32), ("exonic_intronic_breakpoints", C.c_uint32), ("intragenic_duplications", C.c_uint32),
                ("intragenic_inversions", C.c_uint32), ("spliced_same_gene", C.c_uint32), ("spliced_different_genes", C.c_uint32),
                ("read_through_fraction", C.c_float), ("mapped_reads", C.c_uint64), ("pow_reads", _p(C.c_double)), ("pow_intragenic", _p(C.c_double)),
                ("pow_intergenic", _p(C.c_double)), ("n_read_table", C.c_uint32), ("pow_spliced1000", _p(C.c_double)), ("pow_spliced400", _p(C.c_double)),
                ("pow_read_through", _p(C.c_double)), ("pow_proximal", _p(C.c_double)), ("read_through_penalty", C.c_double)]


class ArbError(RuntimeError):
    pass


_LIBS = {}


def load(path=None):
    """Opens the C-ABI library. Default: the CUDA product library; fails loudly if it has not been built."""
    path = path or _build.PRODUCT_LIB
    if path in _LIBS:
        return _LIBS[path]
    if not os.path.exists(path):
        raise ArbError("%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` first (there is no CPU fallback)" % path)
    lib = C.CDLL(path)
    lib.arb_backend.restype = C.c_char_p
    lib.arb_last_error.restype = C.c_char_p
    lib.arb_last_error.argtypes = [C.c_void_p]
    lib.arb_kernel_launches.restype = C.c_uint64
    sizes = (C.c_uint32 * 9)()
    lib.arb_struct_sizes(sizes)
    expect = [C.sizeof(x) for x in (Contigs, Annotation, Params, SoaChunk, Candidates, EvalueInputs, Timings, RunOptions, RunStats)]
    if list(sizes) != expect:
        raise ArbError("struct layout mismatch between include/arriba_b200.h and arriba_b200/lib.py: %s vs %s" % (list(sizes), expect))
    lib.arb_ctx_create.argtypes = [_p(C.c_void_p), C.c_int]
    lib.arb_ctx_destroy.argtypes = [C.c_void_p]
    lib.arb_default_params.argtypes = [_p(Params)]
    for name, args in [("arb_set_params", [_p(Params)]), ("arb_set_contigs", [_p(Contigs)]), ("arb_set_annotation", [_p(Annotation)]),
                       ("arb_push_chunk", [_p(SoaChunk)]), ("arb_run_read_filters", []),
                       ("arb_get_fragment_filters", [_p(C.c_uint8), _p(C.c_uint8)]), ("arb_set_fragment_filters", [_p(C.c_uint8)]),
                       ("arb_get_filter_counts", [_p(C.c_uint32)]), ("arb_find_fusions", [C.c_int32]),
                       ("arb_candidates_size", [_p(C.c_uint32), _p(C.c_uint64), _p(C.c_uint64), _p(C.c_uint64)]),
                       ("arb_get_candidates", [_p(Candidates)]), ("arb_get_slot_swaps", [_p(C.c_uint8)]), ("arb_get_timings", [_p(Timings)]),
                       ("arb_exchange_header", [C.c_int, _p(C.c_uint64), _p(C.c_uint32)]), ("arb_exchange_prepare", [C.c_int, _p(C.c_uint64), C.c_uint32]),
                       ("arb_exchange_buffers", [C.c_int, _p(C.c_void_p), _p(C.c_uint64), _p(C.c_uint32)]), ("arb_exchange_commit", [C.c_int]),
                       ("arb_set_work_partition", [_p(C.c_uint32), _p(C.c_uint8), C.c_uint32, C.c_int, C.c_int]),
                       ("arb_candidates_export", [_p(C.c_void_p), _p(C.c_uint64), _p(C.c_uint64)]), ("arb_candidates_import", [C.c_void_p, C.c_uint64, _p(C.c_uint64), C.c_uint32]),
                       ("arb_swaps_buffer", [_p(C.c_void_p), _p(C.c_uint64)]), ("arb_swaps_apply", []),
                       ("arb_filter_mismappers_part", [C.c_int32, C.c_int, C.c_int, _p(C.c_void_p), _p(C.c_uint64)]), ("arb_filter_mismappers_finish", [_p(C.c_uint64)]),
                       ("arb_set_genomic_breakpoints", [C.c_uint32, _p(C.c_uint16), _p(C.c_uint16), _p(C.c_uint8), _p(C.c_uint8), _p(C.c_int32), _p(C.c_int32)]),
                       ("arb_mark_genomic_support", [C.c_int32, C.c_int32, _p(C.c_uint32)]), ("arb_get_genomic_support", [_p(C.c_int32), _p(C.c_int32)]),
                       ("arb_set_blacklist", [C.c_uint32] + [_p(C.c_uint8)] * 4 + [_p(C.c_uint16)] * 2 + [_p(C.c_int32)] * 4 + [_p(C.c_uint32)] * 2),
                       ("arb_filter_blacklist", [C.c_uint32, _p(C.c_uint32), C.c_float, C.c_int32, _p(C.c_uint8), _p(C.c_uint32)]),
                       ("arb_set_known_fusions", [C.c_uint32] + [_p(C.c_uint8)] * 4 + [_p(C.c_uint16)] * 2 + [_p(C.c_int32)] * 4 + [_p(C.c_uint32)] * 2),
                       ("arb_recover_known_fusions", [C.c_uint32, _p(C.c_uint32), C.c_int32, _p(C.c_uint8), _p(C.c_uint32)]),
                       ("arb_set_tags", [C.c_uint32] + [_p(C.c_uint8)] * 4 + [_p(C.c_uint16)] * 2 + [_p(C.c_int32)] * 4 + [_p(C.c_uint32)] * 2 + [_p(C.c_uint32), C.c_uint32, C.c_char_p, _p(C.c_uint32)]),
                       ("arb_annotate_tags", [C.c_uint32, _p(C.c_uint32), C.c_int32, _p(C.c_uint64)]),
                       ("arb_get_tags", [_p(C.c_uint32), _p(C.c_uint32)]),
                       ("arb_set_protein_domains", [C.c_uint32, _p(C.c_uint16), _p(C.c_int32), _p(C.c_int32), _p(C.c_uint32), _p(C.c_uint32), C.c_uint32, C.c_char_p, _p(C.c_uint32)]),
                       ("arb_retained_protein_domains", [C.c_uint32, _p(C.c_uint32), _p(C.c_uint64)]),
                       ("arb_get_retained_protein_domains", [_p(C.c_uint64), C.c_char_p]),
                       ("arb_set_fill_transcripts", [C.c_uint32, _p(C.c_int32), _p(C.c_int32), _p(C.c_uint32), _p(C.c_int32), _p(C.c_int32)]),
                       ("arb_fill_gaps", [C.c_uint32, C.c_char_p, _p(C.c_uint32), _p(C.c_int32), _p(C.c_uint32), C.c_uint32, _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint8), _p(C.c_uint64)]),
                       ("arb_get_filled", [_p(C.c_uint32), C.c_char_p, _p(C.c_int32)]),
                       ("arb_set_candidate_state", [_p(C.c_uint8), _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32), _p(C.c_float)]),
                       ("arb_set_candidate_lists", [_p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32)]),
                       ("arb_set_splice_sites", [_p(C.c_uint32), _p(C.c_int32)]),
                       ("arb_build_kmer_index", [_p(C.c_uint32), _p(C.c_int32), _p(C.c_int32), C.c_uint32, C.c_uint32, _p(C.c_uint64)]),
                       ("arb_homolog_pairs", [_p(C.c_uint32), _p(C.c_uint32), C.c_uint32, _p(C.c_uint8)]), ("arb_filter_mismappers", [C.c_int32, _p(C.c_uint64)])]:
        fn = getattr(lib, name)
        fn.argtypes = [C.c_void_p] + args
        fn.restype = C.c_int
    _LIBS[path] = lib
    return lib


class Context:
    """One device context (one CUDA device, one stream)."""

    def __init__(self, device=0, lib_path=None):
        self.lib = load(lib_path)
        h = C.c_void_p()
        if self.lib.arb_ctx_create(C.byref(h), device) != 0:
            raise ArbError(self.lib.arb_last_error(None).decode())
        self.h = h
        self._keep = []

    def close(self):
        if self.h:
            self.lib.arb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise ArbError(self.lib.arb_last_error(self.h).decode())

    @property
    def backend(self):
        return self.lib.arb_backend().decode()

    def default_params(self):
        p = Params()
        self.lib.arb_default_params(C.byref(p))
        return p

    def set_params(self, p):
        self._check(self.lib.arb_set_params(self.h, C.byref(p)))

    def set_contigs(self, flags, sequences):
        """flags: uint8 per contig; sequences: list of bytes (or None)."""
        n = len(flags)
        flags = np.ascontiguousarray(flags, np.uint8)
        length = np.array([len(s) if s is not None else 0 for s in sequences], np.uint32)
        arr = (C.c_char_p * n)(*[s if s is not None else None for s in sequences])
        c = Contigs(n, ptr(flags), ptr(length), C.cast(arr, _p(C.c_char_p)))
        self._check(self.lib.arb_set_contigs(self.h, C.byref(c)))

    def set_annotation(self, a):
        """a: dict of numpy arrays named like the struct fields."""
        s = Annotation()
        keep = []
        for name, ctype in Annotation._fields_:
            if name in ("n_genes", "n_exons", "n_contigs"):
                setattr(s, name, int(a[name]))
            else:
                arr = np.require(a[name], requirements=["C", "A"]); keep.append(arr)   # contiguous and naturally aligned, as the C ABI expects
                setattr(s, name, ptr(arr))
        self._check(self.lib.arb_set_annotation(self.h, C.byref(s)))

    def push_chunk(self, ch):
        """ch: dict of numpy arrays named like arb_soa_chunk fields."""
        s = SoaChunk()
        keep = []
        s.n_fragments = int(ch["n_fragments"])
        for name, ctype in SoaChunk._fields_:
            if name in ("n_fragments", "n_cigar", "n_seq_bytes", "n_genes"):
                continue
            arr = np.require(ch[name], requirements=["C", "A"]); keep.append(arr)
            setattr(s, name, ptr(arr))
        s.n_cigar = len(ch["cigar"]); s.n_seq_bytes = len(ch["seq"]); s.n_genes = len(ch["genes"])
        self.n_fragments = s.n_fragments
        self._check(self.lib.arb_push_chunk(self.h, C.byref(s)))

    def run_read_filters(self):
        self._check(self.lib.arb_run_read_filters(self.h))

    def fragment_filters(self):
        f = np.zeros(self.n_fragments, np.uint8); e = np.zeros(self.n_fragments, np.uint8)
        self._check(self.lib.arb_get_fragment_filters(self.h, ptr(f), ptr(e)))
        return f, e

    def set_fragment_filters(self, f):
        f = np.ascontiguousarray(f, np.uint8)
        self._check(self.lib.arb_set_fragment_filters(self.h, ptr(f)))

    def filter_counts(self):
        c = np.zeros(N_FILTERS, np.uint32)
        self._check(self.lib.arb_get_filter_counts(self.h, ptr(c)))
        return c

    def find_fusions(self, max_mate_gap):
        self._check(self.lib.arb_find_fusions(self.h, int(max_mate_gap)))

    def candidates(self):
        n = C.c_uint32(); n1 = C.c_uint64(); n2 = C.c_uint64(); nd = C.c_uint64()
        self._check(self.lib.arb_candidates_size(self.h, C.byref(n), C.byref(n1), C.byref(n2), C.byref(nd)))
        n = n.value
        out = {}
        c = Candidates()
        spec = {"gene1": np.uint32, "gene2": np.uint32, "contig1": np.uint16, "contig2": np.uint16, "breakpoint1": np.int32, "breakpoint2": np.int32,
                "direction1": np.uint8, "direction2": np.uint8, "split_reads1": np.uint32, "split_reads2": np.uint32, "discordant_mates": np.uint32,
                "filter": np.uint8, "bits": np.uint8, "bits2": np.uint8, "anchor_start1": np.int32, "anchor_start2": np.int32, "evalue": np.float32}
        for k, dt in spec.items():
            out[k] = np.zeros(max(n, 1), dt); setattr(c, k, ptr(out[k]))
        for k in ("list1_off", "list2_off", "listd_off"):
            out[k] = np.zeros(n + 1, np.uint32); setattr(c, k, ptr(out[k]))
        for k, m in (("list1", n1.value), ("list2", n2.value), ("listd", nd.value)):
            out[k] = np.zeros(max(m, 1), np.uint32); setattr(c, k, ptr(out[k]))
        self._check(self.lib.arb_get_candidates(self.h, C.byref(c)))
        for k in spec:
            out[k] = out[k][:n]
        out["list1"] = out["list1"][:n1.value]; out["list2"] = out["list2"][:n2.value]; out["listd"] = out["listd"][:nd.value]
        out["n"] = n
        return out

    def timings(self):
        t = Timings()
        self._check(self.lib.arb_get_timings(self.h, C.byref(t)))
        return t

    # ---- one sample on several GPUs: device buffers for the launcher's transport (include/arriba_b200.h; arriba_b200/sharded.py drives these)
    def exchange_header(self, group):
        h = (C.c_uint64 * 16)(); n = C.c_uint32()
        self._check(self.lib.arb_exchange_header(self.h, group, h, C.byref(n)))
        return [int(h[k]) for k in range(n.value)]

    def exchange_prepare(self, group, header):
        h = (C.c_uint64 * len(header))(*header)
        self._check(self.lib.arb_exchange_prepare(self.h, group, h, len(header)))

    def exchange_buffers(self, group):
        ptrs = (C.c_void_p * 32)(); sizes = (C.c_uint64 * 32)(); n = C.c_uint32(32)
        self._check(self.lib.arb_exchange_buffers(self.h, group, ptrs, sizes, C.byref(n)))
        return [(int(ptrs[k] or 0), int(sizes[k])) for k in range(n.value)]

    def exchange_commit(self, group):
        self._check(self.lib.arb_exchange_commit(self.h, group))

    def set_work_partition(self, keys, owner, part, parts):
        keys = np.ascontiguousarray(keys, np.uint32); owner = np.ascontiguousarray(owner, np.uint8)
        self._check(self.lib.arb_set_work_partition(self.h, ptr(keys), ptr(owner), keys.size, part, parts))

    def candidates_export(self):
        blob = C.c_void_p(); n = C.c_uint64(); sizes = (C.c_uint64 * 4)()
        self._check(self.lib.arb_candidates_export(self.h, C.byref(blob), C.byref(n), sizes))
        return int(blob.value or 0), int(n.value), [int(x) for x in sizes]

    def candidates_import(self, all_blobs_ptr, stride, sizes, n_parts):
        s = (C.c_uint64 * (4 * n_parts))(*sizes)
        self._check(self.lib.arb_candidates_import(self.h, C.c_void_p(all_blobs_ptr), stride, s, n_parts))

    def swaps_buffer(self):
        p = C.c_void_p(); n = C.c_uint64()
        self._check(self.lib.arb_swaps_buffer(self.h, C.byref(p), C.byref(n)))
        return int(p.value or 0), int(n.value)

    def swaps_apply(self):
        self._check(self.lib.arb_swaps_apply(self.h))

    def filter_mismappers_part(self, max_mate_gap, part, parts):
        p = C.c_void_p(); n = C.c_uint64()
        self._check(self.lib.arb_filter_mismappers_part(self.h, int(max_mate_gap), part, parts, C.byref(p), C.byref(n)))
        return int(p.value or 0), int(n.value)

    def filter_mismappers_finish(self):
        n = C.c_uint64()
        self._check(self.lib.arb_filter_mismappers_finish(self.h, C.byref(n)))
        return int(n.value)

    # ---- genomic breakpoints from whole-genome sequencing (-d)
    def set_genomic_breakpoints(self, contig1, contig2, direction1, direction2, position1, position2):
        """Records in file order, each normalised so that (contig1, position1) <= (contig2, position2); directions 1 = upstream."""
        cols = [np.ascontiguousarray(a, dt) for a, dt in ((contig1, np.uint16), (contig2, np.uint16), (direction1, np.uint8), (direction2, np.uint8), (position1, np.int32), (position2, np.int32))]
        n = cols[0].size
        assert all(c.size == n for c in cols), "columns differ in length"
        cols = [c if c.size else np.zeros(1, c.dtype) for c in cols]
        self._check(self.lib.arb_set_genomic_breakpoints(self.h, n, *[ptr(c) for c in cols]))

    def mark_genomic_support(self, max_distance=100000, max_itd_length=100):
        """Closest genomic breakpoints of the resident candidates; returns the number of candidates marked."""
        m = C.c_uint32()
        self._check(self.lib.arb_mark_genomic_support(self.h, int(max_distance), int(max_itd_length), C.byref(m)))
        return int(m.value)

    def genomic_support(self):
        """(closest_genomic_breakpoint1, closest_genomic_breakpoint2) of every candidate, -1 = none."""
        n = C.c_uint32()
        self._check(self.lib.arb_candidates_size(self.h, C.byref(n), None, None, None))
        a = np.zeros(max(n.value, 1), np.int32); b = np.zeros(max(n.value, 1), np.int32)
        self._check(self.lib.arb_get_genomic_support(self.h, ptr(a), ptr(b)))
        return a[:n.value], b[:n.value]

    # ---- blacklist (-b)
    RULE_COLUMNS = (("type1", np.uint8), ("type2", np.uint8), ("strand1", np.uint8), ("strand2", np.uint8), ("contig1", np.uint16), ("contig2", np.uint16),
                    ("start1", np.int32), ("end1", np.int32), ("start2", np.int32), ("end2", np.int32), ("gene1", np.uint32), ("gene2", np.uint32))

    def set_blacklist(self, rules):
        """rules: dict of the columns in RULE_COLUMNS, one entry per rule in file order (types and strands as ARB_RULE_* / ARB_RULE_STRAND_*, coordinates 0-based)."""
        cols = [np.ascontiguousarray(rules[k], dt) for k, dt in self.RULE_COLUMNS]
        n = cols[0].size
        assert all(c.size == n for c in cols), "columns differ in length"
        cols = [c if c.size else np.zeros(1, c.dtype) for c in cols]
        self._check(self.lib.arb_set_blacklist(self.h, n, *[ptr(c) for c in cols]))

    def filter_blacklist(self, ids, evalue_cutoff=3.0, max_mate_gap=0):
        """Verdicts (1 = blacklisted) of the candidates `ids` against the rules of set_blacklist."""
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(max(ids.size, 1), np.uint8); n = C.c_uint32()
        self._check(self.lib.arb_filter_blacklist(self.h, ids.size, ptr(ids if ids.size else np.zeros(1, np.uint32)), float(evalue_cutoff), int(max_mate_gap), ptr(out), C.byref(n)))
        return out[:ids.size]

    # ---- known fusions (-k) and tags (-t): the same rule columns as set_blacklist
    def _rule_columns(self, rules):
        cols = [np.ascontiguousarray(rules[k], dt) for k, dt in self.RULE_COLUMNS]
        n = cols[0].size
        assert all(c.size == n for c in cols), "columns differ in length"
        return n, [c if c.size else np.zeros(1, c.dtype) for c in cols]

    def set_known_fusions(self, rules):
        n, cols = self._rule_columns(rules)
        self._check(self.lib.arb_set_known_fusions(self.h, n, *[ptr(c) for c in cols]))

    def recover_known_fusions(self, ids, max_mate_gap=0):
        """Verdicts (1 = rescued) of the candidates `ids` (filter relative_support or min_support, gene1 != gene2) against the rules of set_known_fusions."""
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(max(ids.size, 1), np.uint8); n = C.c_uint32()
        self._check(self.lib.arb_recover_known_fusions(self.h, ids.size, ptr(ids if ids.size else np.zeros(1, np.uint32)), int(max_mate_gap), ptr(out), C.byref(n)))
        return out[:ids.size]

    def set_tags(self, rules, tags):
        """rules: as set_blacklist; tags: the (sanitised) tag of every rule, bytes or str."""
        n, cols = self._rule_columns(rules)
        tags = [t.encode("latin-1") if isinstance(t, str) else bytes(t) for t in tags]
        assert len(tags) == n, "one tag per rule"
        distinct = sorted(set(tags))
        rank = np.array([distinct.index(t) for t in tags] if n else [0], np.uint32)
        off = np.zeros(len(distinct) + 1, np.uint32); off[1:] = np.cumsum([len(t) for t in distinct]) if distinct else []
        chars = b"".join(distinct) + b"\0"
        self._keep.append(chars)
        self._check(self.lib.arb_set_tags(self.h, n, *[ptr(c) for c in cols], ptr(rank), len(distinct), chars, ptr(off)))
        self._tag_names = distinct

    def annotate_tags(self, ids, max_mate_gap=0):
        """The tags of the rows `ids`: a list per candidate (all candidates; the ones not in `ids` have none), each sorted bytewise, as bytes."""
        ids = np.ascontiguousarray(ids, np.uint32)
        pairs = C.c_uint64()
        self._check(self.lib.arb_annotate_tags(self.h, ids.size, ptr(ids if ids.size else np.zeros(1, np.uint32)), int(max_mate_gap), C.byref(pairs)))
        n = C.c_uint32(); n1 = C.c_uint64(); n2 = C.c_uint64(); nd = C.c_uint64()
        self._check(self.lib.arb_candidates_size(self.h, C.byref(n), C.byref(n1), C.byref(n2), C.byref(nd)))
        n = n.value
        off = np.zeros(n + 1, np.uint32); ranks = np.zeros(max(int(pairs.value), 1), np.uint32)
        self._check(self.lib.arb_get_tags(self.h, ptr(off), ptr(ranks)))
        return [[self._tag_names[r] for r in ranks[off[k]:off[k + 1]]] for k in range(n)]

    # ---- protein domains (-p)
    def set_protein_domains(self, contig, start, end, gene, names):
        """The accepted records of a GFF3 file in file order: contig, 0-based start and end, gene, and the decoded name (bytes or str) of every record."""
        cols = [np.ascontiguousarray(contig, np.uint16), np.ascontiguousarray(start, np.int32), np.ascontiguousarray(end, np.int32), np.ascontiguousarray(gene, np.uint32)]
        names = [t.encode("latin-1") if isinstance(t, str) else bytes(t) for t in names]
        n = cols[0].size
        assert all(c.size == n for c in cols) and len(names) == n, "columns differ in length"
        distinct = sorted(set(names))
        index = {t: k for k, t in enumerate(distinct)}
        rank = np.array([index[t] for t in names] if n else [0], np.uint32)
        off = np.zeros(len(distinct) + 1, np.uint32); off[1:] = np.cumsum([len(t) for t in distinct]) if distinct else []
        chars = b"".join(distinct) + b"\0"
        self._keep.append(chars)
        cols = [c if c.size else np.zeros(1, c.dtype) for c in cols]
        self._check(self.lib.arb_set_protein_domains(self.h, n, *[ptr(c) for c in cols], ptr(rank), len(distinct), chars, ptr(off)))

    def retained_protein_domains(self, ids):
        """The retained_protein_domains column (bytes, "." when empty) of every candidate in `ids`, from the tables of set_protein_domains."""
        ids = np.ascontiguousarray(ids, np.uint32)
        nbytes = C.c_uint64()
        self._check(self.lib.arb_retained_protein_domains(self.h, ids.size, ptr(ids if ids.size else np.zeros(1, np.uint32)), C.byref(nbytes)))
        off = np.zeros(ids.size + 1, np.uint64); text = C.create_string_buffer(int(nbytes.value) + 1)
        self._check(self.lib.arb_get_retained_protein_domains(self.h, ptr(off), text))
        raw = text.raw
        return [raw[int(off[x]):int(off[x + 1])] for x in range(ids.size)]

    # ---- gap filling of fusion transcript sequences (-I)
    FILL_THREE, FILL_FORWARD, FILL_ITD = 1, 2, 4

    def set_fill_transcripts(self, first_exon, last_exon, contig, exon_next, exon_prev):
        """The transcripts of the resident annotation (first and last exon, contig) and the exon chains (next / previous exon of the same transcript, -1: none)."""
        t = [np.ascontiguousarray(first_exon, np.int32), np.ascontiguousarray(last_exon, np.int32), np.ascontiguousarray(contig, np.uint32)]
        e = [np.ascontiguousarray(exon_next, np.int32), np.ascontiguousarray(exon_prev, np.int32)]
        n = t[0].size
        assert all(c.size == n for c in t) and e[0].size == e[1].size, "columns differ in length"
        t = [c if c.size else np.zeros(1, c.dtype) for c in t]; e = [c if c.size else np.zeros(1, c.dtype) for c in e]
        self._check(self.lib.arb_set_fill_transcripts(self.h, n, *[ptr(c) for c in t], *[ptr(c) for c in e]))

    def fill_gaps(self, sequences, positions, jobs):
        """Fills the sides of unfilled sequences (bytes, one per row, with the positions of their characters, at least one per character): jobs = (row, transcript, flags) with the
        FILL_* flags. Returns, per job, the filled side (bytes) and its positions: P5 replaces the sequence before its first '|', S3 the one after its last."""
        assert len(sequences) == len(positions)
        row_off = np.zeros(len(sequences) + 1, np.uint32); row_off[1:] = np.cumsum([len(s) for s in sequences]) if sequences else []
        text = b"".join(sequences) + b"\0"
        pos = np.concatenate([np.asarray(p, np.int32) for p in positions] + [np.zeros(1, np.int32)])
        pos_off = np.zeros(len(positions) + 1, np.uint32); pos_off[1:] = np.cumsum([len(p) for p in positions]) if positions else []
        row = np.array([j[0] for j in jobs] or [0], np.uint32); tr = np.array([j[1] for j in jobs] or [0], np.uint32); fl = np.array([j[2] for j in jobs] or [0], np.uint8)
        n = C.c_uint64()
        self._check(self.lib.arb_fill_gaps(self.h, len(sequences), text, ptr(row_off), ptr(pos), ptr(pos_off), len(jobs), ptr(row), ptr(tr), ptr(fl), C.byref(n)))
        off = np.zeros(len(jobs) + 1, np.uint32); chars = C.create_string_buffer(int(n.value) + 1); out_pos = np.zeros(int(n.value) + 1, np.int32)
        self._check(self.lib.arb_get_filled(self.h, ptr(off), chars, ptr(out_pos)))
        raw = chars.raw
        return [(raw[int(off[j]):int(off[j + 1])], out_pos[int(off[j]):int(off[j + 1])].tolist()) for j in range(len(jobs))]

    def slot_swaps(self):
        s = np.zeros(self.n_fragments, np.uint8)
        self._check(self.lib.arb_get_slot_swaps(self.h, ptr(s)))
        return s

    # ---- candidate state, k-mer index, gene homology and re-alignment (filter_homologs, filter_mismappers)
    def set_candidate_state(self, filter, split_reads1, split_reads2, discordant_mates, evalue):
        """Per-candidate columns in candidate order, as arb_get_candidates returns them."""
        cols = [np.ascontiguousarray(a, dt) for a, dt in ((filter, np.uint8), (split_reads1, np.uint32), (split_reads2, np.uint32), (discordant_mates, np.uint32), (evalue, np.float32))]
        cols = [c if c.size else np.zeros(1, c.dtype) for c in cols]
        self._check(self.lib.arb_set_candidate_state(self.h, *[ptr(c) for c in cols]))

    def set_candidate_lists(self, list1_off, list1, list2_off, list2):
        """Replaces the split-read lists (CSR: offsets n + 1, fragment indices) of the resident candidates."""
        cols = [np.ascontiguousarray(a, np.uint32) for a in (list1_off, list1, list2_off, list2)]
        cols = [c if c.size else np.zeros(1, np.uint32) for c in cols]
        self._check(self.lib.arb_set_candidate_lists(self.h, *[ptr(c) for c in cols]))

    def set_splice_sites(self, off, sites):
        """Downstream splice sites per gene: off (n_genes + 1) into the sorted sites of each gene."""
        off = np.ascontiguousarray(off, np.uint32); sites = np.ascontiguousarray(sites, np.int32)
        self._check(self.lib.arb_set_splice_sites(self.h, ptr(off), ptr(sites if sites.size else np.zeros(1, np.int32))))

    def build_kmer_index(self, contig, start, end, n_index_contigs):
        """8-mer index over the intervals [start, end) of positions; returns the number of positions indexed."""
        cols = [np.ascontiguousarray(a, dt) for a, dt in ((contig, np.uint32), (start, np.int32), (end, np.int32))]
        n = cols[0].size
        cols = [c if c.size else np.zeros(1, c.dtype) for c in cols]
        k = C.c_uint64()
        self._check(self.lib.arb_build_kmer_index(self.h, *[ptr(c) for c in cols], n, int(n_index_contigs), C.byref(k)))
        return int(k.value)

    def homolog_pairs(self, gene_a, gene_b):
        """is_homolog(gene_a[j], gene_b[j]) for every j, at the context's max_homolog_identity."""
        a = np.ascontiguousarray(gene_a, np.uint32); b = np.ascontiguousarray(gene_b, np.uint32)
        out = np.zeros(max(a.size, 1), np.uint8)
        self._check(self.lib.arb_homolog_pairs(self.h, ptr(a), ptr(b), a.size, ptr(out)))
        return out[:a.size].astype(bool)

    def filter_mismappers(self, max_mate_gap):
        """Re-aligns the listed reads of the unfiltered candidates; returns the number of (candidate, fragment) items."""
        n = C.c_uint64()
        self._check(self.lib.arb_filter_mismappers(self.h, int(max_mate_gap), C.byref(n)))
        return int(n.value)


# ------------------------------------------------------------------------------------------- whole-run driver
STEP_LOAD_REFERENCE, STEP_INGEST, STEP_ANNOTATE, STEP_UPLOAD, STEP_READ_FILTERS, STEP_FRAGMENT_LENGTH, STEP_FIND_FUSIONS, STEP_COUNT = range(8)
EV_NAMES = ["fetch", "merge_adjacent", "multimappers", "evalue", "non_coding_neighbors", "intragenic_exonic", "min_support", "relative_support", "internal_tandem_duplication",
            "intronic", "in_vitro", "spliced", "select_best", "marginal_read_through", "many_spliced", "short_anchor", "end_to_end", "no_coverage", "kmer_index", "homologs", "mismappers", "select_best2", "isoforms", "confidence"]
EXCHANGE_LABELS, EXCHANGE_CANDIDATES = 0, 1
STEP_NAMES = ["load_reference", "ingest", "annotate", "upload", "read_filters", "fragment_length", "find_fusions"]


class RunOptions(C.Structure):
    _fields_ = [("bam_file", C.c_char_p), ("gtf_file", C.c_char_p), ("assembly_file", C.c_char_p), ("output_file", C.c_char_p),
                ("discarded_output_file", C.c_char_p), ("interesting_contigs", C.c_char_p), ("viral_contigs", C.c_char_p),
                ("params", Params), ("strandedness", C.c_int32), ("fragment_length", C.c_uint32), ("threads", C.c_int32), ("device", C.c_int32),
                ("min_support", C.c_int32), ("min_anchor_length", C.c_uint32), ("min_spliced_events", C.c_uint32), ("high_expression_quantile", C.c_float),
                ("exonic_fraction", C.c_float), ("min_itd_allele_fraction", C.c_float), ("min_itd_support", C.c_uint32),
                ("print_extra_info_for_discarded_fusions", C.c_int32), ("echo_progress", C.c_int32),
                ("top_viral_contigs", C.c_uint32), ("viral_contig_min_covered_fraction", C.c_float),
                ("genomic_breakpoints_file", C.c_char_p), ("max_genomic_breakpoint_distance", C.c_uint32), ("blacklist_file", C.c_char_p),
                ("known_fusions_file", C.c_char_p), ("tags_file", C.c_char_p), ("protein_domains_file", C.c_char_p), ("chimeric_file", C.c_char_p),
                ("fill_sequence_gaps", C.c_int32)]


class RunStats(C.Structure):
    _fields_ = [("n_fragments", C.c_uint64), ("n_records", C.c_uint64), ("mapped_reads", C.c_uint64), ("malformed", C.c_uint64),
                ("strandedness", C.c_int32), ("max_mate_gap", C.c_int32), ("fragment_length_ok", C.c_int32),
                ("mate_gap_mean", C.c_float), ("mate_gap_stddev", C.c_float), ("read_length_mean", C.c_float),
                ("seconds", C.c_double * STEP_COUNT), ("t_inflate", C.c_double), ("t_parse", C.c_double), ("t_finalize", C.c_double),
                ("h2d_bytes", C.c_uint64), ("event_seconds", C.c_double * 32), ("output_seconds", C.c_double), ("n_candidates", C.c_uint64), ("n_unfiltered_candidates", C.c_uint64),
                ("chimeric_records", C.c_uint64), ("chimeric_malformed", C.c_uint64), ("chimeric_total", C.c_uint64)]


def _load_pipeline_api(lib):
    if getattr(lib, "_pipeline_ready", False):
        return
    lib.arb_default_run_options.argtypes = [_p(RunOptions)]
    lib.arb_pipeline_create.argtypes = [_p(C.c_void_p), _p(RunOptions)]
    lib.arb_pipeline_destroy.argtypes = [C.c_void_p]
    lib.arb_pipeline_error.argtypes = [C.c_void_p]; lib.arb_pipeline_error.restype = C.c_char_p
    lib.arb_pipeline_step.argtypes = [C.c_void_p, C.c_int]
    lib.arb_pipeline_run.argtypes = [C.c_void_p]
    lib.arb_pipeline_ctx.argtypes = [C.c_void_p]; lib.arb_pipeline_ctx.restype = C.c_void_p
    lib.arb_pipeline_stats.argtypes = [C.c_void_p, _p(RunStats)]
    lib.arb_pipeline_fragments.argtypes = [C.c_void_p, _p(SoaChunk), _p(C.c_char_p), _p(_p(C.c_uint64))]
    lib.arb_pipeline_genes.argtypes = [C.c_void_p, _p(Annotation)]
    lib.arb_pipeline_coverage.argtypes = [C.c_void_p, C.c_uint32, _p(_p(C.c_uint16)), _p(_p(C.c_uint8)), _p(_p(C.c_uint8)), _p(C.c_uint64)]
    lib.arb_pipeline_events.argtypes = [C.c_void_p, C.c_int]
    lib.arb_pipeline_write_output.argtypes = [C.c_void_p]
    lib.arb_pipeline_candidates.argtypes = [C.c_void_p, _p(Candidates), _p(_p(C.c_uint32)), _p(_p(C.c_uint8)), _p(_p(C.c_uint8))]
    lib.arb_pipeline_attach_device.argtypes = [C.c_void_p]
    lib.arb_pipeline_work_partition.argtypes = [C.c_void_p, C.c_int, _p(_p(C.c_uint32)), _p(_p(C.c_uint8)), _p(C.c_uint32)]
    lib.arb_pipeline_mismappers_begin.argtypes = [C.c_void_p, _p(C.c_int)]
    lib.arb_pipeline_mismappers_end.argtypes = [C.c_void_p]
    lib.arb_pipeline_genomic_support.argtypes = [C.c_void_p, _p(_p(C.c_int32)), _p(_p(C.c_int32))]
    lib._pipeline_ready = True


def _np_from(pointer, n, dtype):
    if n == 0 or not pointer:
        return np.zeros(0, dtype)
    return np.ctypeslib.as_array(pointer, shape=(n,)).astype(dtype, copy=True)


class Pipeline:
    """One run of the hot path on files: the call a user of the library makes (the `arriba` CLI is a thin wrapper over it).

    `bam` is the alignment file: BAM, or SAM text (plain or BGZF-compressed), told apart by the content (DESIGN.md section 5). `chimeric` is STAR's
    separate chimeric alignment file (Chimeric.out.sam, from --chimOutType SeparateSAMold; any of the same formats), read before `bam` (the -c option).
    Either may be a regular file or a path that reads as a stream: a pipe or FIFO ("/dev/stdin", "/dev/fd/N", os.mkfifo) or a character device. A stream
    is read once, in order, while the records are processed; it gives the same results as the same bytes in a file."""

    def __init__(self, bam, gtf, fasta, threads=1, device=0, lib_path=None, strandedness=3, params=None, output=None, discarded=None,
                 genomic_breakpoints=None, max_genomic_breakpoint_distance=100000, blacklist=None, known_fusions=None, tags=None, protein_domains=None,
                 chimeric=None, fill_sequence_gaps=False, extra_info=False, interesting_contigs=None):
        self.lib = load(lib_path)
        _load_pipeline_api(self.lib)
        o = RunOptions()
        self.lib.arb_default_run_options(C.byref(o))
        self._strings = [bam.encode(), gtf.encode(), fasta.encode()]
        o.bam_file, o.gtf_file, o.assembly_file = self._strings
        if output:
            self._strings.append(output.encode()); o.output_file = self._strings[-1]
        if discarded:
            self._strings.append(discarded.encode()); o.discarded_output_file = self._strings[-1]
        if genomic_breakpoints:
            self._strings.append(genomic_breakpoints.encode()); o.genomic_breakpoints_file = self._strings[-1]
        o.max_genomic_breakpoint_distance = max_genomic_breakpoint_distance
        if blacklist:  # read only while the blacklist filter is on (params.filter_mask bit 20)
            self._strings.append(blacklist.encode()); o.blacklist_file = self._strings[-1]
        if known_fusions:  # read only while the known_fusions filter is on (params.filter_mask bit 18)
            self._strings.append(known_fusions.encode()); o.known_fusions_file = self._strings[-1]
        if tags:
            self._strings.append(tags.encode()); o.tags_file = self._strings[-1]
        if protein_domains:
            self._strings.append(protein_domains.encode()); o.protein_domains_file = self._strings[-1]
        if chimeric:
            self._strings.append(chimeric.encode()); o.chimeric_file = self._strings[-1]
        o.fill_sequence_gaps = int(bool(fill_sequence_gaps))  # -I
        o.print_extra_info_for_discarded_fusions = int(bool(extra_info))  # -X
        if interesting_contigs is not None:  # -i: a list of contig names
            self._strings.append(" ".join(interesting_contigs).encode()); o.interesting_contigs = self._strings[-1]
        o.threads = threads; o.device = device; o.strandedness = strandedness
        if params is not None:
            o.params = params
        h = C.c_void_p()
        if self.lib.arb_pipeline_create(C.byref(h), C.byref(o)) != 0:
            raise ArbError(self.lib.arb_pipeline_error(None).decode())
        self.h = h

    def close(self):
        if self.h:
            self.lib.arb_pipeline_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise ArbError(self.lib.arb_pipeline_error(self.h).decode())

    def step(self, s):
        self._check(self.lib.arb_pipeline_step(self.h, s))

    def run(self, upto=STEP_COUNT - 1):
        for s in range(upto + 1):
            self.step(s)

    # ---- one sample on several GPUs (include/arriba_b200.h); the transport is the launcher's, see sharded.py
    def attach_device(self):
        self._check(self.lib.arb_pipeline_attach_device(self.h))

    def work_partition(self, parts):
        k = _p(C.c_uint32)(); o = _p(C.c_uint8)(); n = C.c_uint32()
        self._check(self.lib.arb_pipeline_work_partition(self.h, parts, C.byref(k), C.byref(o), C.byref(n)))
        return _np_from(k, int(n.value), np.uint32), _np_from(o, int(n.value), np.uint8)

    def mismappers_begin(self):
        a = C.c_int()
        self._check(self.lib.arb_pipeline_mismappers_begin(self.h, C.byref(a)))
        return bool(a.value)

    def mismappers_end(self):
        self._check(self.lib.arb_pipeline_mismappers_end(self.h))

    def stats(self):
        s = RunStats()
        self._check(self.lib.arb_pipeline_stats(self.h, C.byref(s)))
        return s

    def context(self):
        """Device context of the pipeline as a (non-owning) Context object."""
        c = Context.__new__(Context)
        c.lib = self.lib; c.h = C.c_void_p(self.lib.arb_pipeline_ctx(self.h)); c._keep = []; c.n_fragments = int(self.stats().n_fragments)
        c.close = lambda: None
        return c

    def fragments(self):
        ch = SoaChunk(); names = C.c_char_p(); off = _p(C.c_uint64)()
        self._check(self.lib.arb_pipeline_fragments(self.h, C.byref(ch), C.byref(names), C.byref(off)))
        n = ch.n_fragments
        out = {"n_fragments": n}
        for k, cnt, dt in (("n_aln", n, np.uint8), ("fflags", n, np.uint8), ("filter", n, np.uint8), ("contig", 3 * n, np.uint16), ("start", 3 * n, np.int32),
                           ("end", 3 * n, np.int32), ("aflags", 3 * n, np.uint8), ("cigar_off", 3 * n, np.uint32), ("cigar_cnt", 3 * n, np.uint16),
                           ("seq_off", 2 * n, np.uint32), ("seq_len", 2 * n, np.uint16), ("genes_off", 3 * n, np.uint32), ("genes_cnt", 3 * n, np.uint16),
                           ("cigar", ch.n_cigar, np.uint32), ("seq", ch.n_seq_bytes, np.uint8), ("genes", ch.n_genes, np.uint32)):
            out[k] = _np_from(getattr(ch, k), cnt, dt)
        name_off = _np_from(off, n + 1, np.uint64)
        raw = C.string_at(C.cast(names, C.c_void_p), int(name_off[-1])) if n else b""
        out["name_off"] = name_off; out["names_blob"] = raw
        return out

    def write_output(self):
        self._check(self.lib.arb_pipeline_write_output(self.h))

    def run_all(self):
        self._check(self.lib.arb_pipeline_run(self.h))

    def events(self, last_stage):
        self._check(self.lib.arb_pipeline_events(self.h, last_stage))

    def candidates(self):
        """Copy of the host candidate table (+ iteration order, confidence, current fragment labels)."""
        c = Candidates(); order = _p(C.c_uint32)(); conf = _p(C.c_uint8)(); labels = _p(C.c_uint8)()
        self._check(self.lib.arb_pipeline_candidates(self.h, C.byref(c), C.byref(order), C.byref(conf), C.byref(labels)))
        n = c.n
        out = {"n": n}
        for k, dt in (("gene1", np.uint32), ("gene2", np.uint32), ("contig1", np.uint16), ("contig2", np.uint16), ("breakpoint1", np.int32), ("breakpoint2", np.int32),
                      ("direction1", np.uint8), ("direction2", np.uint8), ("split_reads1", np.uint32), ("split_reads2", np.uint32), ("discordant_mates", np.uint32),
                      ("filter", np.uint8), ("bits", np.uint8), ("bits2", np.uint8), ("anchor_start1", np.int32), ("anchor_start2", np.int32), ("evalue", np.float32)):
            out[k] = _np_from(getattr(c, k), n, dt)
        for k in ("list1_off", "list2_off", "listd_off"):
            out[k] = _np_from(getattr(c, k), n + 1, np.uint32)
        for k, o in (("list1", "list1_off"), ("list2", "list2_off"), ("listd", "listd_off")):
            out[k] = _np_from(getattr(c, k), int(out[o][-1]) if n else 0, np.uint32)
        out["order"] = _np_from(order, n, np.uint32); out["confidence"] = _np_from(conf, n, np.uint8)
        g1 = _p(C.c_int32)(); g2 = _p(C.c_int32)()
        self._check(self.lib.arb_pipeline_genomic_support(self.h, C.byref(g1), C.byref(g2)))
        out["closest_genomic_breakpoint1"] = _np_from(g1, n, np.int32) if g1 else np.full(n, -1, np.int32)
        out["closest_genomic_breakpoint2"] = _np_from(g2, n, np.int32) if g2 else np.full(n, -1, np.int32)
        out["labels"] = _np_from(labels, int(self.stats().n_fragments), np.uint8)
        return out

    def genes(self):
        a = Annotation()
        self._check(self.lib.arb_pipeline_genes(self.h, C.byref(a)))
        out = {"n_genes": a.n_genes, "n_exons": a.n_exons, "n_contigs": a.n_contigs}
        for k, cnt, dt in (("gene_contig", a.n_genes, np.uint16), ("gene_start", a.n_genes, np.int32), ("gene_end", a.n_genes, np.int32), ("gene_strand", a.n_genes, np.uint8),
                           ("gene_exonic_length", a.n_genes, np.int32), ("gene_flags", a.n_genes, np.uint8), ("exon_gene", a.n_exons, np.uint32),
                           ("exon_start", a.n_exons, np.int32), ("exon_end", a.n_exons, np.int32), ("exon_cds_start", a.n_exons, np.int32), ("exon_cds_end", a.n_exons, np.int32),
                           ("exon_flags", a.n_exons, np.uint8)):
            out[k] = _np_from(getattr(a, k), cnt, dt)
        return out

    def coverage(self, contig):
        cov = _p(C.c_uint16)(); st = _p(C.c_uint8)(); en = _p(C.c_uint8)(); n = C.c_uint64()
        self._check(self.lib.arb_pipeline_coverage(self.h, contig, C.byref(cov), C.byref(st), C.byref(en), C.byref(n)))
        return _np_from(cov, n.value, np.uint16), _np_from(st, n.value, np.uint8), _np_from(en, n.value, np.uint8)
