"""ResultsParser / ResultsManager (mirror of checkm/resultsParser.py) with the hit reduction on the device.

Same public surface and attributes the rest of CheckM reaches into (`.results[binId].markerHits`, `.models`,
`analyseResults`, `parseBinHits`, `printSummary`, `cacheResults`, `parseBinStats*`, `parseMarkerGeneStats`;
hit objects with the `HmmerHitDOM` attribute names) -- SURVEY.md section 8b.  What moved: the per-bin Python loop of
regex parsing -> vetHit -> addHit -> re-reading Pfam-A.hmm.dat -> clan filter -> adjacent-ORF merge
(resultsParser.py:76-119,191-217,340-479) is one `ckm_reduce` call over all bins (checkm_b200/csrc/reduce.cu);
gene counts, completeness and contamination (resultsParser.py:513-537, markerSets.py:206-238) come from
`ckm_genome_check`.  Rows are taken from the binary side-car the search wrote next to each domtblout file when it is
present and current, else from the domtblout text itself (so a stand-alone `checkm qa` on an old `analyze` directory
still works); both go through the same text rounding the reference applies (hmmer.py:268-276)."""
import ast
import ctypes as C
import decimal
import logging
import os
import sys
from collections import defaultdict

import numpy as np

from . import _lib, runtime
from ._lib import CkmError, check
from .common import checkFileExists, reassignStdOut, restoreStdOut
from .defaultValues import DefaultValues
from .engine import HIT_DTYPE
from .hmmer import HMMERParser, read_sidecar
from .util.pfam import PFAM

INT32_MIN = -2 ** 31

QA_DTYPE = np.dtype([('bin', np.int32), ('counts', np.int32, 6), ('n_markers', np.int32), ('n_sets', np.int32),
                     ('unique_hits', np.int32), ('multi_hits', np.int32), ('completeness', np.float64),
                     ('contamination', np.float64)], align=True)
MH_DTYPE = np.dtype([(n, np.int64 if n == 'dict_key' else np.int32) for n, _ in _lib.MarkerHit._fields_], align=True)
assert QA_DTYPE.itemsize == C.sizeof(_lib.QaRow) and MH_DTYPE.itemsize == C.sizeof(_lib.MarkerHit)


class MarkerHit(object):
    """A hit as ResultsManager.markerHits holds it: HmmerHitDOM attribute names, values as the text round trip gives them."""
    __slots__ = ('target_name', 'target_accession', 'target_length', 'query_name', 'query_accession', 'query_length',
                 'full_e_value', 'full_score', 'full_bias', 'dom', 'ndom', 'c_evalue', 'i_evalue', 'dom_score',
                 'dom_bias', 'hmm_from', 'hmm_to', 'ali_from', 'ali_to', 'env_from', 'env_to', 'acc',
                 'target_description')

    def __str__(self):
        return "\t".join(str(getattr(self, f)) for f in self.__slots__)


def _decimal_split(x):
    """x = mant * 10^(exp10-1) with 10 <= mant < 100, from the shortest decimal text of x (exact for 1e-10 etc.)."""
    if x <= 0:
        return INT32_MIN, 0.0
    d = decimal.Decimal(repr(float(x)))
    exp10 = d.adjusted()
    mant = d.scaleb(-(exp10 - 1))
    return int(exp10), float(mant)


def _parse_table_text(path):
    """domtblout text -> (rows, names, descs, query (name, acc) per model id) in file order."""
    rows = []
    parsed = []
    names, name_idx, descs = [], {}, []
    qids, qid_idx = [], {}
    with open(path) as f:
        hp = HMMERParser(f)
        while True:
            hit = hp.next()
            if hit is None:
                break
            s = name_idx.get(hit.target_name)
            if s is None:
                s = name_idx[hit.target_name] = len(names)
                names.append(hit.target_name)
                descs.append(hit.target_description)
            q = qid_idx.get((hit.query_name, hit.query_accession))
            if q is None:
                q = qid_idx[(hit.query_name, hit.query_accession)] = len(qids)
                qids.append((hit.query_name, hit.query_accession))
            parsed.append(hit)
            rows.append((0, s, q, hit.target_length, hit.query_length, hit.dom, hit.ndom, hit.hmm_from, hit.hmm_to,
                         hit.ali_from, hit.ali_to, hit.env_from, hit.env_to, hit.full_score, hit.full_bias, hit.dom_score,
                         hit.dom_bias, hit.acc, hit.full_e_value, hit.c_evalue, hit.i_evalue, 0.0, 0.0))
    arr = np.array(rows, dtype=HIT_DTYPE) if rows else np.zeros(0, dtype=HIT_DTYPE)
    return arr, names, descs, qids, parsed


def load_hit_table(path):
    """Rows of one bin's domtblout: binary side-car if present and not older than the text, else the text."""
    side = path + '.ckm.npz'
    if os.path.exists(side) and os.path.exists(path) and os.path.getmtime(side) >= os.path.getmtime(path):
        return read_sidecar(path) + (None,)
    return _parse_table_text(path)


def device_genome_check(set_lists, counts_per_set_marker, individual):
    """ckm_genome_check over `set_lists` = per bin, list of lists of copy numbers."""
    nb = len(set_lists)
    bin_off = np.zeros(nb + 1, dtype=np.int64)
    set_off = [0]
    flat = []
    for b, sets in enumerate(set_lists):
        for cnts in sets:
            flat.extend(cnts)
            set_off.append(len(flat))
        bin_off[b + 1] = len(set_off) - 1
    set_off = np.asarray(set_off, dtype=np.int64)
    flat = np.asarray(flat, dtype=np.int32)
    out = np.zeros(nb, dtype=QA_DTYPE)
    check(_lib.lib().ckm_genome_check(runtime.engine()._h, nb, bin_off.ctypes.data, set_off.ctypes.data,
                                      flat.ctypes.data if len(flat) else None, 1 if individual else 0, out.ctypes.data))
    return out


class ResultsParser(object):
    def __init__(self, binIdToModels):
        self.logger = logging.getLogger('timestamp')
        self.results = {}
        self.models = binIdToModels

    # ------------------------------------------------------------------ driver
    def analyseResults(self, outDir, binStatsFile, hmmTableFile, bIgnoreThresholds=False,
                       evalueThreshold=DefaultValues.E_VAL, lengthThreshold=DefaultValues.LENGTH,
                       bSkipPseudoGeneCorrection=False, bSkipAdjCorrection=False):
        binStats = self.parseBinStats(outDir, binStatsFile)
        self.parseBinHits(outDir, hmmTableFile, bSkipAdjCorrection, bIgnoreThresholds, evalueThreshold, lengthThreshold,
                          bSkipPseudoGeneCorrection, binStats)
        return binStats

    def cacheResults(self, outDir, binIdToBinMarkerSets, bIndividualMarkers):
        self._writeBinStatsExt(outDir, binIdToBinMarkerSets, bIndividualMarkers)
        self._writeMarkerGeneStats(outDir, binIdToBinMarkerSets, bIndividualMarkers)

    def parseBinHits(self, outDir, hmmTableFile, bSkipAdjCorrection=False, bIgnoreThresholds=False,
                     evalueThreshold=DefaultValues.E_VAL, lengthThreshold=DefaultValues.LENGTH,
                     bSkipPseudoGeneCorrection=False, binStats=None):
        if not self.models:
            self.logger.error('Models must be parsed before identifying HMM hits.')
            sys.exit(1)
        self.logger.info('Parsing HMM hits to marker genes:')
        binIds = list(self.models.keys())
        tables = {}
        import time as _time
        t0 = _time.perf_counter()
        for binId in binIds:
            path = os.path.join(outDir, 'bins', binId, hmmTableFile)
            try:
                tables[binId] = load_hit_table(path)
            except IOError as detail:
                sys.stderr.write(str(detail) + "\n")          # the reference carries on with an empty result
                tables[binId] = (np.zeros(0, dtype=HIT_DTYPE), [], [], [], None)
        self.timing = {'load_tables': _time.perf_counter() - t0}      # seconds per phase of the last call (bench.py reports them)
        try:
            reduced = self._reduce(binIds, tables, bIgnoreThresholds, evalueThreshold, lengthThreshold,
                                   bSkipPseudoGeneCorrection, bSkipAdjCorrection)
        except CkmError as err:
            self.logger.error('reduction engine exited with code: %d (%s)' % (err.code, err))
            sys.exit(err.code)
        for binId in binIds:
            rm = ResultsManager(binId, self.models[binId], bIgnoreThresholds, evalueThreshold, lengthThreshold,
                                bSkipPseudoGeneCorrection, binStats[binId] if binStats is not None else None)
            rm.markerHits = reduced[binId]
            self.results[binId] = rm

    def parseHmmerResults(self, fileName, resultsManager, bSkipAdjCorrection):
        """Single-file form (resultsParser.py:191-217): fills `resultsManager.markerHits`."""
        try:
            table = load_hit_table(fileName)
        except IOError as detail:
            sys.stderr.write(str(detail) + "\n")
            return
        binId = resultsManager.binId
        saved = self.models
        try:
            self.models = {binId: resultsManager.models}
            reduced = self._reduce([binId], {binId: table}, resultsManager.bIgnoreThresholds, resultsManager.evalueThreshold,
                                   resultsManager.lengthThreshold, resultsManager.bSkipPseudoGeneCorrection, bSkipAdjCorrection)
        finally:
            self.models = saved
        resultsManager.markerHits = reduced[binId]

    # ------------------------------------------------------------------ device reduction
    def _reduce(self, binIds, tables, bIgnoreThresholds, evalueThreshold, lengthThreshold, bSkipPseudo, bSkipAdj):
        # global model table = every accession of every bin's model dict
        accs, acc_idx = [], {}
        distinct = {}                           # bins usually share one model dict (HMM file, taxon file): visit it once
        for binId in binIds:
            distinct.setdefault(id(self.models[binId]), self.models[binId])
        for md in distinct.values():
            for acc in md:
                if acc not in acc_idx:
                    acc_idx[acc] = len(accs)
                    accs.append(acc)
        nm = len(accs)
        has = np.zeros((nm, 3), dtype=np.int32)
        cut = np.zeros((nm, 6), dtype=np.float64)
        is_tigr = np.zeros(nm, dtype=np.uint8)
        for md in distinct.values():
            for acc, model in md.items():
                i = acc_idx[acc]
                for z, attr in enumerate(('ga', 'tc', 'nc')):
                    v = getattr(model, attr, None)
                    if v is not None:
                        has[i, z] = 1
                        cut[i, 2 * z], cut[i, 2 * z + 1] = v[0], v[1]
                is_tigr[i] = 1 if 'TIGR' in model.acc else 0
        pf = PFAM(DefaultValues.PFAM_CLAN_FILE)
        if os.path.exists(DefaultValues.PFAM_CLAN_FILE):
            is_pfam, clan, nest_off, nest_idx = pf.reduction_tables(accs)
        else:
            checkFileExists(DefaultValues.PFAM_CLAN_FILE)
        # rows, sequences
        all_rows, scaffold_id, orf_num, name_rank = [], [], [], []
        seq_base, bases = 0, {}
        scaf_ids = {}
        row_q = {}
        text_scores, any_text, parsed_all = [], False, []
        for b, binId in enumerate(binIds):
            rows, names, descs, qids, parsed = tables[binId]
            bases[binId] = seq_base
            if parsed is not None:
                any_text = True
                text_scores.append(np.asarray([(h.full_score, h.dom_score) for h in parsed], dtype=np.float64).reshape(-1, 2))
                parsed_all.extend(parsed)
            else:                               # binary rows: the same rounding the text round trip applies, vectorised
                text_scores.append(np.rint(np.stack([rows['full_score'], rows['dom_score']], axis=1).astype(np.float64) * 10.0) / 10.0)
                parsed_all.extend([None] * len(rows))
            order = {n: r for r, n in enumerate(sorted(set(names)))}
            for n in names:
                cut_at = n.rfind('_')
                scaf = n[0:cut_at]
                scaffold_id.append(scaf_ids.setdefault((b, scaf), len(scaf_ids)))
                try:
                    v = int(n[cut_at + 1:])
                    v = v if -2 ** 31 + 2 <= v <= 2 ** 31 - 2 else INT32_MIN + 1
                except ValueError:
                    v = INT32_MIN
                orf_num.append(v)
                name_rank.append(order[n])
            if len(rows):
                r = rows.copy()
                r['bin'] = b
                r['seq'] += seq_base
                qmap = np.empty(len(qids), dtype=np.int32)
                for q, (qname, qacc) in enumerate(qids):
                    key = qacc if qacc not in ('-', '') else qname
                    if key not in acc_idx or key not in self.models[binId]:
                        raise KeyError(key)               # the reference raises the same KeyError in vetHit
                    qmap[q] = acc_idx[key]
                r['model'] = qmap[r['model']]
                all_rows.append(r)
            seq_base += len(names)
        hits = np.concatenate(all_rows) if all_rows else np.zeros(0, dtype=HIT_DTYPE)
        nseq = seq_base
        scaffold_id = np.asarray(scaffold_id, dtype=np.int32)
        orf_num = np.asarray(orf_num, dtype=np.int32)
        name_rank = np.asarray(name_rank, dtype=np.int32)
        opts = _lib.ReduceOpts()
        opts.ignore_thresholds = 1 if bIgnoreThresholds else 0
        opts.skip_pseudogene = 1 if bSkipPseudo else 0
        opts.skip_adjacent = 1 if bSkipAdj else 0
        opts.individual_markers = 0
        opts.evalue_threshold = float(evalueThreshold)
        opts.evalue_exp10, opts.evalue_mant = _decimal_split(evalueThreshold)
        opts.length_threshold = float(lengthThreshold)
        opts.pseudogene_length = float(DefaultValues.PSEUDOGENE_LENGTH)
        meta = _lib.ReduceMeta()
        keep = [is_pfam, is_tigr, clan, nest_off, nest_idx, scaffold_id, orf_num, name_rank, has, cut]
        meta.is_pfam = is_pfam.ctypes.data
        meta.is_tigr = is_tigr.ctypes.data
        meta.clan = clan.ctypes.data
        meta.nest_off = nest_off.ctypes.data
        meta.nest_idx = nest_idx.ctypes.data if len(nest_idx) else None
        meta.scaffold_id = scaffold_id.ctypes.data if nseq else None
        meta.orf_num = orf_num.ctypes.data if nseq else None
        meta.name_rank = name_rank.ctypes.data if nseq else None
        meta.has_cut = has.ctypes.data
        meta.cutoffs = cut.ctypes.data
        row_scores = np.ascontiguousarray(np.concatenate(text_scores)) if (any_text and len(hits)) else None
        meta.row_scores = row_scores.ctypes.data if row_scores is not None else None
        qa = C.POINTER(_lib.QaRow)()
        nqa = C.c_int32()
        mh = C.POINTER(_lib.MarkerHit)()
        nmh = C.c_int64()
        harr = np.ascontiguousarray(hits)
        import time as _time
        _t1 = _time.perf_counter()
        check(_lib.lib().ckm_reduce(runtime.engine()._h, nm, nseq, len(binIds), harr.ctypes.data_as(C.POINTER(_lib.Hit)),
                                    len(harr), C.byref(opts), C.byref(meta), C.byref(qa), C.byref(nqa), C.byref(mh), C.byref(nmh)))
        _t2 = _time.perf_counter()
        if hasattr(self, 'timing'):
            self.timing['reduce_call'] = _t2 - _t1
        del keep
        if nmh.value:
            buf = (C.c_char * (nmh.value * C.sizeof(_lib.MarkerHit))).from_address(C.addressof(mh.contents))
            marker_hits = np.frombuffer(buf, dtype=MH_DTYPE).copy()
        else:
            marker_hits = np.zeros(0, dtype=MH_DTYPE)
        _lib.lib().ckm_free(qa)
        _lib.lib().ckm_free(mh)
        # back to {binId: {acc: [hits]}} in the reference's dict order: non-Pfam markers in file order, then Pfam markers.
        # Columns are pulled out of the record arrays once (plain Python lists): indexing numpy records hit by hit is what
        # this loop would otherwise spend its time on.
        out = {}
        mh = {f: marker_hits[f].tolist() for f in ('bin', 'model', 'seq_a', 'seq_b', 'target_length', 'hmm_from', 'hmm_to', 'ali_from',
                                                   'ali_to', 'env_from', 'env_to', 'order', 'src_row', 'dict_key')}
        src_rows = harr[marker_hits['src_row']] if len(marker_hits) else harr[:0]
        sc = {f: src_rows[f].tolist() for f in ('seq', 'tlen', 'qlen', 'dom', 'ndom', 'full_score', 'full_bias', 'dom_score', 'dom_bias', 'acc',
                                                'full_evalue', 'c_evalue', 'i_evalue')}
        per_bin = defaultdict(list)
        for z, bb in enumerate(mh['bin']):
            per_bin[bb].append(z)
        concat = DefaultValues.SEQ_CONCAT_CHAR
        for b, binId in enumerate(binIds):
            rows, names, descs, qids, _parsed = tables[binId]
            base = bases[binId]
            qname_of = {}
            for qn, qa_ in qids:
                qname_of.setdefault(qa_ if qa_ not in ('-', '') else qn, qn)
            groups, keys = {}, {}
            for pos, z in enumerate(per_bin.get(b, ())):
                acc = accs[mh['model'][z]]
                lst = groups.get(acc)
                if lst is None:
                    lst = groups[acc] = []
                    dk = mh['dict_key'][z]
                    keys[acc] = (0, pos) if dk < 0 else (1, dk)
                original = parsed_all[mh['src_row'][z]]
                hit = MarkerHit()
                if original is not None:
                    for f in MarkerHit.__slots__:
                        setattr(hit, f, getattr(original, f))
                else:
                    si = sc['seq'][z] - base
                    hit.target_name = names[si]
                    hit.target_accession = '-'
                    hit.query_name = qname_of.get(acc, acc)
                    hit.query_accession = acc
                    hit.query_length = sc['qlen'][z]
                    hit.full_e_value = float('%9.2g' % sc['full_evalue'][z])
                    hit.full_score = float('%6.1f' % sc['full_score'][z])
                    hit.full_bias = float('%5.1f' % sc['full_bias'][z])
                    hit.dom, hit.ndom = sc['dom'][z], sc['ndom'][z]
                    hit.c_evalue = float('%9.2g' % sc['c_evalue'][z])
                    hit.i_evalue = float('%9.2g' % sc['i_evalue'][z])
                    hit.dom_score = float('%6.1f' % sc['dom_score'][z])
                    hit.dom_bias = float('%5.1f' % sc['dom_bias'][z])
                    hit.acc = float('%4.2f' % sc['acc'][z])
                    hit.target_description = descs[si] if descs else ''
                if mh['seq_b'][z] >= 0:
                    # the merged object is hits[i] mutated (resultsParser.py:451-470): scores and description stay
                    hit.target_name = concat.join([names[mh['seq_a'][z] - base], names[mh['seq_b'][z] - base]])
                hit.target_length = mh['target_length'][z]
                hit.hmm_from, hit.hmm_to = mh['hmm_from'][z], mh['hmm_to'][z]
                hit.ali_from, hit.ali_to = mh['ali_from'][z], mh['ali_to'][z]
                hit.env_from, hit.env_to = mh['env_from'][z], mh['env_to'][z]
                lst.append((mh['order'][z], hit))
            ordered = {}
            for acc in sorted(groups, key=lambda k: keys[k]):
                ordered[acc] = [h for _, h in sorted(groups[acc], key=lambda t: t[0])]
            out[binId] = ordered
        if hasattr(self, 'timing'):
            self.timing['hit_objects'] = _time.perf_counter() - _t2
        return out

    # ------------------------------------------------------------------ cached tsv files
    def _writeBinStatsExt(self, directory, binIdToBinMarkerSets, bIndividualMarkers):
        path = os.path.join(directory, 'storage', DefaultValues.BIN_STATS_EXT_OUT)
        self._device_counts(binIdToBinMarkerSets, bIndividualMarkers)
        with open(path, 'w') as fout:
            for binId in self.results:
                ext = self.results[binId].getSummary(binIdToBinMarkerSets[binId], bIndividualMarkers, outputFormat=2)
                ext.update(self.results[binId].geneCopyNumber(binIdToBinMarkerSets[binId]))
                fout.write(binId + '\t' + str(ext) + '\n')

    def _writeMarkerGeneStats(self, directory, binIdToBinMarkerSets, bIndividualMarkers):
        path = os.path.join(directory, 'storage', DefaultValues.MARKER_GENE_STATS)
        with open(path, 'w') as fout:
            for binId in self.results:
                stats = self.results[binId].getSummary(binIdToBinMarkerSets[binId], bIndividualMarkers, outputFormat=8)
                fout.write(binId + '\t' + str(stats) + '\n')

    def _read_dict_file(self, path):
        checkFileExists(path)
        out = {}
        with open(path, 'r') as f:
            for line in f:
                fields = line.split('\t')
                out[fields[0]] = ast.literal_eval(fields[1])
        return out

    def parseBinStats(self, resultsFolder, binStatsFile):
        return self._read_dict_file(os.path.join(resultsFolder, 'storage', binStatsFile))

    def parseBinStatsExt(self, resultsFolder):
        return self._read_dict_file(os.path.join(resultsFolder, 'storage', DefaultValues.BIN_STATS_EXT_OUT))

    def parseMarkerGeneStats(self, resultsFolder):
        return self._read_dict_file(os.path.join(resultsFolder, 'storage', DefaultValues.MARKER_GENE_STATS))

    # ------------------------------------------------------------------ summaries
    def _device_counts(self, binIdToBinMarkerSets, bIndividualMarkers):
        """One ckm_genome_check call for the selected marker set of every bin; results cached on the managers."""
        binIds = [b for b in sorted(self.results.keys()) if b in binIdToBinMarkerSets]
        if not binIds:
            return
        set_lists, orders = [], []
        for binId in binIds:
            ms = binIdToBinMarkerSets[binId].selectedMarkerSet()
            hitsd = self.results[binId].markerHits
            set_lists.append([[len(hitsd.get(marker, ())) for marker in s] for s in ms.markerSet])
        rows = device_genome_check(set_lists, None, bIndividualMarkers)
        for binId, row in zip(binIds, rows):
            ms = binIdToBinMarkerSets[binId].selectedMarkerSet()
            self.results[binId]._cache_counts(ms, bIndividualMarkers, row)

    def _getHeader(self, outputFormat, binMarkerSets, coverageBinProfiles=None, table=None):
        if outputFormat == 1:
            return ['Bin Id', 'Marker lineage', '# genomes', '# markers', '# marker sets', '0', '1', '2', '3', '4', '5+',
                    'Completeness', 'Contamination', 'Strain heterogeneity']
        if outputFormat == 2:
            header = ['Bin Id', 'Marker lineage', '# genomes', '# markers', '# marker sets', 'Completeness', 'Contamination',
                      'Strain heterogeneity', 'Genome size (bp)', '# ambiguous bases', '# scaffolds', '# contigs',
                      'N50 (scaffolds)', 'N50 (contigs)', 'Mean scaffold length (bp)', 'Mean contig length (bp)',
                      'Longest scaffold (bp)', 'Longest contig (bp)', 'GC', 'GC std (scaffolds > 1kbp)', 'Coding density',
                      'Translation table', '# predicted genes', '0', '1', '2', '3', '4', '5+']
            if coverageBinProfiles is not None:
                for bamId in coverageBinProfiles[list(coverageBinProfiles.keys())[0]]:
                    header += ['Coverage (' + bamId + ')', 'Coverage std (' + bamId + ')']
            return header
        if outputFormat == 3:
            return ['Bin Id', 'Node Id', 'Marker lineage', '# genomes', '# markers', '# marker sets', '0', '1', '2', '3', '4',
                    '5+', 'Completeness', 'Contamination', 'Strain heterogeneity']
        if outputFormat == 4:
            return None
        if outputFormat == 5:
            return ['Bin Id', 'Marker Id', 'Gene Id']
        if outputFormat in (6, 7):
            return ['Bin Id', 'Marker Id', 'Gene Ids']
        if outputFormat == 8:
            return ['Bin Id', 'Gene Id', '{Marker Id, Start position, End position}']
        if outputFormat == 9:
            if table is not None:
                return ['Bin Id', 'Contig', 'Gene Number', 'Gene Start', 'Gene End', 'Gene Strand', 'Prot Length', 'Marker Id',
                        'Align Start', 'Align End', 'Sequence']
            return " "
        if outputFormat == 10:
            return ['Scaffold Id', 'Bin Id', 'Length', '# contigs', 'GC', '# ORFs', 'Coding density', 'Marker Ids']
        return None

    def printSummary(self, outputFormat, aai, binIdToBinMarkerSets, bIndividualMarkers, coverageFile, bTabTable, outFile, anaFolder):
        oldStdOut = reassignStdOut(outFile)
        coverageBinProfiles = None
        if coverageFile:
            from .coverage import Coverage
            coverageBinProfiles = Coverage(1).binProfiles(coverageFile)
        self._device_counts(binIdToBinMarkerSets, bIndividualMarkers)
        prettyTableFormats = [1, 2, 3, 9]
        header = self._getHeader(outputFormat, binIdToBinMarkerSets[list(binIdToBinMarkerSets.keys())[0]], coverageBinProfiles, bTabTable)
        pTable = None
        if bTabTable or outputFormat not in prettyTableFormats:
            bTabTable = True
            if header is not None:
                print('\t'.join(header))
        else:
            pTable = _make_pretty_table(header)
        seqsReported = 0
        for binId in sorted(self.results.keys()):
            seqsReported += self.results[binId].printSummary(outputFormat, aai, binIdToBinMarkerSets[binId], bIndividualMarkers,
                                                             coverageBinProfiles, pTable, anaFolder)
        if outputFormat in [6, 7] and seqsReported == 0:
            print('[No marker genes satisfied the reporting criteria.]')
        if not bTabTable:
            if outputFormat in [1, 2]:
                print(pTable.get_string(sortby='Completeness', reversesort=True))
            elif pTable.get_string(print_empty=False):
                print(pTable.get_string(print_empty=False))
        restoreStdOut(outFile, oldStdOut)


def _make_pretty_table(header):
    return _FrameTable(header)


class _FrameTable(object):
    """The one table style CheckM prints (resultsParser.py:246-252: centred cells, first column left-aligned, floats as
    %.2f, a rule of dashes above and below the header and at the bottom, no vertical rules), with the calls its callers
    make: add_row, get_string(sortby=, reversesort=, print_empty=).  Cells are framed as the vendored table class frames
    them when vertical rules are off: a blank where each rule would be plus one blank of padding either side."""

    def __init__(self, header):
        self.header = list(header)
        self.rows = []

    def add_row(self, row):
        if len(row) != len(self.header):
            raise Exception("Row has incorrect number of values, (actual) %d!=%d (expected)" % (len(row), len(self.header)))
        self.rows.append(list(row))

    @staticmethod
    def _cell(v):
        return ('%.2f' % v) if isinstance(v, float) else str(v)

    def get_string(self, sortby=None, reversesort=False, print_empty=True):
        if not self.rows and not print_empty:
            return ''
        rows = self.rows
        if sortby is not None:
            i = self.header.index(sortby)
            rows = sorted(rows, key=lambda r: [r[i]] + r, reverse=reversesort)      # ties fall through to the whole row
        cells = [[self._cell(v) for v in r] for r in rows]
        widths = [max([len(h)] + [len(c[i]) for c in cells]) for i, h in enumerate(self.header)]
        rule = '-' * (sum(widths) + 3 * len(widths) + 1)

        def line(values):
            out = [' ']
            for i, (v, w) in enumerate(zip(values, widths)):
                out.append(' ' + (v.ljust(w) if i == 0 else v.center(w)) + ' ')
                out.append(' ')
            return ''.join(out)

        lines = [rule, line(self.header), rule]
        for c in cells:
            lines.append(line(c))
        lines.append(rule)
        return '\n'.join(lines)


class ResultsManager(object):
    """All marker hits of one bin, plus the summaries derived from them."""

    def __init__(self, binId, models, bIgnoreThresholds=False, evalueThreshold=DefaultValues.E_VAL,
                 lengthThreshold=DefaultValues.LENGTH, bSkipPseudoGeneCorrection=False, binStats=None):
        self.binId = binId
        self.markerHits = {}
        self.bIgnoreThresholds = bIgnoreThresholds
        self.evalueThreshold = evalueThreshold
        self.lengthThreshold = lengthThreshold
        self.bSkipPseudoGeneCorrection = bSkipPseudoGeneCorrection
        self.models = models
        self.binStats = binStats
        self._counts_cache = {}

    # ---- per-hit rules: the device applies these in ckm_reduce; kept callable for code that feeds hits one by one ----
    def vetHit(self, hit):
        model = self.models[hit.query_accession]
        if not self.bSkipPseudoGeneCorrection:
            if float(hit.ali_to - hit.ali_from) / float(hit.query_length) < DefaultValues.PSEUDOGENE_LENGTH:
                return False
        for cutoff, guard in ((model.nc, 'TIGR' in model.acc), (model.ga, True), (model.tc, True), (model.nc, True)):
            if cutoff is not None and not self.bIgnoreThresholds and guard:
                return cutoff[0] <= hit.full_score and cutoff[1] <= hit.dom_score
        if hit.full_e_value > self.evalueThreshold:
            return False
        return float(hit.ali_to - hit.ali_from) / float(hit.query_length) >= self.lengthThreshold

    def addHit(self, hit):
        if not self.vetHit(hit):
            return
        current = self.markerHits.setdefault(hit.query_accession, [])
        for old in current:
            if old.target_name == hit.target_name:
                if old.dom_score < hit.dom_score:
                    current.append(hit)
                    current.remove(old)
                return
        current.append(hit)

    def countUniqueHits(self):
        unique = multi = 0
        for hits in self.markerHits.values():
            if len(hits) == 1:
                unique += 1
            elif len(hits) > 1:
                multi += 1
        return unique, multi

    def hitsToMarkerGene(self, markerSet):
        return dict((marker, len(self.markerHits.get(marker, ()))) for marker in markerSet.getMarkerGenes())

    def _cache_counts(self, markerSet, bIndividualMarkers, row):
        self._counts_cache[(id(markerSet), bool(bIndividualMarkers))] = \
            [int(v) for v in row['counts']] + [float(row['completeness']), float(row['contamination'])]

    def geneCountsForSelectedMarkerSet(self, binMarkerSets, bIndividualMarkers):
        ms = binMarkerSets.selectedMarkerSet()
        cached = self._counts_cache.get((id(ms), bool(bIndividualMarkers)))
        if cached is not None:
            return list(cached)
        return self.geneCounts(ms, self.markerHits, bIndividualMarkers)

    def geneCounts(self, markerSet, markerHits, bIndividualMarkers):
        """[n0, n1, n2, n3, n4, n5+, completeness, contamination] for any `{marker: hits}` dict, computed on the device."""
        sets = [[len(markerHits.get(marker, ())) for marker in s] for s in markerSet.markerSet]
        row = device_genome_check([sets], None, bIndividualMarkers)[0]
        return [int(v) for v in row['counts']] + [float(row['completeness']), float(row['contamination'])]

    def geneCopyNumber(self, binMarkerSets):
        out = dict(('GCN' + k, []) for k in ('0', '1', '2', '3', '4', '5+'))
        wanted = binMarkerSets.selectedMarkerSet().getMarkerGenes()
        for marker in self.models:
            if marker not in wanted:
                continue
            n = len(self.markerHits.get(marker, ()))
            out['GCN5+' if n >= 5 else 'GCN' + str(n)].append(os.path.splitext(marker)[0])
        return out

    def _selected_hits(self, binMarkerSets):
        wanted = binMarkerSets.selectedMarkerSet().getMarkerGenes()
        for marker, hits in self.markerHits.items():
            if marker in wanted:
                yield marker, hits

    def getSummary(self, binMarkerSets, bIndividualMarkers, outputFormat=1):
        summary = {}
        if outputFormat in (1, 2):
            ms = binMarkerSets.selectedMarkerSet()
            data = self.geneCountsForSelectedMarkerSet(binMarkerSets, bIndividualMarkers)
            summary['marker lineage'] = ms.lineageStr
            summary['# genomes'] = ms.numGenomes
            summary['# markers'] = ms.numMarkers()
            summary['# marker sets'] = ms.numSets()
            for i, k in enumerate(('0', '1', '2', '3', '4', '5+')):
                summary[k] = data[i]
            summary['Completeness'] = data[6]
            summary['Contamination'] = data[7]
            if outputFormat == 2:
                summary.update(self.binStats)
        elif outputFormat == 5:
            for marker, hits in self._selected_hits(binMarkerSets):
                summary[marker] = [h.target_name for h in hits]
        elif outputFormat == 6:
            for marker, hits in self._selected_hits(binMarkerSets):
                if len(hits) >= 2:
                    summary[marker] = [h.target_name for h in hits]
        elif outputFormat == 7:
            per_gene = defaultdict(dict)
            for marker, hits in self._selected_hits(binMarkerSets):
                for h in hits:
                    per_gene[h.target_name][marker] = per_gene[h.target_name].get(marker, 0) + 1
            for gene, counts in per_gene.items():
                for marker, n in counts.items():
                    if n > 1:
                        summary.setdefault(gene, {})[marker] = n
        elif outputFormat == 8:
            per_gene = {}
            for marker, hits in self._selected_hits(binMarkerSets):
                for h in hits:
                    per_gene.setdefault(h.target_name, []).append(h)
            for gene, hits in per_gene.items():
                summary[gene] = {}
                for h in hits:
                    summary[gene].setdefault(h.query_accession, []).append([h.ali_from, h.ali_to])
        else:
            print("Unknown output format: ", outputFormat)
        return summary

    def printSummary(self, outputFormat, aai, binMarkerSets, bIndividualMarkers, coverageBinProfiles=None, table=None, anaFolder=None):
        hetero = aai.aaiMeanBinHetero.get(self.binId, 0.0) if aai is not None else 0.0
        if outputFormat in (1, 2):
            ms = binMarkerSets.selectedMarkerSet()
            lineage = ms.lineageStr
            if ms.UID != '0':
                lineage += ' (' + str(ms.UID) + ')'
            data = self.geneCountsForSelectedMarkerSet(binMarkerSets, bIndividualMarkers)
            if outputFormat == 1:
                if table is None:
                    print("%s\t%s\t%d\t%d\t%d\t%s\t%0.2f\t%0.2f\t%0.2f" % (self.binId, lineage, ms.numGenomes, ms.numMarkers(), ms.numSets(),
                                                                         "\t".join(str(data[i]) for i in range(6)), data[6], data[7], hetero))
                else:
                    table.add_row([self.binId, lineage, ms.numGenomes, ms.numMarkers(), ms.numSets()] + data + [hetero])
            else:
                bs = self.binStats
                if table is None:
                    row = self.binId
                    row += '\t%s\t%d\t%d\t%d' % (lineage, ms.numGenomes, ms.numMarkers(), ms.numSets())
                    row += '\t%0.2f\t%0.2f\t%0.2f' % (data[6], data[7], hetero)
                    row += '\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d' % (bs['Genome size'], bs['# ambiguous bases'], bs['# scaffolds'], bs['# contigs'],
                                                                         bs['N50 (scaffolds)'], bs['N50 (contigs)'], bs['Mean scaffold length'],
                                                                         bs['Mean contig length'], bs['Longest scaffold'], bs['Longest contig'])
                    row += '\t%.1f\t%.2f' % (bs['GC'] * 100, bs['GC std'] * 100)
                    row += '\t%.2f\t%d\t%d' % (bs['Coding density'] * 100, bs['Translation table'], bs['# predicted genes'])
                    row += '\t' + '\t'.join(str(data[i]) for i in range(6))
                    if coverageBinProfiles:
                        if self.binId in coverageBinProfiles:
                            for _, cov in coverageBinProfiles[self.binId].items():
                                row += '\t%.2f\t%.2f' % (cov[0], cov[1])
                        else:
                            for _ in coverageBinProfiles[list(coverageBinProfiles.keys())[0]]:
                                row += '\t%.2f\t%.2f' % (0, 0)
                    print(row)
                else:
                    row = [self.binId, lineage, ms.numGenomes, ms.numMarkers(), ms.numSets(), data[6], data[7], hetero,
                           bs['Genome size'], bs['# ambiguous bases'], bs['# scaffolds'], bs['# contigs'], bs['N50 (scaffolds)'],
                           bs['N50 (contigs)'], int(bs['Mean scaffold length']), int(bs['Mean contig length']), bs['Longest scaffold'],
                           bs['Longest contig'], bs['GC'] * 100, bs['GC std'] * 100, bs['Coding density'] * 100,
                           bs['Translation table'], bs['# predicted genes']] + data[0:6]
                    if coverageBinProfiles:
                        if self.binId in coverageBinProfiles:
                            for _, cov in coverageBinProfiles[self.binId].items():
                                row.extend(cov)
                        else:
                            for _ in coverageBinProfiles[list(coverageBinProfiles.keys())[0]]:
                                row.extend([0, 0])
                    table.add_row(row)
        elif outputFormat == 3:
            for ms in binMarkerSets.markerSetIter():
                data = self.geneCounts(ms, self.markerHits, bIndividualMarkers)
                if table is None:
                    print("%s\t%s\t%s\t%d\t%d\t%d\t%s\t%0.2f\t%0.2f\t%0.2f" % (self.binId, ms.UID, ms.lineageStr, ms.numGenomes, ms.numMarkers(),
                                                                             ms.numSets(), "\t".join(str(data[i]) for i in range(6)), data[6], data[7], hetero))
                else:
                    table.add_row([self.binId, ms.UID, ms.lineageStr, ms.numGenomes, ms.numMarkers(), ms.numSets()] + data + [hetero])
        elif outputFormat == 4:
            ms = binMarkerSets.selectedMarkerSet()
            data = self.hitsToMarkerGene(ms)
            print("Node Id: %s; Marker lineage: %s" % (ms.UID, ms.lineageStr) + ''.join('\t' + m for m in data))
            print(self.binId + ''.join('\t' + str(c) for c in data.values()))
            print()
        elif outputFormat == 5:
            for marker, hits in self._selected_hits(binMarkerSets):
                for h in hits:
                    print(self.binId, marker, h.target_name, sep='\t', end='\n')
        elif outputFormat == 6:
            reported = 0
            for marker, hits in self._selected_hits(binMarkerSets):
                if len(hits) >= 2:
                    print(self.binId, marker, sep='\t', end='\t')
                    print(','.join(sorted(h.target_name for h in hits)), end='\n')
                    reported += 1
            return reported
        elif outputFormat == 7:
            reported = 0
            for marker, hits in self._selected_hits(binMarkerSets):
                if len(hits) < 2:
                    continue
                shared = set()
                for i in range(len(hits)):
                    scaffold = hits[i].target_name[0:hits[i].target_name.rfind('_')]
                    for j in range(i + 1, len(hits)):
                        if scaffold == hits[j].target_name[0:hits[j].target_name.rfind('_')]:
                            shared.add(hits[i].target_name)
                            shared.add(hits[j].target_name)
                if len(shared) >= 2:
                    print(self.binId, marker, sep='\t', end='\t')
                    print(','.join(sorted(shared)), end='\n')
                    reported += 1
            return reported
        elif outputFormat == 8:
            per_gene = {}
            for marker, hits in self._selected_hits(binMarkerSets):
                for h in hits:
                    per_gene.setdefault(h.target_name, []).append(h)
            for gene, hits in per_gene.items():
                print(self.binId + '\t' + gene + ''.join('\t%s,%d,%d' % (h.query_accession, h.ali_from, h.ali_to) for h in hits))
        elif outputFormat == 9:
            self._print_marker_fasta(binMarkerSets, table, anaFolder)
        else:
            logging.getLogger('timestamp').error("Unknown output format: %d", outputFormat)
        return 0

    def _print_marker_fasta(self, binMarkerSets, table, anaFolder):
        """Format 9: the marker ORFs of the bin as FASTA (or a table) with alignment coordinates (resultsParser.py:887-968)."""
        if anaFolder is None:
            raise ValueError("AnaFolder must not be None for outputFormat 9")
        info = {}
        for marker, hits in self._selected_hits(binMarkerSets):
            for h in hits:
                info[h.target_name] = (marker, str(h.ali_from), str(h.ali_to))
        seqs, order = {}, []
        header = None
        with open("/".join([anaFolder, "bins", self.binId, "genes.faa"])) as f:
            for line in f:
                if line.startswith('>'):
                    header = line[1:].rstrip()
                    seqs[header] = []
                    order.append(header)
                elif header is not None:
                    seqs[header].append(line.strip())
        keep = [h for h in order if h.split(" # ")[0] in info]

        def contig_and_number(h):
            contig, num = h.split(" # ")[0].rsplit("_", 1)
            return contig, int(num)

        for h in sorted(keep, key=contig_and_number):
            seq = ''.join(seqs[h])
            elems = h.split(" # ")
            gene = elems[0]
            contig, num = gene.rsplit("_", 1)
            start, end, strand = elems[1], elems[2], elems[3]
            marker, afrom, ato = info[gene]
            if table is not None:
                gene_info = "geneId={};start={};end={};strand={};protlen={}".format(num, start, end, strand, str(len(seq)))
                marker_info = "marker={};mstart={};mend={}".format(marker, afrom, ato)
                print(">" + " ".join([self.binId, contig, gene_info, marker_info]), seq, sep="\n")
            else:
                print("\t".join([self.binId, contig, num, start, end, strand, str(len(seq)), marker, afrom, ato, seq]))
