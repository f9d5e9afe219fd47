"""Constants and data-file locations read by the hot path (mirror of checkm/defaultValues.py:26-104).

Values are taken from an installed `checkm` when one is importable (so a drop-in shares CheckM's data root);
otherwise from CHECKM_DATA_PATH, which is what checkm/checkmData.py:115-121 honours as well."""
import os


def _data_root():
    root = os.environ.get('CHECKM_DATA_PATH')
    if root:
        return root
    try:                                          # pragma: no cover - only with a full CheckM install
        from checkm.defaultValues import DefaultValues as _DV
        return _DV.CHECKM_DATA_DIR
    except Exception:
        return os.path.join(os.path.expanduser('~'), '.checkm')


class DefaultValues(object):
    MARKERS_TO_EXCLUDE = {'TIGR00398', 'TIGR00399'}          # defaultValues.py:34

    E_VAL = 1e-10
    LENGTH = 0.7
    PSEUDOGENE_LENGTH = 0.3

    TAXON_MARKER_FILE_HEADER = '# [Taxon Marker File]'
    LINEAGE_MARKER_FILE_HEADER = '# [Lineage Marker File]'
    SEQ_CONCAT_CHAR = '&&'

    CHECKM_DATA_DIR = _data_root()
    PHYLO_HMM_MODELS = os.path.join(CHECKM_DATA_DIR, 'hmms', 'phylo.hmm')
    HMM_MODELS = os.path.join(CHECKM_DATA_DIR, 'hmms', 'checkm.hmm')
    PFAM_CLAN_FILE = os.path.join(CHECKM_DATA_DIR, 'pfam', 'Pfam-A.hmm.dat')
    SELECTED_MARKER_SETS = os.path.join(CHECKM_DATA_DIR, 'selected_marker_sets.tsv')
    TAXON_MARKER_SETS = os.path.join(CHECKM_DATA_DIR, 'taxon_marker_sets.tsv')
    GENOME_TREE_DIR = os.path.join(CHECKM_DATA_DIR, 'genome_tree')                      # defaultValues.py:60-70
    DISTRIBUTION_DIR = os.path.join(CHECKM_DATA_DIR, 'distributions')                   # defaultValues.py:71
    GENOME_TREE_METADATA = 'genome_tree.metadata.tsv'
    GENOME_TREE_MISSING_DUPLICATE = 'missing_duplicate_genes_50.tsv'
    PPLACER_TREE_OUT = 'concatenated.tre'                                               # defaultValues.py:89

    PHYLO_HMM_MODEL_INFO = 'phylo_hmm_info.pkl.gz'
    CHECKM_HMM_MODEL_INFO = 'checkm_hmm_info.pkl.gz'
    HMMER_TABLE_PHYLO_OUT = 'hmmer.tree.txt'
    HMMER_PHYLO_OUT = 'hmmer.tree.ali.txt'
    HMMER_TABLE_OUT = 'hmmer.analyze.txt'
    HMMER_OUT = 'hmmer.analyze.ali.txt'
    PRODIGAL_AA = 'genes.faa'
    PRODIGAL_NT = 'genes.fna'
    PRODIGAL_GFF = 'genes.gff'
    BIN_STATS_PHYLO_OUT = 'bin_stats.tree.tsv'
    BIN_STATS_OUT = 'bin_stats.analyze.tsv'
    BIN_STATS_EXT_OUT = 'bin_stats_ext.tsv'
    MARKER_GENE_STATS = 'marker_gene_stats.tsv'
    MIN_SEQ_LEN_GC_STD = 1000

    @classmethod
    def set_data_root(cls, root):
        """Re-point every data path (tests and embedded use)."""
        cls.CHECKM_DATA_DIR = root
        cls.PHYLO_HMM_MODELS = os.path.join(root, 'hmms', 'phylo.hmm')
        cls.HMM_MODELS = os.path.join(root, 'hmms', 'checkm.hmm')
        cls.PFAM_CLAN_FILE = os.path.join(root, 'pfam', 'Pfam-A.hmm.dat')
        cls.SELECTED_MARKER_SETS = os.path.join(root, 'selected_marker_sets.tsv')
        cls.TAXON_MARKER_SETS = os.path.join(root, 'taxon_marker_sets.tsv')
        cls.GENOME_TREE_DIR = os.path.join(root, 'genome_tree')
        cls.DISTRIBUTION_DIR = os.path.join(root, 'distributions')
