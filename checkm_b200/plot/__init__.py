"""The plots (`gc_plot`, `coding_plot`, `tetra_plot`, `dist_plot`, `gc_bias_plot`, `nx_plot`, `len_hist`, `marker_plot`) behind the
reference's class names (checkm/plot/*.py).  Importing this package imports matplotlib; nothing else in checkm_b200 does."""
