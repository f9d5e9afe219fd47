"""Path and stdout helpers the hot-path classes call (behaviour of the same-named functions of checkm/common.py: same log
messages, same exit codes).  When CheckM itself is importable its own helpers are used, so a drop-in shares one copy."""
import ast
import logging
import os
import sys

import numpy as np

try:                                              # inside a CheckM install: CheckM's own helpers
    from checkm.common import (checkFileExists, checkDirExists, makeSurePathExists, binIdFromFilename,       # noqa: F401
                               getBinIdsFromOutDir, reassignStdOut, restoreStdOut, readDistribution, findNearest)
except Exception:                                 # stand-alone
    def _fatal(message):
        logging.getLogger('timestamp').error(message + '\n')
        sys.exit(1)

    def checkFileExists(inputFile):
        if os.path.exists(inputFile):
            return
        _fatal('Input file does not exists: ' + inputFile)

    def readDistribution(prefix):
        """The dictionary literal of <data root>/distributions/<prefix>.txt (common.py:46-55)."""
        from .defaultValues import DefaultValues
        distFile = os.path.join(DefaultValues.DISTRIBUTION_DIR, prefix + '.txt')
        checkFileExists(distFile)
        with open(distFile, 'r') as f:
            return ast.literal_eval(f.read())

    def findNearest(array, value):
        """The element of array nearest to value; of two equally near ones the first (common.py:58-62)."""
        return array[(np.abs(np.array(array) - value)).argmin()]

    def checkDirExists(inputDir):
        if os.path.exists(inputDir):
            return
        _fatal('Input directory does not exists: ' + inputDir)

    def getBinIdsFromOutDir(outDir):
        """Sub-directories of <outDir>/bins, in directory order (what the reference iterates over)."""
        binDir = os.path.join(outDir, 'bins')
        return [f for f in os.listdir(binDir) if f != 'storage' and os.path.isdir(os.path.join(binDir, f))]

    def makeSurePathExists(path):
        if path:
            try:
                os.makedirs(path, exist_ok=True)
            except OSError:
                _fatal('Specified path does not exist: ' + path)

    def binIdFromFilename(filename):
        """File name without directory, without a trailing .gz, without its last extension."""
        base = os.path.basename(filename)
        base = base[:-3] if base.endswith('.gz') else base
        return os.path.splitext(base)[0]

    class _Redirect(object):
        """stdout diverted into a file for the duration of a report (printSummary's outFile argument)."""
        def __init__(self, path):
            self.previous = sys.stdout
            self.handle = open(path, 'w')
            sys.stdout = self.handle

        def undo(self):
            self.handle.close()
            sys.stdout = self.previous

    def reassignStdOut(outFile):
        if outFile == '':
            return sys.stdout
        try:
            return _Redirect(outFile)
        except IOError:
            _fatal('Error diverting stdout to file: ' + outFile)

    def restoreStdOut(outFile, oldStdOut):
        if outFile != '' and isinstance(oldStdOut, _Redirect):
            oldStdOut.undo()
