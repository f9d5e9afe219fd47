"""A stand-in `matplotlib` that records what a plot does to its figure and axes instead of drawing it.

`install()` puts the stand-in modules into sys.modules (matplotlib, .figure, .backends.backend_agg, .transforms, .patches,
.ticker, .colors, .colorbar) and `uninstall()` takes them out again; nothing is installed on import.  Every method call on a figure, canvas or axes is
appended to LOG as [object, method, args, kwargs]; every attribute set on a tick, tick line or spine, and every rcParams
entry, as [object, '=name', value].  Numbers -- Python or numpy scalars, and the elements of lists, tuples and arrays --
are logged as float.hex of their float64 value, so two logs are equal only if every value is bit-equal.  get_xlim,
get_ylim and get_yticks return fixed values, so plots that read them see the same numbers.  Constructing a Rectangle,
MaxNLocator, ListedColormap, Normalize or ColorbarBase is logged as [instance, class, args, kwargs], the instance named by
class and a counter.  Tick labels returned by set_xticklabels / set_yticklabels measure as the fixed box LABEL_BOX
(get_window_extent, transformed, Bbox.union), so label extents read the same numbers too.  `plot(x, y, ...)` with x and y
of different lengths raises ValueError, as matplotlib does."""
import sys
import types

import numpy as np

LOG = []
XLIM = (-0.25, 0.25)
YLIM = (0.0, 12000.0)
YTICKS = (0.0, 3000.0, 6000.0, 9000.0, 12000.0)
_MODULES = ('matplotlib', 'matplotlib.figure', 'matplotlib.backends', 'matplotlib.backends.backend_agg',
            'matplotlib.transforms', 'matplotlib.patches', 'matplotlib.ticker', 'matplotlib.colors', 'matplotlib.colorbar')
_saved = {}
_figures = [0]
_instances = {}


def canon(v):
    """A value as it is logged: numbers as float.hex strings, sequences as lists, recorders by name."""
    if v is None or isinstance(v, (bool, np.bool_, str)):
        return bool(v) if isinstance(v, np.bool_) else v
    if isinstance(v, (int, float, np.integer, np.floating)):
        return float.hex(float(v))
    if isinstance(v, np.ndarray):
        return canon(v.tolist())
    if isinstance(v, (list, tuple)):
        return [canon(x) for x in v]
    if isinstance(v, dict):
        return {str(k): canon(v[k]) for k in sorted(v, key=str)}
    if isinstance(v, _Recorder):
        return '<%s>' % object.__getattribute__(v, '_name')
    return repr(v)


class _Recorder(object):
    """Logs every method call and every attribute set under its name."""

    def __init__(self, name):
        object.__setattr__(self, '_name', name)

    def __getattr__(self, attr):
        if attr.startswith('__'):
            raise AttributeError(attr)
        name = object.__getattribute__(self, '_name')

        def call(*args, **kwargs):
            LOG.append([name, attr, canon(args), canon(kwargs)])
            return None
        return call

    def __setattr__(self, attr, value):
        LOG.append([object.__getattribute__(self, '_name'), '=' + attr, canon(value)])


class _Axis(_Recorder):
    def __init__(self, name):
        _Recorder.__init__(self, name)
        object.__setattr__(self, 'name', name)
        object.__setattr__(self, 'majorTicks', [_Recorder('%s.tick%d' % (name, i)) for i in range(len(YTICKS))])

    def get_ticklines(self):
        LOG.append([self.name, 'get_ticklines', [], {}])
        return [_Recorder('%s.line%d' % (self.name, i)) for i in range(2 * len(YTICKS))]


class _Box(object):
    """A fixed bounding box, in figure fractions: what every tick label measures."""
    x0, y0, x1, y1 = 0.0, 0.0, 0.125, 0.03125
    width, height = x1 - x0, y1 - y0

    def transformed(self, transform):
        return self


LABEL_BOX = _Box()


class _Label(object):
    def get_window_extent(self, renderer=None):
        return LABEL_BOX


class _Transform(object):
    def inverted(self):
        return self


class Bbox(object):
    @staticmethod
    def union(bboxes):
        LOG.append(['Bbox', 'union', [canon(len(bboxes))], {}])
        return LABEL_BOX


def _logged(kind, **attrs):
    """A class whose construction is logged; attrs name recorders every instance carries (e.g. a colour bar's outline)."""
    def __init__(self, *args, **kwargs):
        k = _instances.get(kind, 0)
        _instances[kind] = k + 1
        name = '%s%d' % (kind, k)
        _Recorder.__init__(self, name)
        LOG.append([name, kind, canon(args), canon(kwargs)])
        for a, suffix in attrs.items():
            object.__setattr__(self, a, _Recorder(name + suffix))
    return type(kind, (_Recorder,), {'__init__': __init__})


class _Spines(object):
    def __init__(self, name):
        self._spines = [(loc, _Recorder('%s.spine.%s' % (name, loc))) for loc in ('left', 'right', 'bottom', 'top')]

    def items(self):
        return list(self._spines)


class Axes(_Recorder):
    def __init__(self, name):
        _Recorder.__init__(self, name)
        object.__setattr__(self, 'xaxis', _Axis(name + '.xaxis'))
        object.__setattr__(self, 'yaxis', _Axis(name + '.yaxis'))
        object.__setattr__(self, 'spines', _Spines(name))

    def _get(self, what, value):
        LOG.append([object.__getattribute__(self, '_name'), what, [], {}])
        return value

    def get_xlim(self):
        return self._get('get_xlim', XLIM)

    def get_ylim(self):
        return self._get('get_ylim', YLIM)

    def get_yticks(self):
        return self._get('get_yticks', np.array(YTICKS))

    def get_yaxis(self):
        return self._get('get_yaxis', object.__getattribute__(self, 'yaxis'))

    def _ticklabels(self, what, labels, kwargs):
        LOG.append([object.__getattribute__(self, '_name'), what, canon((labels,)), canon(kwargs)])
        return [_Label() for _ in labels]

    def set_xticklabels(self, labels, **kwargs):
        return self._ticklabels('set_xticklabels', labels, kwargs)

    def set_yticklabels(self, labels, **kwargs):
        return self._ticklabels('set_yticklabels', labels, kwargs)

    def plot(self, *args, **kwargs):
        LOG.append([object.__getattribute__(self, '_name'), 'plot', canon(args), canon(kwargs)])
        if len(args) >= 2 and all(hasattr(a, '__len__') and not isinstance(a, str) for a in args[:2]) \
                and len(args[0]) != len(args[1]):
            raise ValueError('x and y must have same first dimension, but have shapes (%d,) and (%d,)'
                             % (len(args[0]), len(args[1])))


class Figure(_Recorder):
    def __init__(self, *args, **kwargs):
        name = 'fig%d' % _figures[0]
        _figures[0] += 1
        _Recorder.__init__(self, name)
        LOG.append([name, 'Figure', canon(args), canon(kwargs)])

    def add_subplot(self, *args, **kwargs):
        name = object.__getattribute__(self, '_name')
        LOG.append([name, 'add_subplot', canon(args), canon(kwargs)])
        return Axes('%s.ax%s' % (name, ''.join(str(a) for a in args)))

    def add_axes(self, *args, **kwargs):
        name = object.__getattribute__(self, '_name')
        LOG.append([name, 'add_axes', canon(args), canon(kwargs)])
        k = _instances.get(name, 0)
        _instances[name] = k + 1
        return Axes('%s.axes%d' % (name, k))

    transFigure = _Transform()


class FigureCanvasAgg(object):
    def __init__(self, figure):
        self._figure_name = object.__getattribute__(figure, '_name')
        LOG.append([self._figure_name, 'FigureCanvasAgg', [], {}])

    def draw(self):
        LOG.append([self._figure_name, 'draw', [], {}])

    def get_renderer(self):
        LOG.append([self._figure_name, 'get_renderer', [], {}])
        return _Recorder(self._figure_name + '.renderer')


class _RcParams(dict):
    def __setitem__(self, key, value):
        LOG.append(['rcParams', '=' + key, canon(value)])
        dict.__setitem__(self, key, value)


def reset():
    """Empties the log and numbers figures from 0 again."""
    del LOG[:]
    _figures[0] = 0
    _instances.clear()


def install():
    """The stand-in modules into sys.modules (what was there before is restored by uninstall)."""
    mods = {m: types.ModuleType(m) for m in _MODULES}
    mods['matplotlib'].rcParams = _RcParams()
    mods['matplotlib'].figure = mods['matplotlib.figure']
    mods['matplotlib'].backends = mods['matplotlib.backends']
    mods['matplotlib'].transforms = mods['matplotlib.transforms']
    mods['matplotlib'].patches = mods['matplotlib.patches']
    for sub in ('ticker', 'colors', 'colorbar'):
        setattr(mods['matplotlib'], sub, mods['matplotlib.' + sub])
    mods['matplotlib.backends'].backend_agg = mods['matplotlib.backends.backend_agg']
    mods['matplotlib.figure'].Figure = Figure
    mods['matplotlib.backends.backend_agg'].FigureCanvasAgg = FigureCanvasAgg
    mods['matplotlib.transforms'].Bbox = Bbox
    mods['matplotlib.patches'].Rectangle = _logged('Rectangle')
    mods['matplotlib.ticker'].MaxNLocator = _logged('MaxNLocator')
    mods['matplotlib.colors'].ListedColormap = _logged('ListedColormap')
    mods['matplotlib.colors'].Normalize = _logged('Normalize')
    mods['matplotlib.colorbar'].ColorbarBase = _logged('ColorbarBase', outline='.outline', dividers='.dividers')
    for m in _MODULES:
        if m in sys.modules:
            _saved[m] = sys.modules[m]
        sys.modules[m] = mods[m]
    reset()


def uninstall():
    for m in _MODULES:
        sys.modules.pop(m, None)
        if m in _saved:
            sys.modules[m] = _saved.pop(m)
