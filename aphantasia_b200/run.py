"""Launcher: run an UNMODIFIED reference script (clip_fft.py, illustra.py, ...) against the CUDA drop-in.

    python -m aphantasia_b200.run /path/to/aphantasia/clip_fft.py -t "red square" --size 1280-720 --samples 200 -nv
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
        -m aphantasia_b200.run /path/to/aphantasia/clip_fft.py -t "..." --size 3840-2160 --samples 800 -m ViT-B/16 -nv

Why a launcher: `python /path/clip_fft.py` puts the SCRIPT's directory at sys.path[0], ahead of PYTHONPATH, so
`from aphantasia.image import ...` (clip_fft.py:24-25) would resolve to the reference's own package sitting next to the
script, not to dropin/aphantasia. Here dropin/ is inserted ahead of the script directory, the reference's module names
(`aphantasia`, `clip`, `imageio`, `lpips`, `depth`, `eps`) are imported FIRST and checked to come from dropin/, and only then the
script runs as __main__ (runpy). cppn.py defines its network class in the script itself, where no import can replace it: a
script whose top level defines `class CPPN` and `def main` runs through run_cppn_script instead (see there). Before it runs,
torchvision.transforms.functional.affine is routed through
aphantasia_b200.motion (illustrip.py's per-frame camera motion; clip_fft.py never calls it). Equivalent without this module:
`PYTHONSAFEPATH=1 PYTHONPATH=<repo>/dropin:<repo> python clip_fft.py`. For illustrip.py that runs the drop-in too, but its
per-frame motion stays on torchvision's own path unless `aphantasia_b200.motion.install()` is called before the script runs.
"""
import atexit
import os
import runpy
import sys
import time

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
DROPIN = os.path.join(ROOT, 'dropin')
SHADOWED = ('aphantasia', 'clip', 'imageio', 'lpips', 'depth', 'eps')


def install_dropin(script_dir=None):
    """Puts dropin/ (and the repo root) ahead of everything else on sys.path, evicts foreign copies of the shadowed
    module names, imports ours and verifies their origin. Returns {name: file}."""
    for p in (DROPIN, ROOT):
        while p in sys.path:
            sys.path.remove(p)
    head = [DROPIN, ROOT] + ([script_dir] if script_dir else [])
    sys.path[:0] = head
    for k in [k for k in list(sys.modules) if k.split('.')[0] in SHADOWED]:
        f = getattr(sys.modules[k], '__file__', None) or ''
        if not os.path.abspath(f).startswith(DROPIN + os.sep):
            del sys.modules[k]
    origins = {}
    import importlib
    for name in SHADOWED:
        try:
            m = importlib.import_module(name)
        except ImportError:
            if name in ('imageio', 'lpips'):      # stand-ins for packages this image lacks; a real install is fine too
                continue
            raise
        f = os.path.abspath(getattr(m, '__file__', '') or '')
        origins[name] = f
        if name in ('aphantasia', 'clip', 'depth', 'eps') and not f.startswith(DROPIN + os.sep):
            raise RuntimeError('aphantasia_b200.run: `%s` resolved to %s, not to %s -- the script would run the reference '
                               'PyTorch path, not libaphb200.so' % (name, f, DROPIN))
    return origins


def cppn_script(path):
    """True when the script's top level (read with ast, nothing is run) defines `class CPPN` and `def main`, as cppn.py does."""
    import ast
    with open(path, 'rb') as f:
        tree = ast.parse(f.read(), filename=path)
    classes = {n.name for n in tree.body if isinstance(n, ast.ClassDef)}
    funcs = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
    return 'CPPN' in classes and 'main' in funcs


def check_cppn_equivalence(theirs, ours, nf=8, layers=3, seed=1234):
    """Builds both classes on the CPU under one seed, for every activation, and requires identical state dicts (keys, shapes,
    values): the script's seeded run then starts from the same weights. The global CPU generator is left as it was."""
    import torch
    for act in ('unbias', 'comp', 'relu'):
        sds = []
        for cls in (theirs, ours):
            with torch.random.fork_rng(devices=[]):
                torch.manual_seed(seed)
                sds.append(cls(2, nf, layers, 3, act_fn=act).state_dict())
        a, b = sds
        if list(a) != list(b):
            raise NotImplementedError('aphantasia_b200.run: the script\'s CPPN (act_fn=%r) has state-dict keys %s, ours %s'
                                      % (act, list(a), list(b)))
        for k in a:
            if a[k].shape != b[k].shape or not torch.equal(a[k], b[k]):
                raise NotImplementedError('aphantasia_b200.run: the script\'s CPPN (act_fn=%r) differs from aphantasia_b200.cppn.CPPN '
                                          'in %s (%s vs %s under one seed)' % (act, k, tuple(a[k].shape), tuple(b[k].shape)))


def run_cppn_script(script):
    """Runs a cppn.py-style script with its CPPN replaced by aphantasia_b200.cppn.CPPN: the module body runs under another
    __name__ (so its `if __name__ == '__main__'` does not fire), the two classes are checked to build identical state dicts,
    then `CPPN` is rebound in main's globals, __name__ set to '__main__' and main() called."""
    import builtins
    from . import cppn
    with open(script, 'rb') as f:
        code = compile(f.read(), script, 'exec')
    g = {'__name__': '__aph_cppn_script__', '__file__': script, '__builtins__': builtins, '__package__': None, '__spec__': None}
    exec(code, g)
    check_cppn_equivalence(g['CPPN'], cppn.CPPN)
    main = g['main']
    main.__globals__['CPPN'] = cppn.CPPN
    main.__globals__['__name__'] = '__main__'
    main()


def _summary(t0):
    try:
        from . import _lib
        n = _lib.lib().aph_launch_count() if _lib._lib is not None else 0
    except Exception:
        n = -1
    sys.stderr.write('\n[aphantasia_b200.run] kernels launched by libaphb200.so: %d, wall %.2f s\n' % (n, time.time() - t0))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] in ('-h', '--help'):
        sys.stderr.write(__doc__ + '\n')
        return 2
    script = os.path.abspath(argv[0])
    if not os.path.isfile(script):
        sys.stderr.write('aphantasia_b200.run: no such script: %s\n' % script)
        return 2
    origins = install_dropin(os.path.dirname(script))
    from . import motion
    motion.install()
    if os.environ.get('APH_FUSED_ADAM', '0') == '1':          # row f2: torch.optim.Adam / AdamW over our generators -> fused into their backward
        from . import optim
        optim.install()
    if os.environ.get('APH_RUN_VERBOSE', '0') == '1':
        for k, v in origins.items():
            sys.stderr.write('[aphantasia_b200.run] %s -> %s\n' % (k, v))
    sys.argv = [script] + argv[1:]
    atexit.register(_summary, time.time())
    if cppn_script(script):
        run_cppn_script(script)
    else:
        runpy.run_path(script, run_name='__main__')
    return 0


if __name__ == '__main__':
    sys.exit(main())
