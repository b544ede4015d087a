"""Bit-level record of the GMM refit, to compare two builds of the library.

    TW_SO=path/to/libtw_b200.so python scripts/refit_identity.py dump OUT.npz
    python scripts/refit_identity.py compare A.npz B.npz

dump: pass 0, the delays of its assignments and tw_gmm_refit(want_selected) on bench.py's streams
(hotel 8192 services, media 2046, alibaba 2016, seed 10) and on every tests/golden directory solved
as one batch; stores each mixture table and selected-K array.  compare: every array of A equals B's
bit for bit (float64 tables compared as uint64); exits 1 otherwise."""
import glob
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def dump(out_path):
    from traceweaver_b200 import _lib
    if os.environ.get("TW_SO"):
        _lib.SO_PATH = os.environ["TW_SO"]
    import torch
    from golden_util import Golden, GOLDEN_DIR
    from traceweaver_b200 import shard
    from traceweaver_b200.batch import build_batch, build_batch_from_blocks
    from traceweaver_b200.engine import Engine

    batches = []
    for wl, ns, n_in in (("hotel", 8192, 1000), ("media", 2046, 1000), ("alibaba", 2016, 1250)):
        blocks = shard.generate_slice(shard.stream_spec(wl, ns, n_in, 10), 0, ns)
        batches.append((f"{wl}_{ns}", lambda b=blocks: build_batch_from_blocks(b)))
    by_dir = {}
    for f in sorted(glob.glob(os.path.join(GOLDEN_DIR, "*__*.npz"))):
        by_dir.setdefault(os.path.basename(f).split("__")[0], []).append(f)
    for name, files in sorted(by_dir.items()):
        batches.append((name, lambda fs=files: build_batch([Golden(f).problem() for f in fs])))

    res = {}
    eng = Engine(0)
    for name, make in batches:
        eng.bind(make())
        eng.prepare()
        p0 = eng.params_pass0()
        sc = eng.score(p0, want_used=True)
        r0 = eng.stitch(p0, sc["cut"], undeleted=sc)
        d, c = eng.delays(r0["assign"])
        prm, nsel = eng.gmm_refit(d, c, want_selected=True)
        torch.cuda.synchronize()
        res[f"{name}__mix"] = prm.table.cpu().numpy()
        res[f"{name}__nsel"] = nsel.cpu().numpy()
        print(f"{name}: {res[f'{name}__mix'].shape[0]} terms, selected K histogram "
              f"{np.bincount(res[f'{name}__nsel'], minlength=6).tolist()}", flush=True)
    eng.close()
    np.savez(out_path, **res)


def bits(a):
    return a.view(np.uint64) if a.dtype == np.float64 else a


def compare(pa, pb):
    a, b = np.load(pa), np.load(pb)
    ok = sorted(a.files) == sorted(b.files)
    if not ok:
        print(f"different arrays: {sorted(set(a.files) ^ set(b.files))}")
    for k in sorted(set(a.files) & set(b.files)):
        same = a[k].shape == b[k].shape and np.array_equal(bits(a[k]), bits(b[k]))
        if not same:
            n = int((bits(a[k]) != bits(b[k])).sum()) if a[k].shape == b[k].shape else -1
            print(f"{k}: DIFFERENT ({n} elements)")
        ok = ok and same
    print(f"{len(a.files)} arrays: {'bit-identical' if ok else 'DIFFERENT'}")
    return ok


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "dump":
        dump(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
    else:
        sys.exit(__doc__)
