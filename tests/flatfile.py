"""Write an XGMFLAT1 file (the format oracle/ref_runner `export` produces) from Python structures, so
hand-made edge-case indexes can be loaded by both the oracle and the CUDA path."""
import struct

import numpy as np


def write_flat(path, doclen, terms, wdf_ub_db=None, doccount=None):
    """doclen: array indexed by docid (entry 0 unused, 0 = unused docid).
    terms: list of (name, docids, wdfs), names ascending (like Database::allterms_begin).
    doccount: the number of documents, where some have length 0 (only boolean terms)."""
    doclen = np.asarray(doclen, np.uint32)
    lastdocid = len(doclen) - 1
    used = doclen[1:][doclen[1:] > 0]
    doccount = int(len(used)) if doccount is None else int(doccount)
    total = int(doclen.sum())
    lb = int(used.min()) if doccount else 0
    ub = int(used.max()) if doccount else 0
    db_wub = wdf_ub_db if wdf_ub_db is not None else max([int(np.max(w)) if len(w) else 0 for _, _, w in terms] + [0])
    with open(path, "wb") as f:
        f.write(b"XGMFLAT1")
        f.write(struct.pack("<IIQIIII", doccount, lastdocid, total, len(terms), 0, lb, ub))
        f.write(doclen.tobytes())
        for name, d, w in terms:
            d = np.asarray(d, np.uint32)
            w = np.asarray(w, np.uint32)
            nm = name.encode() if isinstance(name, str) else name
            tf, cf = len(d), int(w.sum())
            if cf == 0 or tf == 1:
                wub = cf
            else:
                wub = max(cf - int(w[0]), int(w[0]))
            wub = min(wub, db_wub)
            f.write(struct.pack("<I", len(nm)) + nm + struct.pack("<IQII", tf, cf, wub, tf))
            f.write(d.tobytes())
            f.write(w.tobytes())
