"""Generate the golden vectors of the host-side reference comparisons in tests/test_host.py by running the UNMODIFIED
reference (the checkout named by $SSLREC_REFERENCE, by default /root/reference) on CPU.  TEST INFRASTRUCTURE ONLY; the outputs are committed.

    python oracle/gen_golden_host.py            # SSLREC_REFERENCE=<checkout> to read the reference from elsewhere

tests/golden/reference_metrics.npz   Metric.eval_batch (trainer/metrics.py:11-80) on random top-k lists, all four metrics
tests/golden/reference_batches.npz   PairwiseTrnData (data_utils/datasets_general_cf.py:6-26) served by DataLoader(shuffle=True)
                                     over two epochs under fixed numpy / torch seeds, and the RNG states it leaves behind
Each body runs in a subprocess inside the reference tree: its config module parses sys.argv at import.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, 'tests', 'golden')

METRICS = r'''
import os, sys
import numpy as np, torch
ref, out = sys.argv[1], sys.argv[2]
os.chdir(ref)
sys.path.insert(0, ref)
sys.argv = ['main.py', '--model', 'lightgcn', '--device', 'cpu']
from config.configurator import configs
configs['test']['metrics'] = ['recall', 'ndcg', 'precision', 'mrr']
configs['test']['k'] = [5, 20, 40]
from trainer.metrics import Metric
rs = np.random.RandomState(5)
n, n_item, kmax = 300, 500, 40
top = np.stack([rs.permutation(n_item)[:kmax] for _ in range(n)])
truths = [rs.choice(n_item, size=rs.randint(1, 50), replace=False).tolist() for _ in range(n)]
for u in range(n):
    for _ in range(rs.randint(0, 5)):
        top[u, rs.randint(0, kmax)] = truths[u][rs.randint(len(truths[u]))]
want = Metric().eval_batch((torch.from_numpy(top), truths), configs['test']['k'])
np.savez_compressed(out, top=top.astype(np.int32), truth_ptr=np.cumsum([0] + [len(t) for t in truths]).astype(np.int32),
                    truth_flat=np.concatenate(truths).astype(np.int32), k=np.array(configs['test']['k']),
                    **{m: np.asarray(want[m], dtype=np.float64) for m in configs['test']['metrics']})
'''

BATCHES = r'''
import os, sys
import numpy as np, scipy.sparse as sp, torch
import torch.utils.data as tdata
ref, out = sys.argv[1], sys.argv[2]
os.chdir(ref)
sys.path.insert(0, ref)
sys.argv = ['main.py', '--model', 'lightgcn', '--device', 'cpu']
from config.configurator import configs
rs = np.random.RandomState(0)
U, I = 90, 30
key = np.unique(rs.randint(0, U, 1500).astype(np.int64) * I + rs.randint(0, I, 1500))
m = sp.coo_matrix((np.ones(len(key)), (key // I, key % I)), shape=(U, I))
configs['data']['user_num'], configs['data']['item_num'] = U, I
from data_utils.datasets_general_cf import PairwiseTrnData
ds = PairwiseTrnData(m)
loader = tdata.DataLoader(ds, batch_size=128, shuffle=True, num_workers=0)
np.random.seed(11); torch.manual_seed(12)
epochs = []
for _ in range(2):
    ds.sample_negs()
    epochs.append(np.concatenate([np.stack([t.long().numpy() for t in b], 1) for b in loader]))
np.savez_compressed(out, epoch0=epochs[0].astype(np.int32), epoch1=epochs[1].astype(np.int32),
                    numpy_state=np.asarray(np.random.get_state()[1][:8], dtype=np.int64),
                    torch_state=torch.get_rng_state()[:16].numpy().astype(np.int64), batch_size=np.int64(128))
'''


def main():
    ref = os.environ.get('SSLREC_REFERENCE', '/root/reference')
    if not os.path.isdir(ref):
        sys.exit('set SSLREC_REFERENCE to a checkout of the reference')
    for body, name in ((METRICS, 'reference_metrics.npz'), (BATCHES, 'reference_batches.npz')):
        subprocess.run([sys.executable, '-c', body, os.path.abspath(ref), os.path.join(OUT, name)], check=True)
        print(os.path.join(OUT, name))


if __name__ == '__main__':
    main()
