"""Convert the reference's ligand-size prior table (utils/evaluation/atom_num_config.py: CONFIG['bounds'], CONFIG['bins'])
into the compact JSON the product loads (targetdiff_b200/data/atom_num_prior.json).  Build container only.

    python tools/make_atom_num_prior.py
"""
import importlib.util
import json
import os

REF = os.environ.get('TARGETDIFF_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'targetdiff_b200', 'data', 'atom_num_prior.json')

spec = importlib.util.spec_from_file_location('atom_num_config', os.path.join(REF, 'utils', 'evaluation', 'atom_num_config.py'))
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)
cfg = mod.CONFIG
out = {'source': 'guanjq/targetdiff utils/evaluation/atom_num_config.py (program-generated empirical table)',
       'bounds': [float(b) for b in cfg['bounds']],
       'bins': [{'num_atoms': [int(n) for n in nums], 'prob': [float(p) for p in probs]} for nums, probs in cfg['bins']]}
with open(OUT, 'w') as f:
    json.dump(out, f, separators=(',', ':'))
print(OUT, os.path.getsize(OUT), 'bytes;', len(out['bounds']), 'bounds,', len(out['bins']), 'bins')
