"""Pin the reference's ligand class maps (utils/transforms.py MAP_ATOM_TYPE_{ONLY,AROMATIC,FULL}_TO_INDEX) as data:
tests/golden/reference_ligand_class_maps.json, which tests/test_type_constraints.py compares with targetdiff_b200.pocket's tables.

    TARGETDIFF_REFERENCE=/path/to/targetdiff python -m oracle.make_class_map_pins

The three dict literals are read with `ast` from the reference file, unmodified and without importing it.  Each map is stored as a
list of [key, index] pairs, the key a list (an atomic number alone for the 'basic' map)."""
import ast
import json
import os

from .refload import REFERENCE_ROOT

NAMES = {'basic': 'MAP_ATOM_TYPE_ONLY_TO_INDEX', 'add_aromatic': 'MAP_ATOM_TYPE_AROMATIC_TO_INDEX', 'full': 'MAP_ATOM_TYPE_FULL_TO_INDEX'}
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'reference_ligand_class_maps.json')


def main():
    src = open(os.path.join(REFERENCE_ROOT, 'utils', 'transforms.py')).read()
    found = {}
    for node in ast.parse(src).body:
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name):
            found[node.targets[0].id] = node.value
    pins = {}
    for mode, name in NAMES.items():
        d = ast.literal_eval(found[name])
        pins[mode] = [[list(k) if isinstance(k, tuple) else [k], int(v)] for k, v in sorted(d.items(), key=lambda kv: kv[1])]
    with open(OUT, 'w') as f:
        f.write('{\n%s\n}\n' % ',\n'.join('%s: %s' % (json.dumps(m), json.dumps(p)) for m, p in pins.items()))
    print('wrote %s: %s' % (OUT, {m: len(p) for m, p in pins.items()}))


if __name__ == '__main__':
    main()
