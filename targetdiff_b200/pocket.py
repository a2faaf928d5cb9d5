"""Pocket ingest without RDKit / PyG: fixed-column PDB ATOM records -> ProteinLigandData with the 27-dim protein atom feature.

Mirrors what the reference does before the sampling path (SURVEY.md 8(f) n1):
  * utils/data.py:67-95  `PDBProtein._enum_formatted_atom_lines` (ATOM records, fixed columns, stop at ENDMDL, element from
    columns 77-78 or the atom-name column), :98-113 (element number, position, backbone flag, residue -> amino-acid index),
    :151-159 `to_dict_atom`;
  * utils/transforms.py:115-132 `FeaturizeProteinAtom`: one-hot over (H, C, N, O, S, Se) + one-hot over 20 amino acids + backbone flag;
  * scripts/sample_for_pocket.py:18-31 `pdb_to_pocket_data` (empty ligand).
Only the periodic-table lookups the featurizer needs are kept (the reference asks RDKit's periodic table)."""
import numpy as np
import torch

from .data import ProteinLigandData

# residue order of the reference's AA_NAME_SYM dict (utils/data.py:24-32): the amino-acid index is the dict position
AA_NAMES = ('ALA', 'CYS', 'ASP', 'GLU', 'PHE', 'GLY', 'HIS', 'ILE', 'LYS', 'LEU', 'MET', 'ASN', 'PRO', 'GLN', 'ARG', 'SER', 'THR',
            'VAL', 'TRP', 'TYR')
AA_INDEX = {n: i for i, n in enumerate(AA_NAMES)}
BACKBONE_NAMES = ('CA', 'C', 'N', 'O')
ATOMIC_NUMBER = {'H': 1, 'D': 1, 'C': 6, 'N': 7, 'O': 8, 'F': 9, 'Na': 11, 'Mg': 12, 'P': 15, 'S': 16, 'Cl': 17, 'K': 19, 'Ca': 20,
                 'Mn': 25, 'Fe': 26, 'Co': 27, 'Ni': 28, 'Cu': 29, 'Zn': 30, 'Se': 34, 'Br': 35, 'I': 53}
PROTEIN_ELEMENTS = (1, 6, 7, 8, 16, 34)            # utils/transforms.py:119 (H, C, N, O, S, Se)
MAX_NUM_AA = 20


def parse_pdb_atoms(block):
    """ATOM records of the first model -> dict of numpy arrays (element, pos, is_backbone, atom_name, atom_to_aa_type, molecule_name)."""
    element, pos, backbone, names, aa = [], [], [], [], []
    title = None
    for line in block.splitlines():
        tag = line[0:6].strip()
        if tag == 'ATOM':
            sym = line[76:78].strip().capitalize()
            if len(sym) == 0:
                sym = line[13:14]
            if sym not in ATOMIC_NUMBER:
                raise ValueError('unknown element %r in PDB line: %s' % (sym, line))
            res = line[17:20].strip()
            if res not in AA_INDEX:
                raise KeyError('non-standard residue %r (the reference raises KeyError here too, utils/data.py:113)' % res)
            name = line[12:16].strip()
            element.append(ATOMIC_NUMBER[sym])
            pos.append((float(line[30:38]), float(line[38:46]), float(line[46:54])))
            backbone.append(name in BACKBONE_NAMES)
            names.append(name)
            aa.append(AA_INDEX[res])
        elif tag == 'HEADER':
            title = line[10:].strip().lower()
        elif tag == 'ENDMDL':
            break
    return {'element': np.array(element, dtype=np.int64), 'molecule_name': title, 'pos': np.array(pos, dtype=np.float32).reshape(-1, 3),
            'is_backbone': np.array(backbone, dtype=bool), 'atom_name': names, 'atom_to_aa_type': np.array(aa, dtype=np.int64)}


def featurize_protein_atoms(element, atom_to_aa_type, is_backbone):
    """[N,27] int64: one-hot element (6) | one-hot amino acid (20) | backbone flag (utils/transforms.py:126-131)."""
    element = torch.as_tensor(element, dtype=torch.long)
    el = (element.view(-1, 1) == torch.tensor(PROTEIN_ELEMENTS).view(1, -1)).long()
    aa = torch.nn.functional.one_hot(torch.as_tensor(atom_to_aa_type, dtype=torch.long), num_classes=MAX_NUM_AA)
    bb = torch.as_tensor(is_backbone).view(-1, 1).long()
    return torch.cat([el, aa, bb], dim=-1)


def pdb_to_pocket_data(pdb_path_or_block):
    """Ligand-less ProteinLigandData for sampling into a pocket (scripts/sample_for_pocket.py:18-31), already featurized."""
    if '\n' in pdb_path_or_block:
        block = pdb_path_or_block
    else:
        with open(pdb_path_or_block, 'r') as f:
            block = f.read()
    d = parse_pdb_atoms(block)
    if len(d['element']) == 0:
        raise ValueError('no ATOM records found')
    data = ProteinLigandData(
        protein_element=torch.from_numpy(d['element']), protein_molecule_name=d['molecule_name'], protein_pos=torch.from_numpy(d['pos']),
        protein_is_backbone=torch.from_numpy(d['is_backbone']), protein_atom_name=d['atom_name'],
        protein_atom_to_aa_type=torch.from_numpy(d['atom_to_aa_type']),
        ligand_element=torch.empty([0], dtype=torch.long), ligand_pos=torch.empty([0, 3], dtype=torch.float))
    data.protein_atom_feature = featurize_protein_atoms(data.protein_element, data.protein_atom_to_aa_type, data.protein_is_backbone)
    return data


# index -> (atomic number, aromatic) of the 13 ligand classes, 'add_aromatic' mode (utils/transforms.py:48-62,69-90)
LIGAND_CLASS_TO_ATOM = ((1, False), (6, False), (6, True), (7, False), (7, True), (8, False), (8, True), (9, False), (15, False), (15, True),
                        (16, False), (16, True), (17, False))
# index -> atomic number of the 8 ligand classes, 'basic' mode (utils/transforms.py:37-46)
LIGAND_CLASS_TO_ATOM_BASIC = (1, 6, 7, 8, 9, 15, 16, 17)
# index -> (atomic number, hybridization, aromatic) of the 23 ligand classes, 'full' mode (utils/transforms.py:11-35)
LIGAND_CLASS_TO_ATOM_FULL = ((1, 'S', False), (6, 'SP', False), (6, 'SP2', False), (6, 'SP2', True), (6, 'SP3', False), (7, 'SP', False),
                             (7, 'SP2', False), (7, 'SP2', True), (7, 'SP3', False), (8, 'SP2', False), (8, 'SP2', True), (8, 'SP3', False),
                             (9, 'SP3', False), (15, 'SP2', False), (15, 'SP2', True), (15, 'SP3', False), (15, 'SP3D', False),
                             (16, 'SP2', False), (16, 'SP2', True), (16, 'SP3', False), (16, 'SP3D', False), (16, 'SP3D2', False),
                             (17, 'SP3', False))
# ligand_atom_mode -> the atomic number of each class
LIGAND_CLASS_ELEMENTS = {'basic': LIGAND_CLASS_TO_ATOM_BASIC, 'add_aromatic': tuple(z for z, _ in LIGAND_CLASS_TO_ATOM),
                         'full': tuple(z for z, _, _ in LIGAND_CLASS_TO_ATOM_FULL)}
ELEMENT_SYMBOL = {z: sym for sym, z in ATOMIC_NUMBER.items() if sym != 'D'}


def element_classes(symbols, mode='add_aromatic'):
    """Sorted class indices of `mode` whose element is one of `symbols` (e.g. ['C', 'N', 'O']): every class of an element, so that
    in 'add_aromatic' 'C' gives the aliphatic and the aromatic carbon, and in 'full' every hybridization.  ValueError for an unknown
    mode, an empty list, or a symbol that no class of the mode has (the message lists the mode's elements)."""
    if mode not in LIGAND_CLASS_ELEMENTS:
        raise ValueError('ligand_atom_mode %r (known: %s)' % (mode, sorted(LIGAND_CLASS_ELEMENTS)))
    zs = LIGAND_CLASS_ELEMENTS[mode]
    known = [ELEMENT_SYMBOL[z] for z in sorted(set(zs))]
    if isinstance(symbols, str):
        symbols = [symbols]
    symbols = list(symbols)
    if not symbols:
        raise ValueError('an element constraint needs at least one element (%s mode: %s)' % (mode, ', '.join(known)))
    want = set()
    for sym in symbols:
        z = ATOMIC_NUMBER.get(str(sym).strip().capitalize()) if isinstance(sym, str) else None
        if z not in zs:
            raise ValueError('element %r is not a ligand class of the %s mode (its elements: %s)' % (sym, mode, ', '.join(known)))
        want.add(z)
    return [c for c, z in enumerate(zs) if z in want]


def get_atomic_number_from_index(index, mode='add_aromatic'):
    assert mode == 'add_aromatic'
    return [LIGAND_CLASS_TO_ATOM[int(i)][0] for i in np.asarray(index).tolist()]


def is_aromatic_from_index(index, mode='add_aromatic'):
    assert mode == 'add_aromatic'
    return [LIGAND_CLASS_TO_ATOM[int(i)][1] for i in np.asarray(index).tolist()]
