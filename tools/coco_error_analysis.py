"""COCO error analysis of a result file on the device, in place of SipMask-mmdetection's tools/coco_error_analysis.py.

For every result type it computes the tool's seven precision arrays ps [7, R, K, 4, 1] (C75, C50, Loc, Sim, Oth, BG, FN;
see sipmask_b200.cocoeval.analyze_json) and writes, under OUT_DIR/<type>/:
  analysis.npz  : ps, recThrs, cat_ids, names
  analysis.txt  : the numbers the tool's plot legends show, per class and for all classes, per area range
  <type>-<class>-<area>.png / <type>-allclass-<area>.png : the tool's plots, when matplotlib is importable

Classes are indexed as p.catIds, the sorted category ids; the original tool indexes them in the file's order of
categories, which is the same order when the annotation file lists its categories sorted by id, as COCO's does.

    python tools/coco_error_analysis.py results.segm.json out/ --ann instances_val2017.json --types bbox segm
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


# fill colour of each error type's band, from the bottom band (C75) to the top one (FN)
BAND_COLOURS = {'C75': (1.0, 1.0, 1.0), 'C50': (1.0, 1.0, 1.0), 'Loc': (.31, .51, .74), 'Sim': (.75, .31, .30),
                'Oth': (.36, .90, .38), 'BG': (.50, .39, .64), 'FN': (1.0, .6, 0.0)}


def makeplot(rec_thrs, ps, out_dir, class_name, iou_type):
    """One PNG per area range, named <type>-<class>-<area>.png: the precision-recall curve of each error type (its mean
    over the classes in ps), drawn as stacked bands from the curve below it (zero under C75) up to its own curve, each
    band labelled '[mean precision]type'."""
    import matplotlib
    matplotlib.use('Agg')
    import matplotlib.pyplot as plt
    from sipmask_b200.cocoeval import ANALYSIS_AREAS, ANALYSIS_TYPES
    for a, area in enumerate(ANALYSIS_AREAS):
        sel = ps[..., a, 0].reshape(len(ANALYSIS_TYPES), len(rec_thrs), -1)       # [type, R, classes]
        curves = sel.mean(axis=2)
        means = sel.mean(axis=(1, 2))
        title = '%s-%s-%s' % (iou_type, class_name, area)
        fig, ax = plt.subplots()
        below = np.zeros(len(rec_thrs))
        for t, name in enumerate(ANALYSIS_TYPES):
            ax.plot(rec_thrs, curves[t], color='k', linewidth=0.5)
            ax.fill_between(rec_thrs, below, curves[t], color=BAND_COLOURS[name],
                            label='[{:.3f}]{}'.format(means[t], name))
            below = curves[t]
        ax.set(xlabel='recall', ylabel='precision', xlim=(0, 1), ylim=(0, 1), title=title)
        ax.legend()
        fig.savefig(os.path.join(out_dir, title + '.png'))
        plt.close(fig)


def table_text(t):
    head = '%-24s %-8s' % ('class', 'area') + ''.join('%8s' % n for n in t['types'])
    lines = [head]
    rows = [('allclass', t['allclass'])] + list(zip(t['names'], t['classes']))
    for name, v in rows:
        for a, area in enumerate(t['areas']):
            lines.append('%-24s %-8s' % (name[:24], area) + ''.join('%8.3f' % x for x in v[:, a]))
    return '\n'.join(lines) + '\n'


def main():
    ap = argparse.ArgumentParser(description='COCO error analysis on the device')
    ap.add_argument('result', help='result file (json)')
    ap.add_argument('out_dir', help='output directory')
    ap.add_argument('--ann', default='data/coco/annotations/instances_val2017.json', help='annotation file')
    ap.add_argument('--types', nargs='+', default=['bbox'], choices=['bbox', 'segm'], help='result types')
    a = ap.parse_args()
    from sipmask_b200 import cocoeval as C
    with open(a.ann) as f:
        gt = C.CocoGroundTruth(json.load(f))
    with open(a.result) as f:
        res = json.load(f)
    ps_by_type = C.analyze_json(gt, bbox_json=res if 'bbox' in a.types else None,
                                segm_json=res if 'segm' in a.types else None)
    try:
        import matplotlib  # noqa: F401
        plots = True
    except ImportError:
        plots = False
        print('matplotlib is not installed: writing the arrays and tables, no plots')
    rec_thrs = C.ANALYSIS_PARAMS.rec_thrs
    for t in a.types:
        out = os.path.join(a.out_dir, t)
        os.makedirs(out, exist_ok=True)
        ps = ps_by_type[t]
        np.savez(os.path.join(out, 'analysis.npz'), ps=ps, recThrs=rec_thrs, cat_ids=np.array(gt.cat_ids),
                 names=np.array(gt.names))
        text = table_text(C.analysis_table(ps, gt))
        with open(os.path.join(out, 'analysis.txt'), 'w') as f:
            f.write(text)
        print('%s:\n%s' % (t, text))
        if plots:
            for k, name in enumerate(gt.names):
                makeplot(rec_thrs, ps[:, :, k], out, name, t)
            makeplot(rec_thrs, ps, out, 'allclass', t)


if __name__ == '__main__':
    main()
